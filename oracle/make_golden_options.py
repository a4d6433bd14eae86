"""Golden vectors for the Matcher's optional flags (exact_count, find_time_range,
hashesfor), produced by the LIVE reference Matcher (audfprint_match.py:149-352) on the
databases and queries already stored in tests/golden/match.npz.

Needs a checkout of the reference (dpwe/audfprint) named by $AFP_REFERENCE:
    AFP_REFERENCE=<checkout> python oracle/make_golden_options.py
Only OUTPUT ARRAYS of the reference are stored; no reference source is copied.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["AFP_REFERENCE"])

import audfprint_match as ref_ma        # noqa: E402  (the reference)
import hash_table as ref_ht             # noqa: E402

from tests import cases                                        # noqa: E402
from tests.conftest import expand_table                        # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
# name -> (exact_count, find_time_range, window, threshcount, search_depth)
CONFIGS = {"tr": (False, True, 2, 5, 100), "ex": (True, False, 2, 5, 100),
           "extr": (True, True, 1, 3, 10), "trb": (False, True, 1, 2, 3)}


def main():
    gm = np.load(os.path.join(OUT, "match.npz"))
    out = {}
    for db in ("db", "db2"):
        table, counts, hashbits, depth, mtb, hpi = expand_table(gm, db)
        ht = ref_ht.HashTable(hashbits=hashbits, depth=depth, maxtime=1 << mtb)
        ht.table[:] = table
        ht.counts[:] = counts
        ht.names = ["track%d" % i for i in range(cases.DB_NTRACKS)]
        ht.hashesperid = np.array(hpi)
        for cfg, (exact, trange, window, thresh, sdepth) in CONFIGS.items():
            mt = ref_ma.Matcher()
            mt.window, mt.threshcount, mt.search_depth = window, thresh, sdepth
            mt.exact_count, mt.find_time_range = exact, trange
            out["cfg_" + cfg] = np.array([exact, trange, window, thresh, sdepth], np.int32)
            for j in range(cases.DB_QUERIES):
                for tag in ("clean", "noisy"):
                    key = "q%d_%s" % (j, tag)
                    q = gm[key + "/q"]
                    rows = mt.match_hashes(ht, q)
                    out["%s/%s/rows_%s" % (db, key, cfg)] = rows
                    if len(rows):
                        _, pairs = mt.match_hashes(ht, q, hashesfor=0)
                        out["%s/%s/pairs_%s" % (db, key, cfg)] = np.asarray(pairs, np.int64)
                    print(db, cfg, key, "rows", len(rows), rows[:1].tolist())
    np.savez_compressed(os.path.join(OUT, "match_options.npz"), **out)


if __name__ == "__main__":
    main()
