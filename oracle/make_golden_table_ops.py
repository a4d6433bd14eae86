"""Golden vectors for the host-side table bookkeeping (merge / remove / slot reuse / retrieve /
list), produced by the LIVE reference HashTable (hash_table.py:91-138, 291-391) on the track
hashes already stored in tests/golden/match.npz.

Needs a checkout of the reference (dpwe/audfprint) named by $AFP_REFERENCE:
    AFP_REFERENCE=<checkout> python oracle/make_golden_table_ops.py
Only OUTPUT ARRAYS of the reference are stored; no reference source is copied.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["AFP_REFERENCE"])

import hash_table as ref_ht             # noqa: E402  (the reference)

from oracle.make_golden_table_ops_replay import run     # noqa: E402
from tests import cases                 # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def main():
    gm = np.load(os.path.join(OUT, "match.npz"))
    out = {}

    def record(tag, ht):
        out[tag + "/table"] = ht.table.copy()
        out[tag + "/counts"] = ht.counts.copy()
        out[tag + "/hashesperid"] = np.asarray(ht.hashesperid).copy()
        out[tag + "/names"] = np.array(["" if n is None else n for n in ht.names])
    _, r9, rlate, lines = run(ref_ht.HashTable, gm, record)
    out["retrieve_track9"], out["retrieve_late"] = r9, rlate
    out["list_lines"] = np.array(lines)
    for k in ("a", "b", "merged", "removed", "reused"):
        c = out[k + "/counts"]
        print(k, "entries", int(c.sum()), "overfull buckets", int(np.sum(c > cases.TABLE_OPS_DEPTH)),
              "names", len(out[k + "/names"]))
    print("retrieve", r9.shape, rlate.shape, lines[:2], lines[-1])
    np.savez_compressed(os.path.join(OUT, "table_ops.npz"), **out)


if __name__ == "__main__":
    main()
