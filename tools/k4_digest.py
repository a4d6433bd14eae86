"""SHA-256 digests of the matcher's (K4) results: packed rows and their offsets, the 8-column
fast-kernel status, the general kernel's query count and, in publish mode, the candidate lists
and counts.  Every setting runs twice, by default (fast kernel, handing over to the general one)
and with force_general_kernel.  Two builds of K4 that compute the same results print the same
lines; run it on each and diff the output.

Under a hashed bitmap (> 2^20 ids) an id whose hash collides with another's joins the member set
when its bit is already set, so which of the two joins depends on which thread gets there first:
status columns 1-3 (members, member hits, admitted single-record ids) vary from run to run there
and are left out of that digest.  The rows do not depend on it.

Inputs are seeded: the table and query generators of tests/test_gpu_match_fast.py.  The settings
cover pruning of single-record ids, pass 3, a member-set-full handover, the hashed bitmap
(> 2^20 ids), search_depth > 1024, a query above 16,384 rows and publish mode.

    python tools/k4_digest.py
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from audfprint_b200 import Matcher  # noqa: E402
from tests.test_gpu_match_fast import as_ht, hpi_of, make_query, make_table, plant  # noqa: E402


def sha(*arrays):
    h = hashlib.sha256()
    for x in arrays:
        h.update(np.ascontiguousarray(x).tobytes())
    return h.hexdigest()[:16]


def run(name, ht, qs, publish=False, hashed=False, **params):
    packed = np.ascontiguousarray(np.concatenate(qs).astype(np.int32))
    qoff = np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.int64)
    for force in (False, True):
        m = Matcher()
        m.window, m.threshcount, m.search_depth = params.get("window", 2), params.get("thresh", 5), params.get("sdepth", 100)
        m.force_general_kernel = force
        if publish:
            rows, roff, cand, cnts = m._publish_call(ht, packed, qoff)
            k = cnts[:, 0]
            extra = " cand %s" % sha(cnts, *[cand[i, :k[i]] for i in range(len(qs))])
        else:
            res = m.match_batch(ht, (packed, qoff), sort=False)
            rows = np.concatenate(res) if res else np.zeros((0, 7), np.int32)
            roff = np.concatenate([[0], np.cumsum([len(r) for r in res])]).astype(np.int64)
            extra = ""
        st = Matcher.last_status(ht, len(qs))
        if hashed:
            st = st[:, [0, 4, 5, 6, 7]]
        print("%-18s %-7s rows %s status %s general %d%s" % (name, "general" if force else "default",
              sha(rows, roff), sha(st), Matcher.last_general_count(ht), extra), flush=True)


def main():
    hb, depth, mtb, nids = 19, 100, 12, 1 << 20
    table, counts = make_table(1, hb, depth, nids, mtb)
    rng = np.random.default_rng(2)
    qs = [make_query(100 + i, 650 + 30 * i, hb) for i in range(8)]
    for i, q in enumerate(qs):
        plant(table, counts, q, hb, depth, mtb, 5000 + i, 300 + 7 * i, 120, rng)
    hpi = hpi_of(table, counts, depth, mtb, nids)
    ht = as_ht(table, counts, hb, depth, mtb, hpi)
    run("pruned", ht, qs)
    run("publish", ht, qs, publish=True)
    run("depth>1024", ht, qs[:2], thresh=1, sdepth=1100)
    run("publish depth>1024", ht, qs[:2], publish=True, sdepth=1100)
    run("rows>16384", ht, [make_query(600, 17000, hb, tmax=4000)])

    light = hpi.copy()                      # short tracks outrank members with one hit: pass 3
    light[5000:5008] = 400
    pick = np.random.default_rng(4).choice(nids, size=300, replace=False)
    light[pick] = np.random.default_rng(5).integers(1, 3, size=300)
    run("pass3", as_ht(table, counts, hb, depth, mtb, light), qs[4:8], thresh=4)

    t2, c2 = make_table(11, 14, 64, 20000, mtb)      # few ids: the member set overflows
    ht2 = as_ht(t2, c2, 14, 64, mtb, hpi_of(t2, c2, 64, mtb, 20000))
    run("set-full", ht2, [make_query(501, 1500, 14), make_query(502, 20, 14, dup=0.0)])

    n3 = 1500000                                      # > 2^20 ids: hashed bitmap
    t3, c3 = make_table(7, hb, depth, n3, 11, fill=0.8)
    q3 = [make_query(400 + i, 750, hb) for i in range(4)]
    rng = np.random.default_rng(8)
    for i, q in enumerate(q3):
        plant(t3, c3, q, hb, depth, 11, 1400000 + i, 20 * i, 100, rng)
    ht3 = as_ht(t3, c3, hb, depth, 11, hpi_of(t3, c3, depth, 11, n3))
    run("hashed-bitmap", ht3, q3, hashed=True)
    run("hashed publish", ht3, q3, publish=True, hashed=True)


if __name__ == "__main__":
    main()
