"""Golden rows of the reference's own mode search on the constructed families of
tests/k4_mode_cases.py: Matcher._approx_match_counts(hits, ids, rawcounts) (audfprint_match.py:241-312)
on each query's hits, with the candidate list in the project's order (k4_reference.candidates), so
that ranking ties play no part.  Once with find_time_range off and once on, at time_quantile 0.02
and 0.5.

Needs a checkout of the reference (dpwe/audfprint) named by $AFP_REFERENCE:
    AFP_REFERENCE=<checkout> python oracle/make_golden_k4_modes.py
Stores only OUTPUT arrays of the reference in tests/golden/k4_modes.npz, per family:
    <name>/rows  int32 (R, 7)  rows of every query, query after query (find_time_range off)
    <name>/roff  int64 (nq+1)  query offsets into rows
    <name>/t02, <name>/t50  int32 (R, 7)  the same with find_time_range on, quantile 0.02 / 0.5
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["AFP_REFERENCE"])

import audfprint_match as ref_ma                # noqa: E402

from tests import k4_mode_cases as mc           # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "k4_modes.npz")


def reference_rows(case, i, find_time_range=False, quantile=0.02):
    m = ref_ma.Matcher()
    m.window, m.threshcount, m.max_alignments_per_id = case.window, case.thresh, case.maxalign
    m.find_time_range, m.time_quantile = find_time_range, quantile
    ids, raw = case.candidates(i)
    return np.asarray(m._approx_match_counts(case.hits(i).astype(np.int32), ids, raw), np.int32).reshape(-1, 7)


def main():
    g = {}
    for case in mc.all_cases():
        nq = len(case.queries)
        for key, kw in (("rows", {}), ("t02", dict(find_time_range=True, quantile=0.02)),
                        ("t50", dict(find_time_range=True, quantile=0.5))):
            parts = [reference_rows(case, i, **kw) for i in range(nq)]
            g["%s/%s" % (case.name, key)] = np.concatenate(parts)
        g["%s/roff" % case.name] = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        print(case.name, nq, "queries", len(g["%s/rows" % case.name]), "rows")
    np.savez_compressed(OUT, **g)


if __name__ == "__main__":
    main()
