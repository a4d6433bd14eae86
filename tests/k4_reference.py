"""Reference for K4's ranked candidate list and its rows, for tables of any size.

It composes the oracle's own functions (oracle/afp_oracle.py): the hits of `orc.get_hits` (stated
here in NumPy for large queries, `hits`), the ranking of `orc.rank_candidates` and the mode search
of `orc.offset_histogram_rows` (stated per id in NumPy, `rows_in_rank_order`).
`tests/test_k4_reference_cpu.py` shows it equal to `orc.match_hashes` / `orc.rank_candidates` and to
`dist.merge_sharded_results`' view of one shard, so that `tests/test_gpu_k4_ranking_edges.py` can hold
the device's candidate lists, in order, to it on constructed tables.

Candidate order is (weight desc, id desc), weight = raw / hashesperid as a double
(audfprint_match.py:136-146 with the project's tie rule); hashesperid 0 gives weight inf.
"""
from __future__ import annotations

import numpy as np

from oracle import afp_oracle as orc


def np_hits(table, counts, hashbits, depth, mtb, q):
    """(ids, dtimes) of every hit in (query row, slot) order, as orc.get_hits."""
    q = np.asarray(q, np.int64).reshape(-1, 2)
    b = q[:, 1] & ((1 << hashbits) - 1)
    n = np.minimum(depth, counts[b]).astype(np.int64)
    rep = np.repeat(np.arange(len(q)), n)
    slot = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    v = table[b[rep], slot].astype(np.int64)
    return (v >> mtb) - 1, (v & ((1 << mtb) - 1)) - q[rep, 0]


def hits(table, counts, hashbits, depth, mtb, q):
    """int64 (N, 4) [id, dtime, bucket, qtime] - orc.get_hits, vectorised."""
    q = np.asarray(q, np.int64).reshape(-1, 2)
    b = q[:, 1] & ((1 << hashbits) - 1)
    n = np.minimum(depth, counts[b]).astype(np.int64)
    ids, dts = np_hits(table, counts, hashbits, depth, mtb, q)
    rep = np.repeat(np.arange(len(q)), n)
    return np.stack([ids, dts, b[rep], q[rep, 0]], axis=1)


def candidates(h, hpi, thresh, sdepth, publish=False):
    """The ranked candidate list of hits `h` (orc.rank_candidates): (ids, raw, weight) in
    (weight desc, id desc) order, depth min(n_above, sdepth) - or, publish=True, the list a table
    shard publishes: depth min(#distinct ids, sdepth), and also (entries, n_above)."""
    hpi = np.asarray(hpi)
    with np.errstate(divide="ignore"):
        ids, raw = orc.rank_candidates(h, hpi, -1 if publish else thresh, sdepth)
        w = raw / hpi[ids].astype(float)
    ids, raw = ids.astype(np.int64), raw.astype(np.int64)
    if not publish:
        return ids, raw, w
    n_above = int(np.count_nonzero(np.unique(h[:, 0], return_counts=True)[1] > thresh))
    return ids, raw, w, (len(ids), n_above)


def rows_in_rank_order(h, ids, raws, window, thresh, maxalign=100):
    """orc.offset_histogram_rows: rows [id, count, dtime, raw, rank, 0, 0] of the ranked
    candidates, in rank order (before the final sort by count).  Each id's histogram starts at its
    own smallest dtime instead of the query's: the bins below are empty and change nothing as long
    as threshcount >= 0 (an empty bin is then never a mode).  With threshcount < 0 the reference
    also reports empty bins below the id's own range; the project refuses such a threshcount."""
    if len(h) == 0:
        return np.zeros((0, 7), np.int32)
    by_id = np.argsort(h[:, 0], kind="stable")
    sid, sdt = h[by_id, 0], h[by_id, 1]
    rows = []
    for rank, (id_, r) in enumerate(zip(ids, raws)):
        if r <= thresh:                   # no dtime bin can exceed threshcount
            continue
        lo, hi = np.searchsorted(sid, [id_, id_ + 1])
        d = sdt[lo:hi]
        tmin = int(d.min())
        bc = np.bincount(d - tmin)
        lm = np.where(orc.local_max_mask(bc), bc, 0)
        found = 0
        while True:
            mode = int(np.argmax(lm))
            if lm[mode] <= thresh:
                break
            a, b = max(0, mode - window), mode + window + 1
            rows.append([int(id_), int(bc[a:b].sum()), mode + tmin, int(r), rank, 0, 0])
            lm[a:b] = 0
            found += 1
            if found > maxalign:
                break
    return np.array(rows, np.int32).reshape(-1, 7)


def np_rows(table, counts, hashbits, depth, mtb, hpi, q, window, thresh, sdepth, maxalign=100):
    """Rows of orc.match_hashes in rank order (not sorted by count), vectorised."""
    h = hits(table, counts, hashbits, depth, mtb, q)
    if len(h) == 0:
        return np.zeros((0, 7), np.int32)
    ids, raw, _ = candidates(h, hpi, thresh, sdepth)
    return rows_in_rank_order(h, ids, raw, window, thresh, maxalign)


def by_count(rows):
    """The final sort of orc.match_hashes (count descending, stable)."""
    return rows[np.argsort(-rows[:, 1], kind="stable")]
