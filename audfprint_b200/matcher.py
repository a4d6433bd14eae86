"""Matcher — drop-in mirror of audfprint_match.Matcher (audfprint_match.py:93-420)
whose probe / candidate ranking / time-offset histogramming run in libafp.so.

Host code keeps only what the reference does after the hot part: the final
`results[(-results[:, 1]).argsort(),]` ordering (the very NumPy call of
audfprint_match.py:335, so equal counts come out as they do in the reference on
the same machine), `max_returns` truncation and message formatting.

The optional second-wave flags (SURVEY.md §8f-4) exact_count and find_time_range run on the
device too: match_batch (and so match_hashes, match_file) makes one afp_match_options_batch
call, which ranks in publish mode and finishes the reference's per-candidate post-processing
(audfprint_match.py:149-244) without materialising the hits.  match_hashes(hashesfor=...) and
tables without a device copy of their own keep the host forms: the hits (afp_get_hits) and the
ranked candidate list (afp_match_batch, publish_candidates) from the device, finished with the
post-processing restated twice - query by query (_match_with_options: O(search_depth) small
NumPy calls per query, as in the reference) and for a whole batch in array operations
(_finish_options_batch).  tests/test_host_mirror_cpu.py holds the two equal row for row, and
tests/test_gpu_match_options.py holds the device finish to _match_with_options.
illustrate (matplotlib) is not provided.
"""
from __future__ import annotations

import ctypes as C
import time

import numpy as np

from . import _lib
from .analyzer import DeviceHashes


def timebits_breaks():
    """int64 [32]: entry k-1 is the smallest positive v for which the reference's key width
    ceil(log(v)/log(2)) (encpowerof2, audfprint_match.py:166) reaches k, evaluated with the very
    NumPy expression the host form uses.  The device counts the entries <= a query's largest
    time, so it reproduces the expression - its power-of-two shortfall included - without a log."""
    global _BREAKS
    if _BREAKS is None:
        def bits(v):
            return int(np.ceil(np.log(max(1, v)) / np.log(2)))
        out = np.empty(32, np.int64)
        for k in range(1, 33):
            # bits() is non-decreasing and reaches k at 2^(k-1) or 2^(k-1) + 1
            lo = 1 << (k - 1)
            out[k - 1] = next(v for v in (lo - 1, lo, lo + 1) if v >= 1 and bits(v) >= k)
            assert bits(out[k - 1] - 1) < k
        _BREAKS = out
    return _BREAKS


_BREAKS = None


class Matcher(object):
    """Provide matching for audfprint fingerprint queries to hash table."""

    # attribute -> default, as set by audfprint_match.py:96-122
    _REFERENCE_DEFAULTS = dict(window=1, threshcount=5, max_returns=1, search_depth=100,
                               sort_by_time=False, verbose=False, illustrate=False, exact_count=False,
                               find_time_range=False, time_quantile=0.02, illustrate_hpf=False,
                               max_alignments_per_id=100)

    def __init__(self):
        for attr, default in self._REFERENCE_DEFAULTS.items():
            setattr(self, attr, default)

    def _params(self):
        if self.illustrate:
            raise NotImplementedError("illustrate is not implemented (SURVEY.md §8f-4)")
        if int(self.threshcount) < 0:
            # the reference's rows are degenerate there (DESIGN.md §8)
            raise ValueError("threshcount must be >= 0, got %d" % int(self.threshcount))
        return _lib.MatcherParams(int(self.window), int(self.threshcount), int(self.search_depth),
                                  int(self.max_alignments_per_id), 0, 0,
                                  1 if getattr(self, "force_general_kernel", False) else 0)

    @staticmethod
    def _run(ctx, p, packed, nq, qoff, options=None, shard_qmax=None):
        """afp_match_batch - or afp_match_options_batch with options = (exact_count,
        find_time_range, time_quantile) - growing the per-query row capacity of the approximate
        rows when a query overflows it.  With shard_qmax (a device int32 [nq] tensor, or its
        address) the options call is afp_match_options_shard_rank instead: the ranking of one shard,
        whose finish waits for the all-reduce of shard_qmax."""
        with ctx.after_torch(packed, shard_qmax):          # torch tensors: written / read on torch's stream
            return Matcher._run_ordered(ctx, p, packed, nq, qoff, options, shard_qmax)

    @staticmethod
    def _run_ordered(ctx, p, packed, nq, qoff, options, shard_qmax):
        total = C.c_int64(0)
        cap = 256
        ptr, on_host = _lib.ptr_of(packed) if len(packed) else (None, 1)     # NumPy (host) or torch CUDA tensor
        qp = qoff.ctypes.data_as(C.POINTER(C.c_int64))
        if hasattr(shard_qmax, "data_ptr"):
            shard_qmax = shard_qmax.data_ptr()
        if options is not None:
            breaks = timebits_breaks()
        while True:
            p.row_capacity = cap
            try:
                if options is None:
                    ctx.check(ctx.lib.afp_match_batch(ctx.h, ptr, on_host, nq, qp, C.byref(p), C.byref(total)))
                else:
                    exact, trange, quant = options
                    args = (ctx.h, ptr, on_host, nq, qp, C.byref(p), int(bool(exact)), int(bool(trange)), float(quant),
                            breaks.ctypes.data_as(C.POINTER(C.c_int64)))
                    if shard_qmax is None:
                        ctx.check(ctx.lib.afp_match_options_batch(*args, C.byref(total)))
                    else:
                        ctx.check(ctx.lib.afp_match_options_shard_rank(*args, C.c_void_p(shard_qmax),
                                                                       C.byref(total)))
                return int(total.value)
            except _lib.RowCapacityError:
                # the reference emits at most max_alignments_per_id + 1 rows per candidate (:309-311)
                bound = max(1, p.search_depth) * (p.max_alignments_per_id + 1)
                if cap >= bound:
                    raise
                cap = min(cap * 8, bound)

    @staticmethod
    def last_general_count(ht):
        """Queries of the last device call that the general kernel (not the fast one) processed."""
        ctx = _lib.context(ht.device)
        n = C.c_int64(0)
        ctx.check(ctx.lib.afp_match_general_count(ctx.h, C.byref(n)))
        return int(n.value)

    @staticmethod
    def last_status(ht, nqueries):
        """int32 (nqueries, 8) of the last device call (afp_fetch_match_status): column 0 is 0 for the
        fast kernel; the reason the fast kernel handed the query to the general kernel: 1 member set
        full, 2 member-hit list full, 3 more than 2048 single-record ids admitted, 4 shard mode with
        > 2^20 ids and fewer members than search_depth, 5 candidate depth > 1024, 7 more than 2048
        members at or above the K-th member's weight bin, 8 internal consistency check; 6 = the
        long-query path (rows * depth >= 2^24, whether or not the fast kernel ran); -1 = the fast
        kernel did not run."""
        ctx = _lib.context(ht.device)
        st = np.zeros((max(nqueries, 1), 8), np.int32)
        ctx.check(ctx.lib.afp_fetch_match_status(ctx.h, st.ctypes.data))
        return st[:nqueries]

    def match_batch(self, ht, queries, sort=True):
        """Match many queries in one device call.

        queries  list of int32 (nq_i, 2) [time, hash] arrays (or one packed
                 (rows, offsets) tuple)
        returns  list of int32 (R_i, 7) rows [id, count, dtime, raw, rank, 0, 0],
                 sorted by count descending like match_hashes."""
        if isinstance(queries, tuple):
            packed, qoff = queries
            if not getattr(packed, "is_cuda", False):       # a torch CUDA tensor (int32 [R][2]) is used in place
                packed = np.ascontiguousarray(packed, dtype=np.int32).reshape(-1, 2)
            qoff = np.ascontiguousarray(qoff, dtype=np.int64)
        else:
            packed, qoff = _lib.pack_rows(queries)
        nq = len(qoff) - 1
        p = self._params()
        if (self.exact_count or self.find_time_range) and hasattr(ht, "_sync_device"):
            # one device call: ranking in publish mode, then the options' finish on the device
            ctx = ht._sync_device()
            total = self._run(ctx, p, packed, nq, qoff, (self.exact_count, self.find_time_range, self.time_quantile))
            rows, roff = self._fetch_rows(ctx, total, nq)
            if sort and len(rows):
                rows = self._sort_by_count(rows, roff)
            return [rows[roff[i]:roff[i + 1]] for i in range(nq)]
        if self.exact_count or self.find_time_range:
            # a table without a device copy of its own (only get_hits): TWO calls for the whole batch - the hits of every query row (afp_get_hits) and
            # the ranked candidate lists + approximate rows (afp_match_batch, publish mode) - then the
            # reference's per-candidate post-processing on the host, query by query
            if nq == 1:                          # match_hashes: the per-query form of the same two calls
                r = self._match_with_options(ht, packed)
                return [r[(-r[:, 1]).argsort(), ] if sort else r]
            hits = ht.get_hits(packed)
            mask = (1 << int(ht.hashbits)) - 1
            per_row = np.minimum(int(ht.depth), ht.counts[packed[:, 1].astype(np.int64) & mask]).astype(np.int64)
            hoff = np.concatenate([[0], np.cumsum(per_row)])[qoff]
            rows, roff, cand, cnts = self._publish_call(ht, packed, qoff)
            if self.threshcount >= 1:
                # the whole batch in one vectorised pass (no per-query Python work)
                out, ooff = self._finish_options_batch(hits, hoff, rows, roff, cand, cnts)
                if sort and len(out):
                    out = self._sort_by_count(out, ooff)
                return [out[ooff[i]:ooff[i + 1]] for i in range(nq)]
            out = []                             # threshcount < 1: empty offset bins can be modes
            for i in range(nq):
                pre = (hits[hoff[i]:hoff[i + 1]], rows[roff[i]:roff[i + 1]], cand[i], cnts[i])
                out.append(self._match_with_options(ht, packed[qoff[i]:qoff[i + 1]], device_results=pre))
            return [r[(-r[:, 1]).argsort(), ] for r in out] if sort else out
        ctx = ht._sync_device()
        rows, roff = self._fetch_rows(ctx, self._run(ctx, p, packed, nq, qoff), nq)
        if sort and len(rows):
            rows = self._sort_by_count(rows, roff)
        return [rows[roff[i]:roff[i + 1]] for i in range(nq)]

    @staticmethod
    def _fetch_rows(ctx, total, nq):
        """The `total` result rows of the last match call (int32 (total, 7)) and their query offsets."""
        rows = np.empty((total, 7), np.int32)
        roff = np.zeros(nq + 1, np.int64)
        ctx.check(ctx.lib.afp_fetch_match_rows(ctx.h, rows.ctypes.data if total else None, 1,
                                               roff.ctypes.data_as(C.POINTER(C.c_int64))))
        return rows, roff

    @staticmethod
    def _sort_by_count(rows, roff):
        """`results[(-results[:, 1]).argsort(),]` (audfprint_match.py:335) for every query of a batch.
        One vectorised pass orders all queries by count descending; only where a query has EQUAL
        counts (the reference's argsort is unstable, so their order is whatever NumPy does on this
        machine) is that query re-ordered with the reference's own per-query call."""
        q = np.repeat(np.arange(len(roff) - 1), np.diff(roff))
        order = np.lexsort((-rows[:, 1].astype(np.int64), q))
        out = rows[order]
        tied = np.nonzero((q[order][1:] == q[order][:-1]) & (out[1:, 1] == out[:-1, 1]))[0]
        for i in np.unique(q[order][tied]):
            r = rows[roff[i]:roff[i + 1]]
            out[roff[i]:roff[i + 1]] = r[(-r[:, 1]).argsort(), ]
        return out

    # ---- exact_count / find_time_range / hashesfor (audfprint_match.py:149-244) ----
    def _device_rows_and_candidates(self, ht, q):
        """One query through afp_match_batch in publish mode: the approximate rows (rank order)
        and the candidate list _best_count_ids would return (ids, rawcounts)."""
        rows, _, cand, cnts = self._publish_call(ht, q, np.array([0, len(q)], np.int64))
        depth = max(0, min(int(cnts[0, 1]), int(self.search_depth), int(cnts[0, 0])))
        rows = rows[rows[:, 4] < depth]          # publish mode also reports the ids past maxdepth
        return rows, cand[0, :depth, 0].astype(np.int64), cand[0, :depth, 1].astype(np.int64)

    def _support(self, hits_by_id, tid, mode):
        """Hits of track `tid` whose offset lies within `window` of `mode` (rows keep the
        query-time order of hits_by_id)."""
        h = hits_by_id.get(int(tid))
        if h is None:
            return np.zeros((0, 4), np.int32)
        return h[np.abs(h[:, 1].astype(np.int64) - int(mode)) <= self.window]

    def _time_range(self, hits_by_id, tid, mode):
        """Quantile-trimmed query-time support of one alignment (audfprint_match.py:173-195)."""
        t = self._support(hits_by_id, tid, mode)[:, 3]
        return (t[int(len(t) * self.time_quantile)],
                t[int(len(t) * (1.0 - self.time_quantile)) - 1])

    @staticmethod
    def _pair_keys(sup, timebits):
        """Distinct (query time, hash) pairs, packed as the reference packs them (:166-167)."""
        return np.unique(sup[:, 3] + (sup[:, 2].astype(np.int64) << timebits))

    @staticmethod
    def _split_by_id(hits):
        """{id: that id's hits in query-time order}."""
        if len(hits) == 0:
            return {}
        h = hits[np.lexsort((hits[:, 3], hits[:, 0]))]
        cut = np.nonzero(np.diff(h[:, 0]))[0] + 1
        return {int(part[0, 0]): part for part in np.split(h, cut)}

    def _match_with_options(self, ht, q, hashesfor=None, device_results=None):
        """Rows of match_hashes for exact_count / find_time_range (unsorted: candidate-rank
        order), plus the matching (time, hash) pairs of row `hashesfor` of the SORTED result.
        device_results = (hits, rows, cand, counts) of this query when match_batch already fetched
        them for the whole batch."""
        q = np.ascontiguousarray(q, dtype=np.int32).reshape(-1, 2)
        if device_results is None:
            hits = ht.get_hits(q)
            approx, ids, raws = self._device_rows_and_candidates(ht, q)
        else:
            hits, rows_q, cand_q, cnt_q = device_results
            depth = max(0, min(int(cnt_q[1]), int(self.search_depth), int(cnt_q[0])))
            approx = rows_q[rows_q[:, 4] < depth]
            ids, raws = cand_q[:depth, 0].astype(np.int64), cand_q[:depth, 1].astype(np.int64)
        by_id = self._split_by_id(hits)
        if not self.exact_count:
            rows = approx.copy()
            if self.find_time_range:
                for r in rows:
                    r[5], r[6] = self._time_range(by_id, r[0], r[2])
        else:
            timebits = 1
            if len(hits):
                timebits = max(1, int(np.ceil(np.log(max(1, int(hits[:, 3].max()))) / np.log(2))))
            out = []
            for rank, (tid, raw) in enumerate(zip(ids, raws)):
                dts = by_id[int(tid)][:, 1].astype(np.int64)
                base = int(dts.min())
                hist = np.bincount(dts - base)
                rises = np.r_[True, hist[1:] >= hist[:-1], False]          # locmax (:48-65)
                for mode in np.nonzero(rises[:-1] & ~rises[1:] & (hist >= self.threshcount))[0] + base:
                    count = len(self._pair_keys(self._support(by_id, tid, mode), timebits))
                    if count >= self.threshcount:
                        lo, hi = self._time_range(by_id, tid, mode) if self.find_time_range else (0, 0)
                        out.append([tid, count, mode, raw, rank, lo, hi])
            rows = np.array(out, np.int32).reshape(-1, 7)
        if hashesfor is None:
            return rows
        srt = rows[(-rows[:, 1]).argsort(), ]
        timebits = max(1, int(np.ceil(np.log(max(1, int(hits[:, 3].max()))) / np.log(2))))
        keys = self._pair_keys(self._support(by_id, srt[hashesfor, 0], srt[hashesfor, 2]), timebits)
        return rows, np.c_[keys & ((1 << timebits) - 1), keys >> timebits]

    def _finish_options_batch(self, hits, hoff, rows, roff, cand, cnts):
        """exact_count / find_time_range post-processing (audfprint_match.py:149-244) of a WHOLE
        batch in array operations - the same rows, in the same order, as _match_with_options
        query by query (needs threshcount >= 1: with 0 the reference also reports empty offset
        bins as modes, which only the dense per-query histogram represents).

        hits  (H,4) [id, dtime, hash, qtime] of all queries, hoff (nq+1) their offsets
        rows  (R,7) approximate rows of the publish-mode device call, roff (nq+1)
        cand  (nq, search_depth, 3) [id, raw, weight] ranked candidates, cnts (nq,2) [entries, n_above]
        Returns (rows (R',7) int32 in (query, candidate rank, offset) order, offsets (nq+1))."""
        nq = len(hoff) - 1
        win = int(self.window)
        depth = np.maximum(0, np.minimum(np.minimum(cnts[:, 1].astype(np.int64), int(self.search_depth)),
                                         cnts[:, 0].astype(np.int64)))
        empty = (np.zeros((0, 7), np.int32), np.zeros(nq + 1, np.int64))
        rq = np.repeat(np.arange(nq), np.diff(roff))
        if not self.exact_count:
            keep = rows[:, 4] < depth[rq]                      # publish mode also reports ids past maxdepth
            out, oq = rows[keep].copy(), rq[keep]
            ooff = np.concatenate([[0], np.cumsum(np.bincount(oq, minlength=nq))]).astype(np.int64)
            if not self.find_time_range or len(out) == 0:
                return out, ooff
            # groups = the distinct (query, id) pairs of the kept rows
            nid = int(max(out[:, 0].max(), hits[:, 0].max() if len(hits) else 0)) + 1
            pair = oq.astype(np.int64) * nid + out[:, 0].astype(np.int64)
            gkey, gidx = np.unique(pair, return_inverse=True)
            srt = self._sorted_group_hits(hits, hoff, gkey, np.arange(len(gkey)), nid, win)
            lo, hi = self._support_ranges(srt, gidx, out[:, 2].astype(np.int64), win)
            tlo, thi = self._range_quantiles(srt, lo, hi)
            out[:, 5], out[:, 6] = tlo, thi
            return out, ooff
        # ---- exact counts: groups = the ranked candidates, in (query, rank) order
        cq = np.repeat(np.arange(nq), depth)
        if len(cq) == 0 or len(hits) == 0:
            return empty
        crank = np.arange(len(cq)) - np.repeat(np.cumsum(depth) - depth, depth)
        cid = cand[cq, crank, 0].astype(np.int64)
        craw = cand[cq, crank, 1].astype(np.int64)
        nid = int(max(cid.max(), hits[:, 0].max())) + 1
        ckey = cq.astype(np.int64) * nid + cid
        perm = np.argsort(ckey, kind="stable")
        srt = self._sorted_group_hits(hits, hoff, ckey[perm], perm, nid, win)
        sg, sdt = srt["g"], srt["dt"]
        if len(sg) == 0:
            return empty
        # sparse offset histogram per group: runs of equal (group, offset)
        first = np.r_[True, (sg[1:] != sg[:-1]) | (sdt[1:] != sdt[:-1])]
        start = np.nonzero(first)[0]
        ug, udt = sg[start], sdt[start]
        ucnt = np.diff(np.r_[start, len(sg)])
        adj_prev = np.r_[False, (ug[1:] == ug[:-1]) & (udt[1:] == udt[:-1] + 1)]
        prev = np.where(adj_prev, np.r_[0, ucnt[:-1]], 0)
        nxt = np.where(np.r_[adj_prev[1:], False], np.r_[ucnt[1:], 0], 0)
        # local maximum of the dense histogram (locmax, audfprint_match.py:48-65) that reaches threshcount
        is_mode = (ucnt >= prev) & (nxt < ucnt) & (ucnt >= int(self.threshcount))
        mg, mode = ug[is_mode], udt[is_mode]
        if len(mg) == 0:
            return empty
        lo, hi = self._support_ranges(srt, mg, mode, win)
        # distinct (query time, hash) pairs inside every support (_unique_match_hashes, :149-171)
        ln = hi - lo
        mj = np.repeat(np.arange(len(mg)), ln)
        src = np.repeat(lo, ln) + (np.arange(int(ln.sum())) - np.repeat(np.cumsum(ln) - ln, ln))
        # packed exactly as the reference packs them: query time + (hash << bits of the query's
        # largest time), encpowerof2 included - a largest time that is a power of two gets one bit
        # too few there, and the (rare) collisions that follow are part of the reference's count
        qmax = np.zeros(nq, np.int64)
        nonempty = np.nonzero(np.diff(hoff))[0]
        if len(nonempty):
            qmax[nonempty] = np.maximum.reduceat(hits[:, 3].astype(np.int64), hoff[nonempty])
        bits_of = {int(m): max(1, int(np.ceil(np.log(max(1, int(m))) / np.log(2)))) for m in np.unique(qmax)}
        tbits = np.array([bits_of[int(m)] for m in qmax], np.int64)[cq[mg]]
        pk = srt["qt"][src].astype(np.int64) + (srt["hash"][src].astype(np.int64) << tbits[mj])
        o = np.lexsort((pk, mj))
        mjs, pks = mj[o], pk[o]
        new = np.r_[True, (mjs[1:] != mjs[:-1]) | (pks[1:] != pks[:-1])]
        count = np.bincount(mjs[new], minlength=len(mg))
        good = count >= int(self.threshcount)
        out = np.zeros((int(good.sum()), 7), np.int32)
        g = mg[good]
        out[:, 0], out[:, 1], out[:, 2], out[:, 3], out[:, 4] = cid[g], count[good], mode[good], craw[g], crank[g]
        if self.find_time_range and len(out):
            out[:, 5], out[:, 6] = self._range_quantiles(srt, lo[good], hi[good])
        ooff = np.concatenate([[0], np.cumsum(np.bincount(cq[g], minlength=nq))]).astype(np.int64)
        return out, ooff

    @staticmethod
    def _sorted_group_hits(hits, hoff, sorted_keys, group_of_key, nid, win):
        """Hits that belong to one of the (query, id) groups, ordered by (group, offset, query time).
        sorted_keys: ascending query * nid + id of the groups; group_of_key: group number of each."""
        hq = np.repeat(np.arange(len(hoff) - 1), np.diff(hoff))
        hk = hq.astype(np.int64) * nid + hits[:, 0].astype(np.int64)
        pos = np.minimum(np.searchsorted(sorted_keys, hk), len(sorted_keys) - 1)
        sel = np.nonzero(sorted_keys[pos] == hk)[0]
        g = np.asarray(group_of_key)[pos[sel]].astype(np.int64)
        dt = hits[sel, 1].astype(np.int64)
        qt = hits[sel, 3].astype(np.int64)
        o = np.lexsort((qt, dt, g))
        g, dt = g[o], dt[o]
        dmin = int(dt.min()) if len(dt) else 0
        span = (int(dt.max()) - dmin if len(dt) else 0) + 2 * win + 4
        # one ascending key for bisection: group-major, offset-minor, with room for +-window probes
        return {"g": g, "dt": dt, "qt": qt[o], "hash": hits[sel, 2][o], "dmin": dmin, "span": span,
                "key": g * span + (dt - dmin + win + 1)}

    @staticmethod
    def _support_ranges(srt, group, mode, win):
        """[lo, hi) into the sorted hits: the entries of `group` within `win` of offset `mode`."""
        base = group.astype(np.int64) * srt["span"] + (mode - srt["dmin"] + win + 1)
        return (np.searchsorted(srt["key"], base - win, side="left"),
                np.searchsorted(srt["key"], base + win, side="right"))

    def _range_quantiles(self, srt, lo, hi):
        """Quantile-trimmed query-time support of every [lo, hi) range (_calculate_time_ranges,
        audfprint_match.py:173-195): the times in ascending order, the reference's two indices."""
        ln = hi - lo
        j = np.repeat(np.arange(len(lo)), ln)
        src = np.repeat(lo, ln) + (np.arange(int(ln.sum())) - np.repeat(np.cumsum(ln) - ln, ln))
        t = srt["qt"][src]
        t = t[np.lexsort((t, j))]
        base = np.cumsum(ln) - ln
        i_lo = (ln * float(self.time_quantile)).astype(np.int64)
        i_hi = (ln * (1.0 - float(self.time_quantile))).astype(np.int64) - 1
        i_hi = np.where(i_hi < 0, i_hi + ln, i_hi)               # Python's negative index
        return t[base + i_lo], t[base + i_hi]

    def _publish_call(self, ht, qrows, qoff):
        """afp_match_batch with publish_candidates: (rows (R,7) with LOCAL ranks, row offsets,
        cand (nq, search_depth, 3) f64 [id, raw, weight], counts (nq, 2) i32 [entries, n_above])."""
        nq = len(qoff) - 1
        p = self._params()
        p.publish_candidates = 1
        ctx = ht._sync_device()
        rows, roff = self._fetch_rows(ctx, self._run(ctx, p, qrows, nq, qoff), nq)
        cand = np.zeros((nq, max(int(self.search_depth), 1), 3), np.float64)
        cnts = np.zeros((nq, 2), np.int32)
        if nq:
            ctx.check(ctx.lib.afp_fetch_match_candidates(ctx.h, cand.ctypes.data, cnts.ctypes.data, 1))
        return rows, roff, cand, cnts

    def match_batch_shard(self, ht, queries):
        """Table-shard side of a sharded match (SURVEY.md §8e): `ht`'s device copy holds only
        this rank's id range.  Returns one record per query for dist.merge_sharded_results:
        {"n_above", "cand" (k,3) [id, raw, weight], "rows" (r,7) with LOCAL ranks}."""
        packed, qoff = _lib.pack_rows(queries)
        rows, roff, cand, cnts = self._publish_call(ht, packed, qoff)
        return [{"n_above": int(cnts[i, 1]), "cand": cand[i, :cnts[i, 0]].copy(),
                 "rows": rows[roff[i]:roff[i + 1]].copy()} for i in range(len(qoff) - 1)]

    def match_batch_shard_packed(self, ht, packed_queries, row_cap=16):
        """match_batch_shard for a packed (rows, offsets) query batch, returning the fixed-size
        float64 records (nq, W) that dist.allgather exchanges — no per-query Python work."""
        from . import dist as afd
        qrows, qoff = packed_queries
        if not getattr(qrows, "is_cuda", False):        # a torch CUDA tensor (int32 [R][2]) is used in place
            qrows = np.ascontiguousarray(qrows, dtype=np.int32).reshape(-1, 2)
        qoff = np.ascontiguousarray(qoff, dtype=np.int64)
        rows, roff, cand, cnts = self._publish_call(ht, qrows, qoff)
        return afd.pack_shard_batch(cand, cnts, rows, roff, row_cap)

    def match_hashes(self, ht, hashes, hashesfor=None):
        """Query hashes -> rows (id, filteredmatches, timoffs, rawmatches, origrank,
        mintime, maxtime), best first (audfprint_match.py:314-352)."""
        q = np.asarray(hashes, dtype=np.int32).reshape(-1, 2)
        if hashesfor is None:
            return self.match_batch(ht, [q])[0]
        self._params()
        rows, pairs = self._match_with_options(ht, q, hashesfor)
        return rows[(-rows[:, 1]).argsort(), ], pairs

    def match_file(self, analyzer, ht, filename, number=None):
        """Read, fingerprint and match one file -> (rows[:max_returns], duration in s, #hashes)
        (audfprint_match.py:354-379): match_files' driver over the one file."""
        return self._match_files(analyzer, ht, [filename], [number])[0][0]

    @staticmethod
    def _print_analyzed(filename, number, seconds, nhashes):
        tag = "#%d" % number if number is not None else ""
        print(time.ctime(), "Analyzed", tag, filename, "of", ('%.3f' % seconds), "s "
              "to", nhashes, "hashes")

    # files per wavfiles2hashes + match_batch round of match_files
    max_files_per_call = 2048

    def match_files(self, analyzer, ht, filenames, start=0):
        """List form of match_file, file i numbered start + i: the same (rows[:max_returns], seconds,
        nhashes) per file, and the verbose "Analyzed" lines in list order.  Every round of
        max_files_per_call files is one Analyzer.wavfiles2hashes and one match_batch; when the
        analyzer and the table share a device the hashes go from the fingerprint workspace to the
        matcher without leaving it (afp_fetch_hashes into device memory).

        With analyzer.fail_on_error, an unreadable file raises the IOError match_file raises and
        leaves the analyzer's counters as they were; nothing is returned (the per-file loop would
        have matched the earlier files by then)."""
        return analyzer._list_form(lambda: self._match_files(analyzer, ht, filenames,
                                                             range(start, start + len(filenames))))

    def _match_files(self, analyzer, ht, filenames, numbers):
        """The driver of match_file and match_files -> (match_file's tuple, duration) per file."""
        self._params()                     # illustrate raises before any file is read
        durs = []
        on_device = hasattr(ht, "_sync_device") and _lib.context(ht.device) is _lib.context(analyzer.device)
        out = []
        for c0 in range(0, len(filenames), max(1, int(self.max_files_per_call))):
            names = filenames[c0:c0 + max(1, int(self.max_files_per_call))]
            queries, round_durs = analyzer._hashes_of_files(names, rows_on_device=on_device)
            durs += round_durs
            secs = []
            for fn, num, q in zip(names, numbers[c0:c0 + len(names)], queries):
                nh = len(q)
                last = q.last_time if isinstance(q, DeviceHashes) else (q[-1][0] if nh else None)
                secs.append(analyzer.n_hop * last / analyzer.target_sr if nh else 0.0)
                if self.verbose:
                    self._print_analyzed(fn, num, secs[-1], nh)
            for q, sec, rows in zip(queries, secs, self.match_batch(ht, self._pack_queries(queries, on_device))):
                if self.sort_by_time:
                    rows = rows[(-rows[:, 2]).argsort(), :]
                out.append((rows[:self.max_returns, :], sec, len(q)))
        return out, durs

    @staticmethod
    def _pack_queries(queries, on_device):
        """Queries -> what match_batch takes: a host list, or one packed (device rows, offsets) tuple."""
        if not on_device:
            return [q for q in queries]
        import torch
        dev = next((q.rows.device for q in queries if isinstance(q, DeviceHashes)), None)
        parts = [q.rows if isinstance(q, DeviceHashes)
                 else torch.from_numpy(np.asarray(q, np.int32).reshape(-1, 2)) for q in queries]
        if dev is None:
            return [np.asarray(q, np.int32).reshape(-1, 2) for q in queries]
        qoff = np.zeros(len(parts) + 1, np.int64)
        qoff[1:] = np.cumsum([len(p) for p in parts])
        packed = torch.cat([p.to(dev) for p in parts]) if qoff[-1] else torch.zeros((0, 2), dtype=torch.int32, device=dev)
        # match_batch orders its read of `packed` after the copies and the concatenation on torch's stream
        return packed.contiguous(), qoff

    def file_match_to_msgs(self, analyzer, ht, qry, number=None):
        """Match one file and format the reference's report lines
        (audfprint_match.py:381-420)."""
        rows, seconds, nhashes = self.match_file(analyzer, ht, qry, number)
        return self._msgs(analyzer, ht, qry, rows, seconds, nhashes)

    def files_match_to_msgs(self, analyzer, ht, filenames, start=0):
        """List form of file_match_to_msgs (match_files, file i numbered start + i): one list of
        report lines per file, in list order."""
        return analyzer._list_form(lambda: self._files_msgs(analyzer, ht, filenames,
                                                            range(start, start + len(filenames))))

    def _files_msgs(self, analyzer, ht, filenames, numbers):
        """The driver of files_match_to_msgs -> (report lines, duration) per file."""
        res, durs = self._match_files(analyzer, ht, filenames, numbers)
        return [self._msgs(analyzer, ht, fn, *r) for fn, r in zip(filenames, res)], durs

    def _msgs(self, analyzer, ht, qry, rows, seconds, nhashes):
        frame_s = analyzer.n_hop / analyzer.target_sr
        head = qry
        if self.verbose:
            head += (' %.1f ' % seconds) + "sec " + str(nhashes) + " raw hashes"
        if len(rows) == 0:
            return ["NOMATCH " + head if self.verbose else head + "\t"]
        if not self.verbose:
            return [head + "\t" + ht.names[row[0]] for row in rows]
        msgs = []
        for tid, aligned, dtime, raw, rank, t_lo, t_hi in rows:
            if self.find_time_range:
                # -R report: matched span of the query and where it starts in the reference track
                # (audfprint_match.py:402-407)
                msg = "Matched {:6.1f} s starting at {:6.1f} s in {:s} to time {:6.1f} s in {:s}".format(
                    (t_hi - t_lo) * frame_s, t_lo * frame_s, qry, (t_lo + dtime) * frame_s, ht.names[tid])
            else:
                msg = "Matched {:s} as {:s} at {:6.1f} s".format(head, ht.names[tid], dtime * frame_s)
            msgs.append(msg + " with {:5d} of {:5d} common hashes at rank {:2d}".format(aligned, raw, rank))
        return msgs
