"""Constructed queries for the last step of K4: each ranked candidate's dtime histogram, its local
maxima, the repeated first arg-max above threshcount, the +-window count and clear and the
max_alignments_per_id cap (audfprint_match.py:280-311; candidate_modes, block_argmax, max_repeat
and candidates_finish in csrc/afp_match_common.cuh, and the long path's driver).

Every family is a Case: a table built with tests/test_gpu_k4_ranking_edges.py's Scene, one or more
queries, the matcher parameters, the paths that can take them, and a check that the edge the
family exists for is reached on the reference side (k4_reference's rows).  place() gives an id a
chosen histogram {dtime: count}, mixing the three ways a hit arises:
  * spread: one record per hit, each in a bucket probed once;
  * mult:   one record in a bucket probed m times at one query time (bucket multiplicity m);
  * probe:  one record in a bucket probed at several query times, so that one bucket group
            yields several dtimes (the per-row query times of the group are what the fast
            kernel's qkeys[r + k] and the long path's key[r + k] read).
The default, mix, puts an id's first and last bin in one probe bucket and gives the bins between
spread and mult in turn.
Planted ids get hashesperid = raw * (1000 + k) for the k-th planted id, so the rank order is the
planting order with no weight tie (ranking ties are tests/test_gpu_k4_ranking_edges.py's job).

Used by tests/test_gpu_k4_mode_edges.py (device == reference), tests/test_k4_modes_cpu.py
(reference == tests/golden/k4_modes.npz) and oracle/make_golden_k4_modes.py."""
from __future__ import annotations

from collections import Counter

import numpy as np

from tests import k4_reference as k4
from tests.test_gpu_k4_ranking_edges import Scene

ALL = ("fast", "general", "long")
NOFAST = ("general", "long")            # more member hits in one warp than the fast kernel holds, or threshcount 0
WINDOWS = (0, 1, 2, 511, 512, 4096)
TIE_GAPS = (2, 31, 32, 33, 1023, 1024, 1025, 2048)


class Case:
    """queries: int32 (n, 2) arrays matched in one call.  long_only: indices of the queries the
    "mixed" path pads onto the long path (the others stay short).  calls > 1: the queries are
    matched one per call, in order, with the same scratch layout."""

    def __init__(self, name, sc, queries, window, thresh, maxalign=100, sdepth=100, paths=ALL, check=None,
                 long_only=None, calls=1):
        self.name, self.sc, self.queries = name, sc, [np.ascontiguousarray(q, np.int32) for q in queries]
        self.window, self.thresh, self.maxalign, self.sdepth = window, thresh, maxalign, sdepth
        self.paths, self.check, self.long_only, self.calls = paths, check, long_only, calls

    def hits(self, i):
        sc = self.sc
        return k4.hits(sc.table, sc.counts, sc.hashbits, sc.depth, sc.mtb, self.queries[i])

    def candidates(self, i):
        ids, raw, _ = k4.candidates(self.hits(i), self.sc.hpi, self.thresh, self.sdepth)
        return ids, raw

    def rows(self, i):
        """k4_reference's rows of query i, in rank order."""
        ids, raw = self.candidates(i)
        return k4.rows_in_rank_order(self.hits(i), ids, raw, self.window, self.thresh, self.maxalign)


def place(sc, id_, hist, how="mix"):
    """Give id_ the dtime histogram `hist` ({dtime: count}).  how = spread | mult | probe (the probe
    bins share one bucket), or mix: first and last bin probe, the others spread and mult in turn."""
    probe = []
    items = sorted(hist.items())
    for i, (d, c) in enumerate(items):
        w = how if how != "mix" else "probe" if i in (0, len(items) - 1) else ("spread", "mult")[i % 2]
        qt = max(0, -d)
        if w == "probe":
            probe.append((d, c))
        elif w == "spread":
            for _ in range(c):
                sc.group([id_], 1, qt, d)
        else:
            sc.group([id_], c, qt, d)
    if probe:
        top = max(0, max(d for d, _ in probe))
        b = sc.group([id_], 0, 0, top)                   # entry time `top`, probed at top - d
        for d, c in probe:
            for _ in range(c):
                sc.probe(b, top - d)


def plant(sc, hists, how="mix", first=1):
    """Ids first, first + 1, ... get hists[k]; returns the ids."""
    ids = []
    for k, h in enumerate(hists):
        id_ = first + k
        place(sc, id_, h, how)
        sc.hpi[id_] = sum(h.values()) * (1000 + k)
        ids.append(id_)
    return ids


def hsum(*parts):
    """{dtime: count} of several (dtime, count) pairs, adding the counts of equal dtimes."""
    c = Counter()
    for d, n in parts:
        c[d] += n
    return dict(c)


def scene(**kw):
    kw.setdefault("hashbits", 14)
    kw.setdefault("nids", 1 << 12)
    return Scene(**kw)


def modes(rows, id_):
    return [int(r[2]) for r in rows if r[0] == id_]


def counts(rows, id_):
    return [int(r[1]) for r in rows if r[0] == id_]


# ---- families -----------------------------------------------------------------------------------
def local_max():
    """Plateaus of 2 and 3 bins (the right bin is the mode), at the id's first and last bin,
    v == left > right and left < v == right, rising and falling ramps, one bin and [k, k]."""
    sc = scene()
    hists = [{10: 3, 11: 5, 12: 5, 13: 2}, {20: 4, 21: 4, 22: 4, 23: 1}, {5: 6, 6: 6, 7: 2}, {30: 2, 31: 7, 32: 7},
             {0: 1, 1: 2, 2: 3, 3: 4, 4: 5}, {0: 5, 1: 4, 2: 3, 3: 2, 4: 1}, {7: 3}, {8: 3, 9: 3}]
    ids = plant(sc, hists)
    want = [12, 22, 6, 32, 4, 0, 7, 9]

    def check(r):
        assert [modes(r[0], i) for i in ids] == [[m] for m in want]
    return Case("local_max", sc, [sc.query()], 0, 1, maxalign=5, check=check)


def argmax_ties():
    """Equal maxima TIE_GAPS bins apart (same lane, other lanes, other warps, the same thread on a
    later stride of block_argmax), from the id's first bin and from one bin further in; a tie that
    appears only after the top bin is cleared.  window 0: the lower dtime comes first."""
    sc = scene()
    hists = [{100: 4, 100 + g: 4} for g in TIE_GAPS] + [{90: 1, 100: 4, 100 + g: 4} for g in TIE_GAPS]
    hists += [{100: 9, 300: 5, 600: 5}, {50: 6, 51: 1, 1074: 6}]
    ids = plant(sc, hists)
    n = len(TIE_GAPS)

    def check(r):
        for k, g in enumerate(TIE_GAPS):
            assert modes(r[0], ids[k]) == modes(r[0], ids[n + k]) == [100, 100 + g]
        assert modes(r[0], ids[-2]) == [100, 300, 600] and modes(r[0], ids[-1]) == [50, 1074]
    return Case("argmax_ties", sc, [sc.query()], 0, 1, maxalign=3, check=check)


def threshold(thresh):
    """threshcount 5: local maxima equal to it (no row) and one above; a candidate whose raw count
    is above it with every bin at or below it (the quick filter rejects it); a top bin of exactly
    threshcount + 1.  threshcount 1: bins of 1 and 2.  threshcount 0 (general kernel and long path
    only): every non-empty local maximum is a mode."""
    sc = scene()
    if thresh == 5:
        hists = [{100: 5, 110: 6, 120: 5, 130: 7}, {100: 3, 200: 3}, {300: 6, 305: 2}]
        want = [[130, 110], [], [300]]
    elif thresh == 1:
        hists = [{10: 2, 20: 1, 30: 2, 31: 1}, {5: 1, 50: 1}, {7: 2}]
        want = [[10, 30], [], [7]]
    else:
        hists = [{10: 1, 12: 1, 20: 2}, {40: 1}]
        want = [[20, 10, 12], [40]]
    ids = plant(sc, hists)

    def check(r):
        cand, raw = r.cand[0]
        assert [modes(r[0], i) for i in ids] == want
        assert np.all(np.isin(ids, cand)) and np.all(raw > thresh)
    return Case("thresh_%d" % thresh, sc, [sc.query()], 1, thresh, paths=ALL if thresh else NOFAST, check=check)


def window(w):
    """A second maximum exactly `window` away (counted and cleared) and window + 1 away (kept); two
    modes whose count windows overlap; a window wider than the id's span.  For window >= 512,
    2 * window + 1 > 1024 threads: the count and clear loops take several strides."""
    sc = scene()
    hists = [{1000: 9, 1000 + w: 5} if w else {1000: 9, 1001: 5},
             {1000: 9, 1001 + w: 5},
             hsum((2000, 8), (2000 + w, 2), (2001 + w, 7)) if w else {2000: 8, 2002: 7},
             {5000: 4, 5003: 3}]
    ids = plant(sc, hists)

    def check(r):
        rows = r[0]
        if w:
            assert modes(rows, ids[0]) == [1000] and counts(rows, ids[0]) == [14]
            assert counts(rows, ids[2]) == [10, 9]
        assert modes(rows, ids[1]) == ([1000, 1001 + w] if w else [1000]) and counts(rows, ids[0])[0] == 9 + (w > 0) * 5
        if w >= 3:
            assert counts(rows, ids[3]) == [7]
    return Case("window_%d" % w, sc, [sc.query()], w, 1, check=check)


def maxalign(ma):
    """Candidates with 1, maxalign + 1 and maxalign + 2 qualifying modes."""
    sc = scene()
    hists = [{100: 5}, {100: 5, 200: 4}, {100: 5, 200: 4, 300: 3}][:ma + 3]
    hists = hists[ma:] if ma == 0 else hists
    ids = plant(sc, hists)

    def check(r):
        nmodes = [len(h) for h in hists]
        assert ma + 1 in nmodes and ma + 2 in nmodes
        assert [len(modes(r[0], i)) for i in ids] == [min(n, ma + 1) for n in nmodes]
    return Case("maxalign_%d" % ma, sc, [sc.query()], 1, 1, maxalign=ma, check=check)


def extremes(mtb):
    """With the batch's largest query time Q: entries at time 0 probed at Q (dtime -Q, the lowest
    bin bias - Q = window + 2) and entries at 2^mtb - 1 probed at time 0 (the highest bin: its
    right neighbour and the count window reach the end of the histogram).  mtb 20: two ids whose
    modes lie about 10^6 bins apart, one of them an equal maximum."""
    Q = 9000 if mtb == 14 else 5000
    top = (1 << mtb) - 1
    sc = scene(hashbits=10, mtb=mtb, nids=1024) if mtb == 20 else scene()
    if mtb == 14:
        ids = plant(sc, [{-Q: 3, 1 - Q: 1}, {top: 3, top - 1: 2}], how="mult")
        want = [[-Q], [top]]
    else:
        ids = plant(sc, [{-Q: 3, top: 3}, {top: 4, 17: 2}], how="mult")
        want = [[-Q, top], [top, 17]]

    def check(r):
        assert [modes(r[0], i) for i in ids] == want and int(r.q[0][:, 0].max()) == Q
    return Case("extremes_mtb%d" % mtb, sc, [sc.query()], 2, 1, maxalign=3, check=check)


def batch_bias():
    """Three queries in one call: the first one's largest query time (above 12000) sets the bias for the
    others, whose dtimes lie at the ends of their own ranges."""
    sc = scene()
    qs = []
    for k, h in enumerate([{-12000: 3, 500: 2}, {16383: 3, 16380: 2}, {0: 4, 2: 4}]):
        sc.rows = []
        plant(sc, [h], first=10 + k)
        qs.append(sc.query())

    def check(r):
        assert [modes(r[i], 10 + i) for i in range(3)] == [[-12000, 500], [16383, 16380], [0, 2]]
    return Case("batch_bias", sc, qs, 1, 1, check=check)


def long_mixed():
    """A long query whose query times run past 2^mtb (above 20000), with two short queries of small
    query times in the same call: the long path's bias comes from the long queries alone."""
    sc = scene()
    qs = []
    for k, h in enumerate([{-20000: 3, -3617: 2, 100: 5}, {16383: 3, 7: 2}, {-4: 3, 0: 3}]):
        sc.rows = []
        plant(sc, [h], how="mult" if k else "mix", first=20 + k)
        qs.append(sc.query())

    def check(r):
        assert int(r.q[0][:, 0].max()) > (1 << sc.mtb) and int(r.q[1][:, 0].max()) < 100
        assert modes(r[0], 20) == [100, -20000, -3617]
    return Case("long_mixed", sc, qs, 1, 1, paths=("mixed",), long_only={0}, check=check)


def hi_bin_reuse():
    """Candidates in rank order whose count window (rank 1) and left neighbour (rank 2) cover the
    previous candidate's highest bin: the histogram must be left zeroed between candidates."""
    sc = scene()
    ids = plant(sc, [{100: 5, 105: 3}, {104: 6}, {106: 2}])

    def check(r):
        assert counts(r[0], ids[1]) == [6] and modes(r[0], ids[2]) == [106]
    return Case("hi_bin_reuse", sc, [sc.query()], 1, 1, check=check)


def many_queries():
    """300 queries (more than 2 x the H100's 132 SMs): every CTA of the fast and general kernels
    runs several, each one's candidates covering bins the previous ones touched."""
    sc = scene()
    qs = []
    for k in range(300):
        sc.rows = []
        s = k % 7
        plant(sc, [{100 + s: 3, 103 + s: 2}, {102 + s: 4, 104 + s: 1}], how=("mult", "probe")[k % 2], first=1 + 2 * k)
        qs.append(sc.query())

    def check(r):
        assert len(r.q) == 300 and all(len(x) == 3 for x in r.rows)
    return Case("many_queries", sc, qs, 1, 1, paths=("fast", "general"), check=check)


def many_candidates():
    """One query with 300 row-capable candidates: more than the long path's mode CTAs (at most one
    per SM), so its grid-stride loop gives each CTA several, all with the same bins."""
    sc = scene()
    ids = np.arange(1, 301)
    for s in range(0, 300, 60):
        sc.group(ids[s:s + 60], 3, 0, 200)
        sc.group(ids[s:s + 60], 2, 0, 202)
    sc.hpi[ids] = 5 * (1000 + ids)

    def check(r):
        assert len(r.cand[0][0]) == 300 and len(r.rows[0]) == 600
        assert np.array_equal(r.rows[0][:, 2], np.tile([200, 202], 300))
    return Case("many_candidates", sc, [sc.query()], 1, 1, sdepth=300, check=check)


def two_long():
    """Two queries of one call on the long path (and on the others), one after the other on the
    same histograms."""
    sc = scene()
    qs = []
    for k, h in enumerate([{300: 4, 302: 3}, {301: 5, 303: 2}]):
        sc.rows = []
        plant(sc, [h], first=40 + k)
        qs.append(sc.query())

    def check(r):
        assert counts(r[0], 40) == [4, 3] and counts(r[1], 41) == [5, 2]
    return Case("two_long", sc, qs, 1, 1, check=check)


def consecutive():
    """Two calls with the same scratch layout (same rows, largest query time and table): the second
    one's candidate reads the bins the first one's touched last."""
    sc = scene()
    qs = []
    for k, h in enumerate([{100: 5, 105: 3}, {104: 6, 106: 2}]):
        sc.rows = []
        plant(sc, [h], how="mult", first=50 + k)
        qs.append(sc.query())
    n = max(len(q) for q in qs)
    qs = [np.concatenate([q, np.zeros((n - len(q), 2), np.int32)]) for q in qs]    # bucket 0 is empty

    def check(r):
        assert len(r.q[0]) == len(r.q[1]) and r.q[0][:, 0].max() == r.q[1][:, 0].max()
        assert counts(r[1], 51) == [6, 2]
    return Case("consecutive_calls", sc, qs, 1, 1, check=check, calls=2)


def row_capacity(n):
    """One candidate with n isolated modes, max_alignments_per_id 300: 256 rows fit the default
    row capacity, 257 take the retry - on the long path through slot_cap = row capacity < 301."""
    sc = scene()
    ids = plant(sc, [{3 * i: 2 for i in range(n)}], how="mult")

    def check(r):
        assert len(r[0]) == n and modes(r[0], ids[0]) == [3 * i for i in range(n)]
    return Case("rows_%d" % n, sc, [sc.query()], 0, 1, maxalign=300, check=check)


def quick_filter_long():
    """Candidates of 2048 hits (the long path's quick filter, QF_LONG) and of 2049 (none): in each,
    a top bin equal to threshcount 5 (no row) and one of 6 (one row)."""
    sc = scene()
    hists = []
    for raw in (2048, 2049):
        for top in (5, 6):
            n5, rest = divmod(raw - top, 5)
            h = {2 * i: 5 for i in range(n5)}
            h[2 * n5] = rest or 0
            h[2 * n5 + 4] = top
            hists.append({d: c for d, c in h.items() if c})
    ids = plant(sc, hists, how="mult")

    def check(r):
        cand, raw = r.cand[0]
        assert list(cand) == ids and list(raw) == [2048, 2048, 2049, 2049]
        assert [len(modes(r[0], i)) for i in ids] == [0, 1, 0, 1]
    return Case("quick_filter_long", sc, [sc.query()], 1, 5, check=check)


def many_hits_one_bin():
    """70,000 hits at one dtime (one bucket holding the id 50 times, probed 1400 times) plus a tail."""
    sc = scene()
    sc.group([1] * 50, 1400, 0, 500)
    place(sc, 1, {501: 3, 510: 7, 600: 2})
    sc.hpi[1] = 7

    def check(r):
        assert modes(r[0], 1) == [500, 510] and counts(r[0], 1) == [70003, 7]
    return Case("many_hits_one_bin", sc, [sc.query()], 1, 5, paths=NOFAST, check=check)


def all_cases():
    return ([local_max(), argmax_ties()] + [threshold(t) for t in (5, 1, 0)] + [window(w) for w in WINDOWS] +
            [maxalign(0), maxalign(1), extremes(14), extremes(20), batch_bias(), long_mixed(), hi_bin_reuse(),
             many_queries(), many_candidates(), two_long(), consecutive(), row_capacity(256), row_capacity(257),
             quick_filter_long(), many_hits_one_bin()])


class RefView:
    """What a family's check reads: rows[i] (k4_reference, rank order), cand[i] = (ids, raw), q[i]."""

    def __init__(self, case):
        self.q = case.queries
        self.rows = [case.rows(i) for i in range(len(case.queries))]
        self.cand = [case.candidates(i) for i in range(len(case.queries))]

    def __getitem__(self, i):
        return self.rows[i]


def reached(case):
    """Run the family's reference-side check; returns the RefView."""
    r = RefView(case)
    case.check(r)
    return r
