"""K4's long-query path (afp_match_long.cu): queries of rows * depth >= 2^24 - whole shows,
broadcast days - matched over the whole grid with memory sized by their actual hits.

The oracle's get_hits loops over query rows in Python; for queries of 10^5 rows and more the
same semantics are stated here in NumPy (_np_rows), checked first against the oracle on small
queries.  The general kernel is the other side of the A/B comparisons (force_general_kernel)."""
import os

import numpy as np
import pytest

from audfprint_b200 import HashTable, Matcher
from oracle import afp_oracle as orc
from tests import cases
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu

LONG_HITS = 1 << 24
LONG_STATUS = 6


# ---- NumPy statement of get_hits -> rank_candidates -> offset_histogram_rows -------------------
def _np_hits(table, counts, hashbits, depth, mtb, q):
    """(ids, dtimes) of every hit in (query row, slot) order, as orc.get_hits."""
    q = np.asarray(q, np.int64).reshape(-1, 2)
    b = q[:, 1] & ((1 << hashbits) - 1)
    n = np.minimum(depth, counts[b]).astype(np.int64)
    rep = np.repeat(np.arange(len(q)), n)
    slot = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    v = table[b[rep], slot].astype(np.int64)
    return (v >> mtb) - 1, (v & ((1 << mtb) - 1)) - q[rep, 0]


def _np_rows(table, counts, hashbits, depth, mtb, hpi, q, window, thresh, sdepth, maxalign=100):
    """Rows [id, count, dtime, raw, rank, 0, 0] in rank order (not sorted by count)."""
    ids, dts = _np_hits(table, counts, hashbits, depth, mtb, q)
    if len(ids) == 0:
        return np.zeros((0, 7), np.int32)
    uid, raw = np.unique(ids, return_counts=True)
    order = np.argsort(raw / hpi[uid].astype(float), kind="stable")[::-1]
    order = order[:min(int(np.count_nonzero(raw > thresh)), sdepth)]
    by_id = np.argsort(ids, kind="stable")
    sid, sdt = ids[by_id], dts[by_id]
    rows = []
    for rank, k in enumerate(order):
        id_, r = int(uid[k]), int(raw[k])
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
            rows.append([id_, int(bc[a:b].sum()), mode + tmin, r, rank, 0, 0])
            lm[a:b] = 0
            found += 1
            if found > maxalign:
                break
    return np.array(rows, np.int32).reshape(-1, 7)


def _by_count(rows):
    return rows[np.argsort(-rows[:, 1], kind="stable")]


def _table(hashbits, depth, mtb, tracks):
    """HashTable whose track i holds the (time, hash) rows tracks[i], appended in order."""
    nb = 1 << hashbits
    table = np.zeros((nb, depth), np.uint32)
    counts = np.zeros(nb, np.int32)
    hpi = np.zeros(len(tracks), np.uint32)
    for i, th in enumerate(tracks):
        th = np.asarray(th, np.int64).reshape(-1, 2)
        b = th[:, 1] & (nb - 1)
        order = np.argsort(b, kind="stable")
        b, t = b[order], th[order, 0]
        first = np.searchsorted(b, b)                     # rank within the same bucket
        slot = counts[b] + (np.arange(len(b)) - first)
        assert np.all(slot < depth)
        table[b, slot] = (((i + 1) << mtb) | (t & ((1 << mtb) - 1))).astype(np.uint32)
        np.add.at(counts, b, 1)
        hpi[i] = len(th)
    ht = HashTable(hashbits=hashbits, depth=depth, maxtime=1 << mtb)
    ht.table, ht.counts, ht.hashesperid = table, counts, hpi
    ht.names = ["t%d" % i for i in range(len(tracks))]
    return ht


def _rows_of(m, ht, q, force=False):
    m.force_general_kernel = force
    try:
        return m.match_batch(ht, [q], sort=False)[0]
    finally:
        m.force_general_kernel = False


def _matcher(window, thresh, sdepth, maxalign=100):
    m = Matcher()
    m.window, m.threshcount, m.search_depth, m.max_alignments_per_id = window, thresh, sdepth, maxalign
    return m


# ---- fixtures --------------------------------------------------------------------------------
DEPTH = 1024        # shows of 16,384+ rows are long at this depth
HB, MTB = 16, 15


@pytest.fixture(scope="module")
def shows():
    """A depth-1024 table of the long.npz tracks (one stored twice: equal hashesperid, tied
    weights), 1,500 filler tracks of 40 random hashes, and 'shows' made of the tracks at time
    offsets (repeats: several alignments per id, negative dtimes) with noise rows."""
    g = np.load(os.path.join(GOLDEN, "long.npz"))
    rng = np.random.default_rng(2024)
    real = [g["t%d/wf2h_s1" % s].astype(np.int64) for s in cases.LONG_SEEDS]
    tracks = real + [real[0]]
    for _ in range(1500):
        tracks.append(np.stack([rng.integers(0, 8000, 40), rng.integers(0, 1 << 20, 40)], 1))
    ht = _table(HB, DEPTH, MTB, tracks)

    def show(parts, noise, seed):
        r = np.random.default_rng(seed)
        rows, t0 = [], 0
        for k, frac in parts:
            tr = real[k][:max(1, int(len(real[k]) * frac))].copy()
            tr[:, 0] += t0
            rows.append(tr)
            t0 = int(tr[-1, 0]) + 50
        nz = np.stack([r.integers(0, t0, noise), r.integers(0, 1 << 20, noise)], 1)
        q = np.concatenate(rows + [nz])
        return q[np.lexsort((q[:, 1], q[:, 0]))].astype(np.int32)

    a = show([(0, 1.0), (1, 0.5), (0, 1.0), (2, 1.0), (0, 0.4)], 1500, 1)
    b = show([(1, 1.0), (2, 0.6), (1, 1.0), (0, 1.0)], 600, 2)
    return ht, [a, b]


def test_numpy_statement_equals_the_oracle():
    """_np_rows (vectorised) == orc.match_hashes (row loop) on small random queries."""
    rng = np.random.default_rng(3)
    hashbits, depth, mtb, nids = 10, 16, 10, 200
    nb = 1 << hashbits
    table = ((rng.integers(1, nids + 1, (nb, depth), dtype=np.int64) << mtb)
             + rng.integers(0, 700, (nb, depth))).astype(np.uint32)
    counts = rng.integers(0, depth + 4, nb).astype(np.int32)
    hpi = np.full(nids, 37, np.uint32)
    hpi[::3] = 20
    for seed, nq, window, thresh, sdepth, maxalign in ((0, 300, 1, 2, 50, 100), (1, 900, 2, 1, 5, 1),
                                                       (2, 60, 1, 0, 100, 2), (3, 0, 1, 1, 10, 100)):
        r = np.random.default_rng(seed)
        q = np.stack([r.integers(0, 500, nq), r.integers(0, 1 << 20, nq)], 1).astype(np.int32)
        want = orc.match_hashes(table, counts, hashbits, depth, mtb, hpi, q, window=window, threshcount=thresh,
                                search_depth=sdepth, max_alignments_per_id=maxalign)
        got = _np_rows(table, counts, hashbits, depth, mtb, hpi, q, window, thresh, sdepth, maxalign)
        assert np.array_equal(_by_count(got), want), seed


def test_query_beyond_the_former_limit():
    """rows * depth >= 2^30 (formerly AFP_ERR_UNSUPPORTED): 262,144 rows against a sparse
    2^12 x 4096 table with aligned entries planted for five ids; rows equal the NumPy statement."""
    rng = np.random.default_rng(11)
    hashbits, depth, mtb, nids = 12, 4096, 16, 400
    nb = 1 << hashbits
    nq = 1 << 18
    q = np.stack([np.sort(rng.integers(0, 40000, nq)), rng.integers(0, 1 << 20, nq)], 1).astype(np.int32)
    counts = rng.integers(0, 24, nb).astype(np.int32)
    table = np.zeros((nb, depth), np.uint32)
    valid = np.arange(depth)[None, :] < counts[:, None]
    table[valid] = ((rng.integers(5, nids, int(valid.sum())) + 1) << mtb) + rng.integers(0, 1 << mtb, int(valid.sum()))
    for k, off in enumerate((-1500, -3, 0, 700, 1900)):
        sel = rng.choice(np.nonzero(q[:, 0] >= 2000)[0], 150 + 40 * k, replace=False)
        for t, h in q[sel]:
            b = int(h) & (nb - 1)
            table[b, counts[b]] = ((k + 1) << mtb) + int(t) + off
            counts[b] += 1
    valid = np.arange(depth)[None, :] < counts[:, None]
    hpi = np.maximum(np.bincount((table[valid] >> mtb).astype(np.int64) - 1, minlength=nids), 1).astype(np.uint32)
    hpi[:5] = 10                          # the planted ids outrank the random ones
    ht = HashTable(hashbits=hashbits, depth=depth, maxtime=1 << mtb)
    ht.table, ht.counts, ht.hashesperid = table, counts, hpi
    assert nq * depth >= 1 << 30
    m = _matcher(2, 5, 100)
    got = m.match_batch(ht, [q], sort=False)[0]
    assert Matcher.last_status(ht, 1)[0, 0] == LONG_STATUS
    want = _np_rows(table, counts, hashbits, depth, mtb, hpi, q, 2, 5, 100)
    assert np.array_equal(got, want)
    for k, off in enumerate((-1500, -3, 0, 700, 1900)):
        assert np.any((got[:, 0] == k) & (got[:, 2] == off)), k
    srt = m.match_hashes(ht, q)
    assert sorted(map(tuple, srt)) == sorted(map(tuple, want)) and np.array_equal(srt[:, 1], _by_count(want)[:, 1])


@pytest.mark.parametrize("window", [1, 2])
def test_long_path_equals_general_kernel(shows, window):
    """Every row, rank column included, and in the same order, on both paths."""
    ht, qs = shows
    for q in qs:
        assert LONG_HITS <= len(q) * DEPTH < 2 * LONG_HITS
    seen_multi = seen_neg = seen_cap = seen_tie = False
    for thresh in (0, 1, 5):
        for sdepth in (1, 100, 1500):
            for maxalign in ((100, 1) if sdepth == 100 else (100,)):
                m = _matcher(window, thresh, sdepth, maxalign)
                for q in qs:
                    got = _rows_of(m, ht, q)
                    assert Matcher.last_status(ht, 1)[0, 0] == LONG_STATUS
                    want = _rows_of(m, ht, q, force=True)
                    assert Matcher.last_general_count(ht) == 1
                    assert np.array_equal(got, want), (window, thresh, sdepth, maxalign)
                    ids, n = np.unique(got[:, 0], return_counts=True)
                    seen_multi |= bool(np.any(n[ids < 3] > 1))
                    seen_neg |= bool(np.any(got[:, 2] < 0))
                    seen_cap |= bool(np.any(n == maxalign + 1))
                    seen_tie |= {0, 3} <= set(got[:, 0].tolist())
    assert seen_multi and seen_neg and seen_cap and seen_tie


def test_publish_lists_and_options(shows):
    """Publish mode: candidate lists equal on both paths; exact_count / find_time_range rows on a
    long show from the batch finish equal the per-query host form."""
    ht, qs = shows
    q = qs[0]
    qoff = np.array([0, len(q)], np.int64)
    for thresh, sdepth in ((5, 100), (0, 1500), (1, 3)):
        m = _matcher(2, thresh, sdepth)
        rows_l, roff_l, cand_l, cnt_l = m._publish_call(ht, q, qoff)
        assert Matcher.last_status(ht, 1)[0, 0] == LONG_STATUS
        m.force_general_kernel = True
        rows_g, roff_g, cand_g, cnt_g = m._publish_call(ht, q, qoff)
        m.force_general_kernel = False
        assert np.array_equal(cnt_l, cnt_g)
        k = int(cnt_l[0, 0])
        assert k == min(sdepth, len(np.unique(_np_hits(ht.table, ht.counts, HB, DEPTH, MTB, q)[0])))
        assert np.array_equal(cand_l[0, :k], cand_g[0, :k])
        assert np.array_equal(rows_l, rows_g)
    short = qs[1][:3000]
    for opt in ("exact_count", "find_time_range"):
        m = _matcher(2, 5, 100)
        setattr(m, opt, True)
        single = m.match_hashes(ht, q)
        batch = m.match_batch(ht, [q, short])
        assert sorted(map(tuple, batch[0])) == sorted(map(tuple, single)), opt
        assert np.array_equal(batch[0][:, 1], single[:, 1])
        assert len(single) > 0 and single[0, 0] < 4           # one of the tracks the show is made of
        assert sorted(map(tuple, batch[1])) == sorted(map(tuple, m.match_hashes(ht, short)))


def test_mixed_batch(shows):
    """Short (incl. empty and 1-row) and long queries in one batch: the short ones' rows equal a
    batch without the long ones; status 6 exactly for the long ones; the general-kernel count
    excludes them; a long query with no hits and one with nabove == 0 return no rows."""
    ht, qs = shows
    rng = np.random.default_rng(5)
    empty_b = np.nonzero(ht.counts == 0)[0]
    # zero hits: every row probes an empty bucket
    nohit = np.stack([np.arange(LONG_HITS // DEPTH), np.full(LONG_HITS // DEPTH, empty_b[0])], 1).astype(np.int32)
    # nabove == 0 at threshcount 5: each bucket probed once, buckets holding only filler entries
    # with no id more than 5 times in total
    ids, _ = _np_hits(ht.table, ht.counts, HB, DEPTH, MTB, np.stack([np.zeros(1 << HB), np.arange(1 << HB)], 1))
    per_b = np.minimum(DEPTH, ht.counts).astype(np.int64)
    start = np.cumsum(per_b) - per_b
    owner = np.repeat(np.arange(1 << HB), per_b)
    filler_only = np.ones(1 << HB, bool)
    np.logical_and.at(filler_only, owner, ids >= 4)
    cand_b = rng.permutation(np.nonzero(filler_only & (ht.counts > 0))[0])
    picked, seen = [], {}
    for b in cand_b:
        bid = ids[start[b]:start[b] + per_b[b]]
        if all(seen.get(int(i), 0) + 1 <= 5 for i in bid):
            for i in bid:
                seen[int(i)] = seen.get(int(i), 0) + 1
            picked.append(b)
    picked = np.array(picked)
    nrow = LONG_HITS // DEPTH
    lowq = np.stack([np.arange(nrow), np.concatenate([picked, empty_b[1:]])[:nrow]], 1).astype(np.int32)
    assert len(picked) > 100
    short = [qs[1][:2000], np.zeros((0, 2), np.int32), qs[0][100:700], qs[0][:1]]
    batch = [short[0], qs[0], short[1], short[2], nohit, short[3], qs[1], lowq]
    long_ix = [1, 4, 6, 7]
    m = _matcher(2, 5, 100)
    got = m.match_batch(ht, batch, sort=False)
    st = Matcher.last_status(ht, len(batch))
    ngen = Matcher.last_general_count(ht)
    assert [i for i in range(len(batch)) if st[i, 0] == LONG_STATUS] == long_ix
    ref = m.match_batch(ht, short, sort=False)
    assert Matcher.last_general_count(ht) == ngen
    for i, j in zip((0, 2, 3, 5), range(4)):
        assert np.array_equal(got[i], ref[j]), i
    assert len(got[2]) == 0 and len(got[5]) == 0
    assert len(got[4]) == 0 and len(got[7]) == 0
    for i in (1, 6):
        assert np.array_equal(got[i], _rows_of(m, ht, batch[i], force=True))
    # the general kernel on its own: the long ones still go to the long path
    m.threshcount = 0                         # (the fast kernel does not run at threshcount 0)
    got0 = m.match_batch(ht, batch, sort=False)
    st0 = Matcher.last_status(ht, len(batch))
    assert [i for i in range(len(batch)) if st0[i, 0] == LONG_STATUS] == long_ix
    assert np.all(st0[[0, 2, 3, 5], 0] == -1)
    assert Matcher.last_general_count(ht) == 4
    assert np.array_equal(got0[1], _rows_of(m, ht, batch[1], force=True))


def test_row_capacity_retry(shows):
    """A long query with more than 256 rows goes through the RowCapacityError retry."""
    ht, qs = shows
    m = _matcher(1, 0, 1500)
    got = _rows_of(m, ht, qs[0])
    assert len(got) > 256
    assert Matcher.last_status(ht, 1)[0, 0] == LONG_STATUS
    assert np.array_equal(got, _rows_of(m, ht, qs[0], force=True))
    want = _np_rows(ht.table, ht.counts, HB, DEPTH, MTB, ht.hashesperid, qs[0], 1, 0, 1500)
    assert np.array_equal(got, want)
