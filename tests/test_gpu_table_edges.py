"""The device hash table (csrc/afp_store.cu, csrc/afp_table_edit.cu, the probe / restriction /
pruning-bound code of csrc/afp_match.cu) against the sequential statement of tests/table_reference.py,
bit for bit, on constructed (time, hash) rows at the edges of the kernels' branches and constants:
the one-thread / one-CTA / global-memory ranking of a bucket's batch entries (16 / 8192), the
1024-entry overflow compaction blocks and more than 1024 of them, the carry of the partial-sum scan
(more than 2^20 buckets, in store and retrieve), the last-writer-wins slot scratch across table geometries, id and time masking up to the
entry 0xFFFFFFFF, the 32-slot ballot chunks and the id bitmap of remove / retrieve, the radix-sort
width of retrieve and its repeated-id gather, the hit probe's hash mask, the id-range restriction
and the pruning bound."""
import ctypes as C
import random

import numpy as np
import pytest

from audfprint_b200 import _lib
from tests import table_reference as ref

pytestmark = pytest.mark.gpu


def val(id_, t, mtb):
    return ((id_ + 1) << mtb) + t


def assert_same(ht, st):
    assert np.array_equal(ht.counts, st.counts)
    assert np.array_equal(ht.table, st.table)
    assert np.array_equal(ht.hashesperid, st.hashesperid)
    assert ht.names == st.names


def device_arrays(ctx, hashbits, depth):
    table = np.empty((1 << hashbits, depth), np.uint32)
    counts = np.empty(1 << hashbits, np.int32)
    ctx.check(ctx.lib.afp_table_download(ctx.h, table.ctypes.data, counts.ctypes.data))
    return table, counts


def device_bound(ctx):
    out = C.c_uint32(0)
    ctx.check(ctx.lib.afp_table_pruning_bound(ctx.h, C.byref(out)))
    return int(out.value)


def patch_form_store(st0, ids, rows):
    """The batch through the patch form of the ABI: afp_table_store_batch, then
    afp_table_fetch_overflow (bucket, count, value), random.randint(0, count) drawn here, one patch
    per slot (the last writer wins) through afp_table_apply_patches.  Returns (table, counts)."""
    ctx = _lib.context(None)
    ctx.table_key = None                                   # the context's table is ours now
    hpi = np.ascontiguousarray(st0.hashesperid, np.uint32)
    table, counts = np.ascontiguousarray(st0.table), np.ascontiguousarray(st0.counts)
    ctx.check(ctx.lib.afp_table_upload(ctx.h, table.ctypes.data, counts.ctypes.data, st0.hashbits, st0.depth,
                                       st0.maxtimebits, hpi.ctypes.data if len(hpi) else None, len(hpi), 1))
    roff = np.zeros(len(rows) + 1, np.int64)
    roff[1:] = np.cumsum([len(r) for r in rows])
    flat = np.ascontiguousarray(np.concatenate([np.asarray(r, np.int32).reshape(-1, 2) for r in rows]))
    ids = np.asarray(ids, np.int64)
    nov = C.c_int64(0)
    ctx.check(ctx.lib.afp_table_store_batch(ctx.h, flat.ctypes.data if len(flat) else None, 1,
                                            roff.ctypes.data_as(C.POINTER(C.c_int64)), len(rows),
                                            ids.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(nov)))
    n = int(nov.value)
    bucket, cnt, value = np.empty(n, np.uint32), np.empty(n, np.int32), np.empty(n, np.uint32)
    ctx.check(ctx.lib.afp_table_fetch_overflow(ctx.h, bucket.ctypes.data, cnt.ctypes.data, value.ctypes.data))
    last = {}
    for b, c, v in zip(bucket.tolist(), cnt.tolist(), value.tolist()):
        s = random.randint(0, c)
        if s < st0.depth:
            last[(b, s)] = v
    pb = np.array([k[0] for k in last], np.uint32)
    ps = np.array([k[1] for k in last], np.int32)
    pv = np.array(list(last.values()), np.uint32)
    ctx.check(ctx.lib.afp_table_apply_patches(ctx.h, pb.ctypes.data, ps.ctypes.data, pv.ctypes.data, len(pb)))
    out = device_arrays(ctx, st0.hashbits, st0.depth)
    ctx.table_key = None
    return out


def check_store(st0, batch, seed, forms=("hashes", "patch")):
    """One store_batch of `batch` [(name or id, rows)] on a table holding `st0`, in both forms of
    the ABI, against the statement's store loop from the same `random` state: table, counts,
    hashesperid, names and the next random.random() bit for bit.  Returns the statement's state."""
    names = [n for n, _ in batch]
    rows = [np.asarray(r, np.int32).reshape(-1, 2) for _, r in batch]
    want = st0.copy()
    random.seed(seed)
    ids = []
    for name, r in zip(names, rows):
        ids.append(ref.name_to_id(want, name))
        ref.store(want, ids[-1], r)
    want_next = random.random()
    if "hashes" in forms:
        ht = ref.mirror(st0)
        random.seed(seed)
        assert ht.store_batch(names, rows) == [len(r) for r in rows]
        assert random.random() == want_next, "the RNG replay must leave `random` where the statement does"
        assert ht._dev_newer and not ht._store_pending
        assert_same(ht, want)
    if "patch" in forms:
        random.seed(seed)
        table, counts = patch_form_store(st0, ids, rows)
        assert random.random() == want_next
        assert np.array_equal(counts, want.counts) and np.array_equal(table, want.table)
    return want


def filled(hashbits, depth, mtb, nids, seed, counts):
    """A table whose bucket b holds min(counts[b], depth) entries of random ids < nids (slots past
    the count are 0), hashesperid = the entries of every id + 1."""
    rng = np.random.default_rng(seed)
    counts = np.asarray(counts, np.int32)
    n = np.minimum(counts, depth)
    valid = np.arange(depth)[None, :] < n[:, None]
    ids = rng.integers(0, nids, valid.shape)
    table = np.where(valid, ((ids + 1) << mtb) + rng.integers(0, 1 << mtb, valid.shape), 0).astype(np.uint32)
    hpi = np.bincount(ids[valid], minlength=nids).astype(np.uint32) + 1
    return ref.State(hashbits, depth, mtb, table, counts, ["t%d" % i for i in range(nids)], hpi)


# ---- store ------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 15, 16, 17, 8192, 8193])
@pytest.mark.parametrize("before", ["empty", "depth-1", "depth", "far above"])
def test_one_bucket_across_the_ranking_paths(n, before):
    """n entries of one batch in one bucket: ranked by one thread (n <= 16), by one CTA from
    shared memory (17..8192) and from global memory (8193), with the bucket's count before the
    batch at 0, depth - 1, depth and far above depth, so that the run crosses `depth` inside each
    path.  The hashes differ above hashbits and some are negative; the times are unsorted."""
    hb, depth, mtb, b = 4, 10, 12, 9
    c0 = {"empty": 0, "depth-1": depth - 1, "depth": depth, "far above": 5 * depth + 3}[before]
    st = filled(hb, depth, mtb, 3, 1, [2, 0, 10, 4, 0, 0, 7, 1, 0, c0, 3, 0, 0, 12, 0, 1])
    rng = np.random.default_rng(n)
    hot = np.stack([rng.integers(-5000, 5000, n), b + 16 * rng.integers(-40000, 40000, n)], axis=1)
    other = rng.integers(0, 16, 60)
    other = np.stack([rng.integers(0, 4096, 60), np.where(other == b, 0, other)], axis=1)
    check_store(st, [("x", hot), ("t1", other[:30]), (0, other[30:])], seed=n + c0)


def test_one_bucket_spread_over_many_files():
    """A bucket's entries arrive from 40 files of one batch: the same name twice, an integer id
    naming an existing track, empty files in between, rows sorted neither by time nor by hash;
    one bucket takes 9,000 of them (global-memory CTA ranking across files)."""
    hb, depth, mtb = 6, 8, 12
    st = filled(hb, depth, mtb, 2, 2, np.arange(64) % 11)
    rng = np.random.default_rng(4)
    batch = []
    for f in range(40):
        name = ["a", "b", 1, "a", "c"][f % 5]
        if f % 7 == 3:
            batch.append((name, np.zeros((0, 2), np.int32)))
            continue
        n = 300 + int(rng.integers(0, 200))
        h = np.where(rng.random(n) < 0.75, 5, rng.integers(-1000, 1000, n))
        batch.append((name, np.stack([rng.integers(0, 6000, n), h], axis=1)))
    assert sum(int((r[:, 1] % 64 == 5).sum()) for _, r in batch) > 8192
    want = check_store(st, batch, seed=9)
    assert want.names == ["t0", "t1", "a", "b", "c"]


@pytest.mark.parametrize("depth", [1, 2])
def test_overflow_slots_with_many_writers(depth):
    """Depth 1 and 2: almost every entry overflows and many entries of one batch draw the same
    slot; the sequential loop lets the last one win.  The seed is chosen so that the batch's last
    entry is a winner, and winners come from different files."""
    hb, mtb = 3, 10
    st = filled(hb, depth, mtb, 1, 3, [0, 1, 2, 5, 0, 3, depth, 9])
    rng = np.random.default_rng(depth)
    batch = [("f%d" % f, np.stack([rng.integers(0, 1000, 200), rng.integers(0, 6, 200)], axis=1)) for f in range(5)]
    batch.append(("z", np.array([[1023, 6]])))                   # the last entry: bucket 6, full before it
    lastval = val(6, 1023, mtb)
    for seed in range(100):
        want = st.copy()
        random.seed(seed)
        for name, r in batch:
            ref.store(want, ref.name_to_id(want, name), r)
        winners = {int(v) >> mtb for v in want.table[want.counts > depth].ravel()} - {0, 1}
        if lastval in want.table[6] and len(winners) >= 3:
            break
    else:
        raise AssertionError("no seed lets the last entry win")
    check_store(st, batch, seed=seed)


@pytest.mark.parametrize("m", [1023, 1024, 1025])
def test_overflow_compaction_block_edges(m):
    """Batches of 1023, 1024 and 1025 entries in which the overflowing entries sit at both ends
    of the 1024-entry compaction blocks and of their warps (0, 1, 31, 32, 1022, 1023, 1024, last),
    mixed with entries that find room."""
    hb, depth, mtb = 10, 3, 12
    st = filled(hb, depth, mtb, 2, 5, np.where(np.arange(1024) < 100, depth, 0))
    rng = np.random.default_rng(m)
    full = np.zeros(m, bool)
    full[[i for i in (0, 1, 31, 32, 1022, 1023, 1024, m - 1) if i < m]] = True
    full |= rng.random(m) < 0.1
    h = np.where(full, rng.integers(0, 100, m), rng.integers(100, 1024, m))
    rows = np.stack([rng.integers(0, 4096, m), h], axis=1)
    check_store(st, [("x", rows[:m // 3]), ("y", rows[m // 3:m // 3]), ("x", rows[m // 3:])], seed=m)


def test_more_than_2_20_entries_in_one_batch():
    """1.2 M entries in one batch on a 2^16 x 8 table (most overflow, all through the batch): the
    overflow compaction scans 1,172 per-block counts, more than one scan block of 1024.  (The
    partial-sum carry of that scan needs more than 2^30 entries; the bucket scans of 2^21 and 2^22
    buckets below reach it.)"""
    rng = np.random.default_rng(6)
    m = 1_200_000
    rows = np.stack([rng.integers(-(1 << 31), 1 << 31, m), rng.integers(-(1 << 31), 1 << 31, m)], axis=1)
    st = ref.State(16, 8, 14, names=["a"], hashesperid=[0])
    check_store(st, [("a", rows[:500_000]), ("b", rows[500_000:])], seed=12)


@pytest.mark.parametrize("hb", [1, 21, 22])
def test_bucket_scan_carry_and_extreme_buckets(hb):
    """Tables of 2, 2^21 and 2^22 buckets: for the larger two the bucket histogram's scan
    carries across 1024 x 1024 buckets.  Entries land in bucket 0, the last bucket (overflowing
    both) and all over."""
    depth, mtb = 2 if hb > 1 else 3, 10
    nb = 1 << hb
    rng = np.random.default_rng(hb)
    st = ref.State(hb, depth, mtb, names=["p"], hashesperid=[5])
    st.table[[0, nb - 1], 0] = val(0, 7, mtb)
    st.counts[[0, nb - 1]] = 1
    n = 40_000
    h = rng.integers(-(1 << 31), 1 << 31, n)
    h[:12] = [0, nb - 1, nb, -1, 0, nb - 1, 2 * nb, nb - 1, 0, -nb, 3 * nb - 1, 0]
    h[-3:] = [nb - 1, 0, nb - 1]
    rows = np.stack([rng.integers(0, 1 << mtb, n), h], axis=1)
    check_store(st, [("a", rows[:n // 2]), ("p", rows[n // 2:])], seed=hb)


@pytest.mark.parametrize("mtb", [1, 24])
def test_masking_and_the_largest_id(mtb):
    """Hashes at and above 2^hashbits and negative, times at and above 2^maxtimebits and negative,
    1 and 24 time bits; with 24 bits the largest id that fits ((id + 2) << 24 == 2^32) stores the
    entry 0xFFFFFFFF.  One id past it - given as an existing name or as an integer id - raises with
    nothing changed, and the table takes a valid batch afterwards."""
    hb, depth = 5, 4
    nids = 1 << (32 - mtb) if mtb == 24 else 6
    st = ref.State(hb, depth, mtb, names=["n%d" % i for i in range(nids)])
    top = min(nids - 1, (1 << (32 - mtb)) - 2)
    rng = np.random.default_rng(mtb)
    n = 400
    t = rng.integers(-(1 << 31), 1 << 31, n)
    t[:6] = [(1 << mtb) - 1, 1 << mtb, -1, -(1 << mtb), (1 << mtb) + 1, 0]
    h = rng.integers(-(1 << 31), 1 << 31, n)
    h[:6] = [31, 32, -1, -32, 1 << 30, -(1 << 31)]
    rows = np.stack([t, h], axis=1)
    want = check_store(st, [("n%d" % top, rows[:6]), ("n0", rows[6:100]), (top, rows[100:300]), ("n1", rows[300:])],
                       seed=mtb)
    if mtb == 24:
        assert (want.table == 0xFFFFFFFF).any()
        ht = ref.mirror(want)
        state = random.getstate()
        for bad in (["n255"], [255], ["n0", "n255"]):             # id 255: (255 + 2) << 24 > 2^32
            with pytest.raises(ValueError):
                ht.store_batch(bad, [rows[:10]] * len(bad))
            assert random.getstate() == state
            assert not getattr(ht, "_store_pending", False) and not ht._dev_newer
            assert_same(ht, want)
        random.seed(4)
        assert ht.store_batch(["n1"], [rows[:50]]) == [50]
        nxt = random.random()
        random.seed(4)
        ref.store(want, 1, rows[:50])
        assert random.random() == nxt
        assert_same(ht, want)


def test_slot_scratch_across_table_geometries():
    """Overflowing stores on 2^12 x 8, then 2^10 x 100, then 2^14 x 2 tables on one device context:
    the table-sized last-writer scratch must be all-zero again after every call, whatever its
    size was."""
    rng = np.random.default_rng(8)
    for seed, (hb, depth, n, span) in enumerate([(12, 8, 60_000, 1 << 12), (10, 100, 150_000, 256),
                                                 (14, 2, 60_000, 1 << 14), (12, 8, 60_000, 1 << 12)]):
        st = ref.State(hb, depth, 12)
        rows = np.stack([rng.integers(0, 4096, n), rng.integers(0, span, n)], axis=1)
        want = check_store(st, [("a", rows[:n // 2]), ("b", rows[n // 2:])], seed=seed, forms=("hashes",))
        assert (want.counts > depth).any()


def test_integer_id_outside_the_names_changes_nothing():
    """store_batch with an integer id outside [0, len(names)) raises IndexError before any device
    work: table, counts, names, hashesperid and `random` unchanged, no half-finished batch left
    behind, and the table takes the next batch."""
    st = filled(6, 4, 12, 2, 11, np.arange(64) % 7)
    ht = ref.mirror(st)
    rows = np.stack([np.arange(50), np.arange(50) * 7], axis=1)
    state = random.getstate()
    for bad in (["c", 3], [2], [-1], ["a", 1, 4]):
        with pytest.raises(IndexError):
            ht.store_batch(bad, [rows] * len(bad))
        assert not getattr(ht, "_store_pending", False)
        assert random.getstate() == state
        assert_same(ht, st)
    batch = [("c", rows), (2, rows[:9]), (0, rows[10:])]          # id 2 is "c", new in this batch
    random.seed(6)
    assert ht.store_batch([n for n, _ in batch], [r for _, r in batch]) == [50, 9, 40]
    nxt = random.random()
    want = st.copy()
    random.seed(6)
    for name, r in batch:
        ref.store(want, ref.name_to_id(want, name), r)
    assert random.random() == nxt
    assert_same(ht, want)


# ---- remove / retrieve ------------------------------------------------------------------------

NIDS = 70


def edit_table(depth, seed=0):
    """2^9 buckets of `depth` slots, 70 ids (41..44 without entries); counts below, at and above
    depth; track 7 in the first slot, the last valid slot, slots 31/32 and 63/64, every slot (a
    bucket emptied), and the whole first chunk with survivors in the second."""
    hb, mtb = 9, 10
    rng = np.random.default_rng(depth * 10 + seed)
    nb = 1 << hb
    counts = rng.choice([0, 1, max(depth - 1, 1), depth, depth + 1, 3 * depth + 2, 1 + depth // 2], nb)
    counts[:8] = depth
    counts[8] = 5 * depth
    st = filled(hb, depth, mtb, NIDS, depth + seed, counts)
    ids = (st.table.astype(np.int64) >> mtb) - 1
    t = st.table & np.uint32((1 << mtb) - 1)
    remap = np.where((ids >= 41) & (ids <= 44) | (ids == 7), 45, ids)
    table = np.where(st.table != 0, ((remap + 1) << mtb) + t, 0).astype(np.uint32)
    seven = lambda s: val(7, s, mtb)                            # noqa: E731
    table[1, :] = [seven(s) for s in range(depth)]              # every slot
    table[2, 0] = seven(0)                                      # first slot
    table[3, depth - 1] = seven(1)                              # last valid slot
    table[8, depth - 1] = seven(2)                              # last slot of an overfull bucket
    for s in (31, 32, 63, 64):
        if s < depth:
            table[4 if s < 40 else 5, s] = seven(s)
    table[6, :min(32, depth)] = seven(3)                        # the first chunk; survivors in the second
    st.table = table
    ids = (table.astype(np.int64) >> mtb) - 1
    valid = np.arange(depth)[None, :] < np.minimum(st.counts, depth)[:, None]
    st.hashesperid = (np.bincount(ids[valid & (table != 0)], minlength=NIDS) + 1).astype(np.uint32)
    return st


REMOVE_SETS = [[7], [0, NIDS - 1, 31, 32, 33], [0, 5], [7, 3, 60, 41], list(range(0, NIDS, 2))]
RETRIEVE_SETS = ([[3], [3, 0], [NIDS - 1, 3, 0], [0, 1, 2, 3], [5, 4, 3, 2, 1], [3, 7, 3, 3, 0, 7],
                  [3, 41, 7, 42, 0, 43, 44, 9], [44, 0, 41]]
                 + [list(np.random.default_rng(k).permutation([i for i in range(NIDS) if not 41 <= i <= 44])[:k])
                    for k in (2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 64, 65)])


def check_remove(st, ids, capsys):
    want = st.copy()
    removed = [ref.remove(want, i) for i in ids]
    ht = ref.mirror(st)
    names = [st.names[i] if k % 2 else i for k, i in enumerate(ids)]       # names and integer ids
    capsys.readouterr()
    ht.remove_batch(names)
    lines = capsys.readouterr().out.splitlines()
    assert lines == ["Removed %s ( %d hashes)." % (nm, r) for nm, r in zip(names, removed)]
    assert ht._dev_newer
    assert_same(ht, want)
    return ht, want


def check_retrieve(ht, st, ids):
    got = ht.retrieve_batch(ids)
    assert len(got) == len(ids)
    for i, rows in zip(ids, got):
        assert rows.dtype == np.int32 and np.array_equal(rows, ref.retrieve(st, i)), i


@pytest.mark.parametrize("depth", [1, 31, 32, 33, 64, 65, 100])
def test_remove_and_retrieve_at_chunk_edges(depth, capsys):
    """Depths around the 32-slot ballot chunks: remove_batch of id sets with id 0, the largest
    id, the bitmap word edges 31/32/33, a largest requested id below ids present in the table,
    ids without entries and every second id equals the statement's removes one by one (removed
    counts included); retrieve_batch of 1-5, 2^k and 2^k + 1 distinct ids, repeated ids and ids
    without entries among ids with many equals the statement before and after a removal."""
    st = edit_table(depth)
    assert (st.counts > depth).any() and (st.counts < depth).any()
    for ids in REMOVE_SETS:
        check_remove(st, ids, capsys)
    ht = ref.mirror(st)
    for ids in RETRIEVE_SETS:
        check_retrieve(ht, st, ids)
    ht, want = check_remove(st, [7, 12, 33], capsys)
    assert want.counts[1] == 0 and not want.table[1].any()
    check_retrieve(ht, want, list(range(NIDS)))
    check_retrieve(ht, want, [9, 7, 9, 0, 33, 68])


def test_retrieve_and_remove_on_2_21_buckets(capsys):
    """2^21 x 4: the per-bucket count scan of retrieve carries across 1024 x 1024 buckets."""
    hb, depth, mtb, nids = 21, 4, 10, 20
    rng = np.random.default_rng(21)
    nb = 1 << hb
    counts = np.where(rng.random(nb) < 0.15, rng.integers(1, 7, nb), 0)
    counts[[0, nb - 1]] = [3, 9]
    st = filled(hb, depth, mtb, nids, 21, counts)
    ht = ref.mirror(st)
    check_retrieve(ht, st, [0, 19, 5, 0, 7, 8, 9, 10, 11, 12])
    check_retrieve(ht, st, list(range(17)))
    ht, want = check_remove(st, [3, 19], capsys)
    check_retrieve(ht, want, [0, 3, 18, 19, 2])


# ---- hits, restriction, pruning bound ---------------------------------------------------------

def hits_table():
    counts = np.resize([0, 3, 7, 8, 9, 20, 1], 1 << 10)
    return filled(10, 8, 12, 30, 13, counts)


def test_get_hits_edges():
    """The probe against orc.get_hits: buckets with counts 0, below, at and above depth; query
    hashes above hashbits (the top hash bit set) and negative; 3,000 query rows; a query without
    hits; an empty query."""
    st = hits_table()
    ht = ref.mirror(st)
    rng = np.random.default_rng(14)
    n = 3000
    q = np.stack([rng.integers(-5000, 5000, n), rng.integers(-(1 << 31), 1 << 31, n)], axis=1).astype(np.int32)
    q[:6, 1] = [512, 1023, -1, 1 << 30, 512 + 1024 * 77, -512]
    for qq in (q, q[:1025], q[:1], q[::-1]):
        assert np.array_equal(ht.get_hits(qq), ref.get_hits(st, qq))
    empty = np.nonzero(st.counts == 0)[0][:40]
    none = np.stack([np.arange(40), empty + 1024 * np.arange(40)], axis=1).astype(np.int32)
    assert ht.get_hits(none).shape == (0, 4)
    assert ht.get_hits(np.zeros((0, 2), np.int32)).shape == (0, 4)


@pytest.mark.parametrize("lo,hi", [(0, 30), (5, 5), (0, 0), (20, 30), (29, 30), (0, 1), (13, 14), (3, 17)])
def test_restricted_table_and_its_hits(lo, hi):
    """restrict_device_ids(lo, hi): the device table equals the statement's restriction, and its
    hits equal the full table's hits of ids in [lo, hi), in order."""
    st = hits_table()
    ht = ref.mirror(st)
    ctx = ht.restrict_device_ids(lo, hi)
    want = st.copy()
    ref.restrict(want, lo, hi)
    table, counts = device_arrays(ctx, st.hashbits, st.depth)
    assert np.array_equal(counts, want.counts) and np.array_equal(table, want.table)
    rng = np.random.default_rng(lo * 31 + hi)
    q = np.stack([rng.integers(0, 4096, 2000), rng.integers(-(1 << 20), 1 << 20, 2000)], axis=1).astype(np.int32)
    full = ref.get_hits(st, q)
    assert np.array_equal(ht.get_hits(q), full[(full[:, 0] >= lo) & (full[:, 0] < hi)])
    assert np.array_equal(ht.table, st.table) and np.array_equal(ht.counts, st.counts)


def test_pruning_bound_follows_every_edit():
    """afp_table_pruning_bound equals the statement after an upload, a store_batch that adds the
    smallest track, a remove_batch of that track, and an upload in which a live entry names a
    track whose hashesperid is 0 (and one in which only removed tracks have 0)."""
    st = hits_table()
    st.hashesperid[[4, 11]] += 1000
    ht = ref.mirror(st)
    ctx = ht._sync_device()
    bound = lambda s: ref.pruning_bound(s.table, s.counts, s.hashesperid, s.maxtimebits)   # noqa: E731
    assert device_bound(ctx) == bound(st) > 0
    rows = np.stack([np.arange(3), np.arange(3) * 7], axis=1)     # buckets 0, 7, 14: empty, no draws
    ht.store_batch(["small"], [rows])
    want = st.copy()
    ref.store(want, ref.name_to_id(want, "small"), rows)
    assert device_bound(ctx) == bound(want) == 3
    ht.remove_batch(["small"])
    ref.remove(want, want.names.index("small"))
    assert device_bound(ctx) == bound(want) == st.hashesperid.min()
    assert_same(ht, want)
    zero = st.copy()
    zero.hashesperid[17] = 0                                     # id 17 still has live entries
    assert bound(zero) == 0
    ht0 = ref.mirror(zero)
    assert device_bound(ht0._sync_device()) == 0
    gone = st.copy()
    ref.remove(gone, 17)
    ht1 = ref.mirror(gone)
    assert device_bound(ht1._sync_device()) == bound(gone) > 0
