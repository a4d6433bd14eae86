"""HashTable.merge_batch (csrc/afp_table_merge.cu) against the host merge, tests/merge_reference.py's
statement and the reference's table-ops fixture: table, counts, names, hashesperid, the next
np.random draw and the matcher's pruning bound, bit for bit."""
import ctypes as C
import os
import random

import numpy as np
import pytest

from audfprint_b200 import HashTable, Matcher, _lib
from audfprint_b200.hash_table import AfpStateError
from audfprint_b200.synth import synth_table
from tests import cases
from tests import merge_reference as mref
from tests import table_reference as ref
from tests.conftest import GOLDEN
from tests.test_table_merge_cpu import StatementTable, random_state

pytestmark = pytest.mark.gpu


class DeviceMergeTable(HashTable):
    """The mirror class with merge routed through merge_batch."""

    def merge(self, ht):
        self.merge_batch([ht])


def pruning_bound(ht):
    ctx = ht._sync_device()
    out = C.c_uint32(0)
    ctx.check(ctx.lib.afp_table_pruning_bound(ctx.h, C.byref(out)))
    return int(out.value)


def _same(ht, st):
    return (np.array_equal(ht.table, st.table) and np.array_equal(ht.counts, st.counts)
            and ht.names == st.names and np.array_equal(ht.hashesperid, st.hashesperid)
            and ht.hashesperid.dtype == np.uint32)


def check_merge(a, others, seed):
    """merge_batch of mirrors of `others` into a mirror of `a` equals the host merge loop and the
    statement, including the next np.random draw and a fresh upload's pruning bound."""
    np.random.seed(seed)
    st = a.copy()
    for o in others:
        mref.merge(st, o)
    want_next = np.random.random()
    np.random.seed(seed)
    host = ref.mirror(a)
    for o in others:
        host.merge(ref.mirror(o))
    assert np.random.random() == want_next
    assert _same(host, st)
    np.random.seed(seed)
    dev = ref.mirror(a)
    dev.dirty = False
    dev.merge_batch([ref.mirror(o) for o in others])
    assert dev._dev_newer and dev.dirty
    assert np.random.random() == want_next
    bound = pruning_bound(dev)                               # the merged device copy, as merge left it
    assert _same(dev, st)
    fresh = ref.mirror(st)
    assert bound == pruning_bound(fresh) == ref.pruning_bound(st.table, st.counts, st.hashesperid, st.maxtimebits)
    return st


def edge_tables(depth, in_depth, hb=7, in_hb=7, mtb=8):
    """Every combination of our count (0, 1, below, at and above depth) with the incoming count that
    makes the pool depth - 1, depth or depth + 1 entries, or is above the incoming depth; stale
    values past every count, names with None."""
    rng = np.random.default_rng(depth * 1000 + in_depth)
    ours = sorted({0, 1, depth // 2, max(0, depth - 1), depth, depth + 1, 3 * depth + 2})
    combos = []
    for c in ours:
        h = min(c, depth)
        for add in sorted({depth - 1 - h, depth - h, depth + 1 - h, 1, in_depth, in_depth + 4, 2 * in_depth + 1}):
            if add >= 1:
                combos.append((c, add if add <= in_depth else in_depth + 3 + add))
    nb, in_nb = 1 << hb, 1 << in_hb
    assert len(combos) <= min(nb, in_nb)
    a = random_state(rng, hb, depth, mtb, 9, 0, over=0.0)
    b = random_state(rng, in_hb, in_depth, mtb, 6, 0, over=0.0)
    slots = rng.permutation(min(nb, in_nb))[:len(combos)]      # neither ascending nor descending
    for s, (c, add) in zip(slots, combos):
        a.counts[s], b.counts[s] = c, add
    return a, b


@pytest.mark.parametrize("depth,in_depth", [(1, 1), (2, 2), (6, 6), (6, 3), (6, 9), (100, 100), (100, 40),
                                            (2, 100), (100, 1)])
def test_every_pool_edge(depth, in_depth):
    """Pools of depth - 1, depth and depth + 1; our counts 0, below, at and above depth; incoming
    counts above its own depth; depth 1, 2, 6 and 100, incoming depth smaller and larger."""
    a, b = edge_tables(depth, in_depth)
    st = check_merge(a, [b], depth * 7 + in_depth)
    assert (st.counts > depth).any()


@pytest.mark.parametrize("hb,in_hb", [(8, 6), (6, 8)])
def test_incoming_hashbits(hb, in_hb):
    """Incoming hashbits smaller, and larger with all its live buckets inside our table."""
    rng = np.random.default_rng(hb)
    a = random_state(rng, hb, 6, 10, 11, 6)
    b = random_state(rng, in_hb, 4, 10, 5, 4)
    b.counts[1 << hb:] = 0
    check_merge(a, [b], hb + 40)


def test_three_tables_and_none_names():
    """A list of three tables (one of them twice) against three host merges; names with None."""
    rng = np.random.default_rng(3)
    a = random_state(rng, 7, 6, 8, 10, 6)
    b, c = random_state(rng, 7, 6, 8, 4, 6), random_state(rng, 6, 9, 8, 7, 9)
    b.names[1] = None
    check_merge(a, [b, c, b], 17)


@pytest.mark.parametrize("in_depth", [32768, 32769])
def test_index_width_limit(in_depth):
    """Pools of 65536 entries (the largest with 16-bit pool indices) and 65537 (32-bit)."""
    rng = np.random.default_rng(in_depth)
    a = random_state(rng, 1, 32768, 8, 5, 0, over=0.0)
    b = random_state(rng, 1, in_depth, 8, 5, 0, over=0.0)
    a.counts[:] = 32768
    b.counts[:] = in_depth + 1
    check_merge(a, [b], 2)


def test_reference_table_ops(golden_match):
    """The reference's store / merge / remove / reuse script with the merge on the device: the
    merged, removed and reused states equal the reference's, and np.random ends where the
    statement leaves it."""
    from oracle.make_golden_table_ops_replay import run
    want = np.load(os.path.join(GOLDEN, "table_ops.npz"))
    run(StatementTable, golden_match, lambda tag, st: None)
    want_next = np.random.random()
    seen = []

    def record(tag, ht):
        seen.append(tag)
        assert np.array_equal(ht.table, want[tag + "/table"]), tag
        assert np.array_equal(ht.counts, want[tag + "/counts"]), tag
        assert np.array_equal(ht.hashesperid, want[tag + "/hashesperid"]), tag
        assert ["" if n is None else n for n in ht.names] == want[tag + "/names"].tolist(), tag
    _, r9, rlate, lines = run(DeviceMergeTable, golden_match, record)
    assert np.random.random() == want_next
    assert seen == ["a", "b", "merged", "removed", "reused"]
    assert np.array_equal(r9, want["retrieve_track9"]) and np.array_equal(rlate, want["retrieve_late"])
    assert lines == want["list_lines"].tolist()


def _names_table(n, mtb=24, hb=4, depth=3):
    ht = HashTable(hashbits=hb, depth=depth, maxtime=1 << mtb)
    ht.names = ["x%d" % i for i in range(n)]
    ht.hashesperid = np.ones(n, np.uint32)
    ht.table[:, 0] = np.uint32(((n - 1 + 1) << mtb) + 5)         # the table's largest id
    ht.counts[:] = 1
    return ht


def test_largest_id_and_errors_leave_everything_unchanged():
    """With 8 id bits the largest id that fits is 254: a merge that reaches it works, one past it
    raises OverflowError; every error case leaves table, counts, names, hashesperid, the device
    copy and np.random as they were."""
    a = _names_table(200)
    a.merge_batch([_names_table(1)])                             # the device copy now leads
    ctx = _lib.context(a.device)
    key = ctx.table_key

    def snapshot():
        return (a.table.copy(), a.counts.copy(), list(a.names), a.hashesperid.copy(), np.random.get_state()[2])
    assert ctx.table_key == key == a._dev_key and a._dev_newer
    np.random.seed(4)
    before = snapshot()
    other = HashTable(hashbits=4, depth=3, maxtime=1 << 12)
    big = HashTable(hashbits=5, depth=3, maxtime=1 << 24)
    big.counts[20] = 1
    pending = _names_table(2)
    tok = pending.store_batch_begin(["y"], [np.zeros((1, 2), np.int32)])
    cases_ = [(OverflowError, [_names_table(10), _names_table(45)]), (AssertionError, [_names_table(1), other]),
              (IndexError, [big]), (ValueError, [_names_table(1), a]), (AfpStateError, [pending])]
    for exc, tables in cases_:
        with pytest.raises(exc):
            a.merge_batch(tables)
        after = snapshot()
        assert all(np.array_equal(x, y) for x, y in zip(before[:2] + before[3:4], after[:2] + after[3:4]))
        assert before[2] == after[2] and before[4] == after[4]
    pending.store_batch_finish(tok)
    a.merge_batch([_names_table(54)])                            # ids up to 254 = 2^8 - 2
    assert len(a.names) == 255 and a.names[-1] == "x53"
    st = ref.State(a.hashbits, a.depth, a.maxtimebits, a.table, a.counts, a.names, a.hashesperid)
    assert pruning_bound(a) == ref.pruning_bound(st.table, st.counts, st.hashesperid, st.maxtimebits) == 1
    with pytest.raises(OverflowError):
        a.merge_batch([_names_table(1)])
    assert a.merge_batch([]) == 0 and len(a.names) == 255
    # a pending store on the table itself
    tok = a.store_batch_begin(["x0"], [np.zeros((1, 2), np.int32)])
    with pytest.raises(AfpStateError):
        a.merge_batch([other])
    a.store_batch_finish(tok)


def test_shard_device_copy_refuses():
    a = _names_table(5, mtb=12)
    a.restrict_device_ids(0, 3)
    with pytest.raises(AfpStateError):
        a.merge_batch([_names_table(2, mtb=12)])
    assert len(a.names) == 5


def test_incoming_device_copy_is_read_first(golden_match):
    """An incoming table whose device copy leads (store_batch) is pulled before `self` takes the
    device; the result equals the host merge of host-built tables."""
    gm = golden_match
    random.seed(8)
    b = HashTable(hashbits=10, depth=6, maxtime=1 << 12)
    b.store_batch(["b%d" % i for i in range(6)], [gm["track%d/hashes" % i][:400] for i in range(6)])
    random.seed(8)
    hb_ = HashTable(hashbits=10, depth=6, maxtime=1 << 12)
    for i in range(6):
        hb_.store("b%d" % i, gm["track%d/hashes" % i][:400])
    a = HashTable(hashbits=10, depth=6, maxtime=1 << 12)
    for i in range(6, 10):
        a.store("a%d" % i, gm["track%d/hashes" % i][:400])
    host = ref.mirror(a)
    np.random.seed(12)
    host.merge(hb_)
    nxt = np.random.random()
    assert b._dev_newer
    np.random.seed(12)
    a.merge_batch([b])
    assert np.random.random() == nxt and _same(a, host)


@pytest.mark.parametrize("force_general", [False, True])
def test_matching_on_the_merged_device_table(golden_match, force_general):
    """Two halves of the golden 40-track database (2^12 x 8, overflowing buckets) merged on the
    device: the matcher rows and get_hits equal those of a fresh upload of the host merge."""
    gm = golden_match
    half = cases.DB_NTRACKS // 2
    random.seed(1234)
    parts = []
    for lo in (0, half):
        ht = HashTable(hashbits=12, depth=8, maxtime=1 << 12)
        for i in range(lo, lo + half):
            ht.store("track%d" % i, gm["track%d/hashes" % i])
        parts.append(ht)
    np.random.seed(77)
    host = ref.mirror(parts[0])
    host.merge(parts[1])
    np.random.seed(77)
    dev = ref.mirror(parts[0])
    dev.merge_batch([parts[1]])
    qs = [gm["q%d_clean/q" % j] for j in range(cases.DB_QUERIES)]
    m = Matcher()
    m.force_general_kernel = force_general
    got = m.match_batch(dev, qs)
    assert dev._dev_newer
    hits = [dev.get_hits(q) for q in qs]
    fresh = ref.mirror(host)
    want = m.match_batch(fresh, qs)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))
    assert all(np.array_equal(h, fresh.get_hits(q)) for h, q in zip(hits, qs))
    assert sum(len(r) for r in got) > 0
    assert _same(dev, host)


def test_bench_geometry_every_bucket_overflows():
    """Two 2^20 x 100 tables, every bucket full with counts above depth, 500,000 ids each: the
    device merge equals the permutation of every pool gathered on the host (the replay is
    np.random.permutation, tests/test_table_merge_cpu.py; spot-checked here against it)."""
    mtb, depth, nids = 12, 100, 500_000
    t1, c1, h1 = synth_table(20, depth, nids, mtb, seed=1)
    t2, c2, h2 = synth_table(20, depth, nids, mtb, seed=2)
    names = ["a%d" % i for i in range(nids)]

    def table(t, c, h, nm):
        ht = HashTable(hashbits=20, depth=1, maxtime=1 << mtb)
        ht.table, ht.counts, ht.hashesperid, ht.depth, ht.names = t, c, h, depth, nm
        return ht
    np.random.seed(6)
    st0 = np.random.get_state()
    dev = table(t1.copy(), c1.copy(), h1, list(names))
    assert dev.merge_batch([table(t2, c2, h2, ["b%d" % i for i in range(nids)])]) == 1 << 20
    nxt = np.random.random()
    # the expected table: pool = our 100 entries then the incoming 100 shifted, permuted
    state = np.empty(625, np.uint32)
    state[:624], state[624] = st0[1], st0[2]
    idx = np.empty((1 << 20, depth), np.int32)
    sizes = np.full(1 << 20, 2 * depth, np.int32)
    assert _lib.load().afp_np_permutation_replay(state.ctypes.data, sizes.ctypes.data, 1 << 20, depth,
                                                 idx.ctypes.data) == 0
    np.random.set_state((st0[0], state[:624], int(state[624]), st0[3], st0[4]))
    assert np.random.random() == nxt
    np.random.set_state(st0)
    for b in range(3):                                       # the replay is np.random.permutation
        pool = np.concatenate([t1[b], t2[b] + np.uint32(nids << mtb)])
        assert np.array_equal(np.random.permutation(pool)[:depth], pool[idx[b]])
    shifted = t2 + np.uint32(nids << mtb)
    want = np.where(idx < depth, np.take_along_axis(t1, np.minimum(idx, depth - 1), axis=1),
                    np.take_along_axis(shifted, np.maximum(idx - depth, 0), axis=1))
    assert np.array_equal(dev.counts, c1 + c2)
    assert np.array_equal(dev.table, want)
    assert len(dev.names) == 2 * nids and np.array_equal(dev.hashesperid, np.concatenate([h1, h2]))
    assert pruning_bound(dev) == min(h1[h1 > 0].min(), h2[h2 > 0].min())
