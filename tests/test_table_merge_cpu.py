"""The host half of HashTable.merge_batch and the statement its device kernels are held to:
afp_np_permutation_replay (csrc/afp_table_merge.cu) against np.random.permutation, and
tests/merge_reference.py's merge against the table the reference merged (table_ops.npz) and the
host mirror's merge."""
import os

import numpy as np
import pytest

from audfprint_b200 import _lib
from tests import merge_reference as mref
from tests import table_reference as ref
from tests.conftest import GOLDEN


def _state():
    st = np.random.get_state()
    s = np.empty(625, np.uint32)
    s[:624], s[624] = st[1], st[2]
    return s


def _replay(state, sizes, keep):
    sizes = np.ascontiguousarray(sizes, np.int32)
    out = np.full((len(sizes), keep), -1, np.int32)
    rc = _lib.load().afp_np_permutation_replay(state.ctypes.data, sizes.ctypes.data, len(sizes), keep,
                                               out.ctypes.data)
    return rc, out


def _advance(nwords):
    """Move the global generator's position by drawing nwords raw 32-bit words."""
    if nwords:
        np.random.randint(0, 1 << 32, size=nwords, dtype=np.uint64)   # one word per value below 2^32


def _check_pools(sizes, keep, seed, skip):
    np.random.seed(seed)
    _advance(skip)
    np.random.standard_normal()                         # leaves a cached Gaussian in the state
    before = np.random.get_state()
    assert before[3] == 1
    state = _state()
    rc, got = _replay(state, sizes, keep)
    assert rc == 0
    want = np.stack([np.random.permutation(np.arange(n, dtype=np.uint32))[:keep] for n in sizes])
    after = np.random.get_state()
    assert np.array_equal(got, want)
    assert np.array_equal(state[:624], after[1]) and int(state[624]) == after[2]
    # written back as merge_batch does: the cached Gaussian survives
    np.random.set_state((before[0], state[:624].copy(), int(state[624]), before[3], before[4]))
    assert np.random.standard_normal() == before[4]


@pytest.mark.parametrize("skip", [0, 1, 300, 623, 624, 625, 1247])
def test_replay_equals_numpy_permutation_every_pool_size(skip):
    """Pools of 2 .. 2 * depth entries (depth 100) and their first `depth` survivors, from states
    whose position lies at, inside and across the 624-word blocks."""
    depth = 100
    sizes = np.arange(depth, 2 * depth + 1)
    _check_pools(sizes, depth, 11 + skip, skip)
    for n in range(2, 2 * depth + 1):                                  # every size, whole permutation
        _check_pools([n], n, 3 + n, skip)


def test_replay_at_the_rejection_mask_edges():
    """Sizes at 2^k and 2^k +- 1 (the mask of random_interval changes there), up to 2^17 + 1."""
    sizes = sorted({max(2, (1 << k) + d) for k in range(1, 18) for d in (-1, 0, 1)})
    for n in sizes:
        _check_pools([n], min(n, 300), 1000 + n, n % 700)
    _check_pools(sizes, 2, 5, 17)                                    # all of them in one call


def test_replay_rejects_bad_sizes():
    np.random.seed(9)
    state = _state()
    keep = state.copy()
    for sizes, k in (([5, 3], 4), ([0], 1), ([7], 0), ([-1], 1)):
        rc, _ = _replay(state, sizes, k)
        assert rc == -2 and np.array_equal(state, keep)
    bad = state.copy()
    bad[624] = 625
    assert _replay(bad, [3], 2)[0] == -2
    assert _replay(state, np.zeros(0, np.int32), 3)[0] == 0 and np.array_equal(state, keep)


class StatementTable(ref.State):
    """The statement behind the HashTable methods the table-ops script calls, merge included."""

    def __init__(self, hashbits, depth, maxtime):
        super().__init__(hashbits, depth, int(maxtime).bit_length() - 1)

    def store(self, name, rows):
        ref.store(self, ref.name_to_id(self, name), rows)

    def merge(self, other):
        mref.merge(self, other)

    def remove(self, name):
        ref.remove(self, ref.name_to_id(self, name))

    def retrieve(self, name):
        return ref.retrieve(self, ref.name_to_id(self, name))

    def list(self, emit):
        for track, nh in zip(self.names, self.hashesperid):
            if track:
                emit("%s (%s hashes)" % (track, nh))


def test_statement_merge_replays_the_reference_table_ops(golden_match):
    """The reference's store / merge / remove / reuse sequence (2^10 x 6, most buckets overflow)
    with the statement's merge: the merged, removed and reused states equal the reference's."""
    from oracle.make_golden_table_ops_replay import run
    want = np.load(os.path.join(GOLDEN, "table_ops.npz"))
    seen = []

    def record(tag, st):
        seen.append(tag)
        assert np.array_equal(st.table, want[tag + "/table"]), tag
        assert np.array_equal(st.counts, want[tag + "/counts"]), tag
        assert np.array_equal(st.hashesperid, want[tag + "/hashesperid"]), tag
        assert ["" if n is None else n for n in st.names] == want[tag + "/names"].tolist(), tag
    _, r9, rlate, lines = run(StatementTable, golden_match, record)
    assert seen == ["a", "b", "merged", "removed", "reused"]
    assert np.array_equal(r9, want["retrieve_track9"]) and np.array_equal(rlate, want["retrieve_late"])


def random_state(rng, hashbits, depth, mtb, nnames, fill, over=0.3):
    """A table whose counts run from 0 to above depth, with stale values past every count and
    entries of ids in [0, nnames); some names are None."""
    nb = 1 << hashbits
    counts = rng.integers(0, fill + 1, nb).astype(np.int32)
    counts[rng.random(nb) < over] += depth
    ids = rng.integers(0, max(1, nnames), (nb, depth))
    table = (((ids + 1) << mtb) + rng.integers(0, 1 << mtb, (nb, depth))).astype(np.uint32)
    names = ["n%d" % rng.integers(1 << 30) if rng.random() > 0.2 else None for _ in range(nnames)]
    return ref.State(hashbits, depth, mtb, table, counts, names, rng.integers(0, 500, nnames))


@pytest.mark.parametrize("case", [(5, 6, 5, 6), (5, 6, 4, 3), (5, 6, 6, 9), (6, 2, 6, 1), (4, 100, 4, 100),
                                  (4, 1, 3, 1)])
def test_statement_merge_equals_the_host_mirror(case):
    """Random tables of several geometries (incoming hashbits smaller, equal and larger with its
    live buckets inside; depth smaller and larger): the statement and the mirror's merge give the
    same table, counts, names, hashesperid and np.random state, and the first statement agrees
    with a second merge on top."""
    hb, depth, hb2, depth2 = case
    rng = np.random.default_rng(sum(case))
    a = random_state(rng, hb, depth, 8, 7, depth)
    b = random_state(rng, hb2, depth2, 8, 5, depth2)
    b.counts[1 << hb:] = 0
    c = random_state(rng, min(hb, hb2), depth2, 8, 3, depth2)
    np.random.seed(sum(case) + 1)
    st = a.copy()
    mref.merge(st, b)
    mref.merge(st, c)
    after = np.random.random()
    np.random.seed(sum(case) + 1)
    ht = ref.mirror(a)
    ht.merge(ref.mirror(b))
    ht.merge(ref.mirror(c))
    assert np.random.random() == after
    assert np.array_equal(ht.table, st.table) and np.array_equal(ht.counts, st.counts)
    assert ht.names == st.names and np.array_equal(ht.hashesperid, st.hashesperid)
    assert (st.counts > depth).any()
