"""tests/table_reference.py (the sequential statement the device hash-table kernels are held to
by tests/test_gpu_table_edges.py) against tables the reference built (table_ops.npz, both
match.npz databases) and against the host mirror's store / remove / retrieve / get_entry."""
import os
import random

import numpy as np
import pytest

from audfprint_b200 import HashTable
from tests import cases
from tests import table_reference as ref
from tests.conftest import GOLDEN, expand_table


mirror = ref.mirror


class StatementTable(ref.State):
    """The statement behind the HashTable methods the table-ops script calls (merge is the host
    mirror's: its np.random.permutation draws are not part of the statement)."""

    def __init__(self, hashbits, depth, maxtime):
        super().__init__(hashbits, depth, int(maxtime).bit_length() - 1)

    def store(self, name, rows):
        ref.store(self, ref.name_to_id(self, name), rows)

    def merge(self, other):
        a = mirror(self)
        a.merge(mirror(other))
        self.table, self.counts, self.names, self.hashesperid = a.table, a.counts, a.names, a.hashesperid

    def remove(self, name):
        ref.remove(self, ref.name_to_id(self, name))

    def retrieve(self, name):
        return ref.retrieve(self, ref.name_to_id(self, name))

    def list(self, emit):
        for track, nh in zip(self.names, self.hashesperid):
            if track:
                emit("%s (%s hashes)" % (track, nh))


def test_statement_replays_the_reference_table_ops(golden_match):
    """The store / merge / remove / slot-reuse sequence the reference ran on a 2^10 x 6 table
    (most buckets overflow): every snapshot, both retrieves and the list lines."""
    from oracle.make_golden_table_ops_replay import run
    want = np.load(os.path.join(GOLDEN, "table_ops.npz"))
    seen = []

    def record(tag, st):
        seen.append(tag)
        assert np.array_equal(st.table, want[tag + "/table"]), tag
        assert np.array_equal(st.counts, want[tag + "/counts"]), tag
        assert np.array_equal(st.hashesperid, want[tag + "/hashesperid"]), tag
        assert ["" if n is None else n for n in st.names] == want[tag + "/names"].tolist(), tag
    st, r9, rlate, lines = run(StatementTable, golden_match, record)
    assert seen == ["a", "b", "merged", "removed", "reused"]
    assert np.array_equal(r9, want["retrieve_track9"]) and r9.dtype == np.int32
    assert np.array_equal(rlate, want["retrieve_late"])
    assert lines == want["list_lines"].tolist()
    assert st.names[3] == "late"


@pytest.mark.parametrize("db", ["db", "db2"])
def test_statement_rebuilds_the_match_databases(golden_match, db):
    """Both 40-track databases of match.npz (2^20 x 20; 2^12 x 8 with overflowing buckets) from
    random.seed(1234), and the hits of every golden query on them."""
    gm = golden_match
    table, counts, hashbits, depth, mtb, hpi = expand_table(gm, db)
    st = ref.State(hashbits, depth, mtb)
    random.seed(1234)
    for i in range(cases.DB_NTRACKS):
        ref.store(st, ref.name_to_id(st, "track%d" % i), gm["track%d/hashes" % i])
    assert np.array_equal(st.counts, counts) and np.array_equal(st.table, table)
    assert np.array_equal(st.hashesperid, hpi)
    assert st.names == ["track%d" % i for i in range(cases.DB_NTRACKS)]
    assert ref.pruning_bound(st.table, st.counts, st.hashesperid, mtb) == hpi.min()
    for j in range(cases.DB_QUERIES):
        key = "q%d_clean" % j
        assert np.array_equal(ref.get_hits(st, gm[key + "/q"]), gm["%s/%s/hits" % (db, key)]), key


def _random_ops(seed, nops):
    """A seeded sequence of (op, name, rows): stores of new and known names, removes that free
    names for reuse, retrieves; hashes beyond hashbits and negative, times beyond maxtimebits."""
    rng = np.random.default_rng(seed)
    ops, live = [], []
    for k in range(nops):
        r = rng.random()
        if r < 0.6 or not live:
            name = "n%d" % rng.integers(12)
            n = int(rng.integers(0, 120))
            rows = np.stack([rng.integers(-600, 600, n), rng.integers(-300, 300, n)], axis=1).astype(np.int32)
            ops.append(("store", name, rows))
            if name not in live:
                live.append(name)
        elif r < 0.8:
            name = live.pop(int(rng.integers(len(live))))
            ops.append(("remove", name, None))
        else:
            ops.append(("retrieve", live[int(rng.integers(len(live)))], None))
    return ops


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_statement_equals_the_host_mirror(seed, capsys):
    """Random store / remove / retrieve sequences on a 2^5 x 6 table with 8 time bits (buckets
    overflow, names are freed and taken again): after every step the statement and the host
    methods hold the same table, counts, names and hashesperid, `get_entry` equals the
    statement's hits, and `random` ends in the same state."""
    hb, depth, mtb = 5, 6, 8
    ops = _random_ops(seed, 60)
    random.seed(seed)
    st = ref.State(hb, depth, mtb)
    got = []
    for op, name, rows in ops:
        if op == "store":
            ref.store(st, ref.name_to_id(st, name), rows)
        elif op == "remove":
            got.append(ref.remove(st, st.names.index(name)))
        else:
            got.append(ref.retrieve(st, st.names.index(name)))
        got.append((st.table.copy(), st.counts.copy(), list(st.names), st.hashesperid.copy()))
    after = random.random()

    random.seed(seed)
    ht = HashTable(hashbits=hb, depth=depth, maxtime=1 << mtb)
    k = 0
    for op, name, rows in ops:
        if op == "store":
            ht.store(name, rows)
        elif op == "remove":
            capsys.readouterr()
            ht.remove(name)
            assert capsys.readouterr().out == "Removed %s ( %d hashes).\n" % (name, got[k])
            k += 1
        else:
            assert np.array_equal(ht.retrieve(name), got[k])
            k += 1
        table, counts, names, hpi = got[k]
        k += 1
        assert np.array_equal(ht.table, table) and np.array_equal(ht.counts, counts)
        assert ht.names == names and np.array_equal(ht.hashesperid, hpi)
    assert random.random() == after
    assert (st.counts > depth).any()
    for h in range(1 << hb):
        hits = ref.get_hits(st, [[0, h], [0, h - (1 << hb)]])
        n = len(hits) // 2
        assert np.array_equal(ht.get_entry(h), hits[:n, :2]), h
        assert np.array_equal(hits[:n], hits[n:])


def test_statement_restrict_and_pruning_bound():
    """restrict keeps one id range among the valid slots; the pruning bound is the smallest
    non-zero hashesperid unless a valid slot names a zero-hashesperid id (slots past the count
    do not count)."""
    mtb = 4
    v = lambda i, t: ((i + 1) << mtb) + t                                          # noqa: E731
    table = np.array([[v(0, 1), v(2, 2), v(1, 3)], [v(2, 5), v(3, 6), 0], [v(3, 7), v(1, 1), v(0, 0)]], np.uint32)
    table = np.vstack([table, np.zeros((1, 3), np.uint32)])
    counts = np.array([5, 2, 1, 0], np.int32)
    st = ref.State(2, 3, mtb, table, counts, ["a", "b", "c", "d"], [4, 2, 3, 1])
    assert ref.pruning_bound(st.table, st.counts, st.hashesperid, mtb) == 1
    assert ref.pruning_bound(st.table, st.counts, [4, 2, 3, 0], mtb) == 0              # id 3 at (1, 1)
    assert ref.pruning_bound(st.table, st.counts, [4, 0, 3, 5], mtb) == 0              # id 1 at (0, 2)
    assert ref.pruning_bound(st.table, np.array([1, 1, 1, 0]), [4, 0, 3, 5], mtb) == 3  # id 1 only past counts
    assert ref.pruning_bound(st.table, st.counts, [0, 0, 0, 0], mtb) == 0
    r = st.copy()
    ref.restrict(r, 1, 3)
    assert r.table.tolist() == [[v(2, 2), v(1, 3), 0], [v(2, 5), 0, 0], [0, v(1, 1), v(0, 0)], [0, 0, 0]]
    assert r.counts.tolist() == [2, 1, 0, 0]
    r = st.copy()
    ref.restrict(r, 0, 0)
    assert not r.counts.any() and not r.table[:, 0].any()
    r = st.copy()
    assert ref.remove(r, 0) == 2                                                   # (0, 0) and (2, 2), past the count
    assert r.table.tolist() == [[v(2, 2), v(1, 3), 0], [v(2, 5), v(3, 6), 0], [v(3, 7), 0, 0], [0, 0, 0]]
    assert r.counts.tolist() == [2, 2, 1, 0] and r.names[0] is None and r.hashesperid[0] == 0


def test_store_batch_checks_integer_ids_before_the_device():
    """An integer id outside the table's names raises IndexError before any device call (so also
    on a machine without a GPU) and changes nothing; an id that a new name of the same batch
    creates is in range."""
    ht = HashTable(hashbits=4, depth=2, maxtime=1 << 8)
    ht.names, ht.hashesperid = ["a", None], np.array([3, 0], np.uint32)
    rows = np.zeros((1, 2), np.int32)
    for bad in (["x", 2], [-1], ["a", 3, "y"], [2, "z"]):
        with pytest.raises(IndexError):
            ht.store_batch(bad, [rows] * len(bad))
        assert ht.names == ["a", None] and ht.hashesperid.tolist() == [3, 0]
        assert not getattr(ht, "_store_pending", False)
    assert ht._plan_ids(["x", "y", 2, 1, "a"])[0].tolist() == [1, 2, 2, 1, 0]
