"""HashTable.remove / retrieve on the device table, a batch of names per pass
(csrc/afp_table_edit.cu): against the live reference's table-ops fixture, the host methods and a
vectorised NumPy statement of the semantics."""
import os
import random

import numpy as np
import pytest

from audfprint_b200 import Analyzer, HashTable, Matcher, _lib
from audfprint_b200.hash_table import AfpStateError
from audfprint_b200.synth import synth_query, synth_table, synth_track
from tests.conftest import GOLDEN, expand_table

pytestmark = pytest.mark.gpu


class DeviceEditTable(HashTable):
    """The mirror class with store / remove / retrieve routed through the batched device forms."""

    def store(self, name, timehashpairs):
        self.store_batch([name], [timehashpairs])

    def remove(self, name):
        self.remove_batch([name])

    def retrieve(self, name):
        return self.retrieve_batch([name])[0]


def _table(table, counts, hashbits, depth, mtb, hpi, names=None):
    ht = HashTable(hashbits=hashbits, depth=depth, maxtime=1 << mtb)
    ht.table, ht.counts = table.copy(), counts.copy()
    ht.hashesperid = np.asarray(hpi, np.uint32).copy()
    ht.names = list(names) if names is not None else ["track%d" % i for i in range(len(hpi))]
    return ht


def _same_state(a, b):
    return (np.array_equal(a.table, b.table) and np.array_equal(a.counts, b.counts)
            and np.array_equal(a.hashesperid, b.hashesperid) and a.names == b.names)


def pruning_bound(ht):
    """The device table's pruning bound (smallest non-zero hashesperid; 0 = no pruning)."""
    import ctypes as C
    ctx = _lib.context(ht.device)
    out = C.c_uint32(0)
    ctx.check(ctx.lib.afp_table_pruning_bound(ctx.h, C.byref(out)))
    return int(out.value)


def numpy_remove(table, counts, hpi, names, ids, mtb):
    """The remove semantics as array operations: a bucket holding an entry of a removed id keeps
    its other entries below min(count, depth) in slot order, zero-fills the rest and takes their
    number as its count; per-id removed counts over the whole row."""
    table, counts, hpi, names = table.copy(), counts.copy(), hpi.copy(), list(names)
    depth = table.shape[1]
    gone = np.zeros(len(hpi) + 1, bool)
    gone[np.asarray(ids, np.int64) + 1] = True
    owner = table >> np.uint32(mtb)                       # id + 1; 0 = empty slot
    owner[owner > len(hpi)] = 0
    mine = gone[owner]
    rows = np.nonzero(mine.any(axis=1))[0]
    removed = np.bincount(owner[rows][mine[rows]].astype(np.int64) - 1, minlength=len(hpi))[np.asarray(ids, np.int64)]
    sub, msub = table[rows], mine[rows]
    valid = np.arange(depth)[None, :] < np.minimum(counts[rows], depth)[:, None]
    keep = valid & ~msub
    order = np.argsort(~keep, axis=1, kind="stable")
    new = np.take_along_axis(sub, order, axis=1)
    new[~np.take_along_axis(keep, order, axis=1)] = 0
    table[rows] = new
    counts[rows] = keep.sum(axis=1)
    for i in ids:
        names[i] = None
        hpi[i] = 0
    return table, counts, hpi, names, removed


def test_device_edits_replay_the_reference_table_ops(golden_match, capsys):
    """The scripted store / merge / remove / slot-reuse / retrieve / list sequence of
    oracle/make_golden_table_ops.py (2^10 x 6 table, most buckets overflow) with store, remove and
    retrieve on the device: every snapshot, both retrieves and the list lines equal the reference's."""
    from oracle.make_golden_table_ops_replay import run
    want = np.load(os.path.join(GOLDEN, "table_ops.npz"))
    seen = []

    def record(tag, ht):
        seen.append(tag)
        assert np.array_equal(ht.table, want[tag + "/table"]), tag
        assert np.array_equal(ht.counts, want[tag + "/counts"]), tag
        assert np.array_equal(ht.hashesperid, want[tag + "/hashesperid"]), tag
        assert ["" if n is None else n for n in ht.names] == want[tag + "/names"].tolist(), tag
    ht, r9, rlate, lines = run(DeviceEditTable, golden_match, record)
    assert seen == ["a", "b", "merged", "removed", "reused"]
    assert np.array_equal(r9, want["retrieve_track9"]) and r9.dtype == np.int32
    assert np.array_equal(rlate, want["retrieve_late"])
    assert lines == want["list_lines"].tolist()
    assert ht.names[3] == "late" and "Removed track3 ( 335 hashes)." in capsys.readouterr().out


@pytest.mark.parametrize("db", ["db", "db2"])
def test_batch_equals_the_host_loop(golden_match, capsys, db):
    """Both golden databases (roomy; 2^12 x 8 with overflowing buckets): remove_batch of seeded
    subsets equals the host remove loop (arrays, names, printed lines); retrieve_batch of every
    track, with repeats and integer ids, equals host retrieve."""
    table, counts, hashbits, depth, mtb, hpi = expand_table(golden_match, db)
    n = len(hpi)
    rng = np.random.default_rng(7)
    ten = ["track%d" % i for i in rng.choice(n, 10, replace=False)]
    ten[4] = int(ten[4][5:])                                    # one given as an integer id
    for subset in ([], ["track%d" % int(rng.integers(n))], ten, ["track%d" % i for i in rng.permutation(n)]):
        host = _table(table, counts, hashbits, depth, mtb, hpi)
        capsys.readouterr()
        for name in subset:
            host.remove(name)
        want_out = capsys.readouterr().out
        dev = _table(table, counts, hashbits, depth, mtb, hpi)
        dev.remove_batch(subset)
        assert capsys.readouterr().out == want_out
        assert dev._dev_newer == bool(subset)
        assert _same_state(dev, host), subset
    host = _table(table, counts, hashbits, depth, mtb, hpi)
    dev = _table(table, counts, hashbits, depth, mtb, hpi)
    req = ["track%d" % i for i in range(n)] + ["track3", 5, "track0", 39, "track3"]
    got = dev.retrieve_batch(req)
    assert len(got) == len(req)
    for name, rows in zip(req, got):
        want = host.retrieve(name)
        assert rows.dtype == np.int32 and np.array_equal(rows, want), name
    # after a device removal: removed tracks come back empty, the others unchanged
    dev.remove_batch(ten)
    for i, rows in enumerate(dev.retrieve_batch(list(range(n)))):
        want = host.retrieve(i) if dev.names[i] is not None else np.zeros((0, 2), np.int32)
        assert np.array_equal(rows, want), i


def test_bench_geometry():
    """2^20 x 100, 1 M ids, every bucket full and counts above depth: remove_batch of 1000 names
    equals the NumPy statement of the semantics, which equals the host loop on 3 of them;
    retrieve_batch of 1000 names equals host retrieve on a sample."""
    mtb = 12
    table, counts, hpi = synth_table(hashbits=20, depth=100, nids=1_000_000, maxtimebits=mtb, seed=5)
    names = ["t%d" % i for i in range(len(hpi))]
    rng = np.random.default_rng(9)
    pick = rng.choice(len(hpi), 1000, replace=False)
    ht = _table(table, counts, 20, 100, mtb, hpi, names)
    got = ht.retrieve_batch([names[i] for i in pick])
    host = _table(table, counts, 20, 100, mtb, hpi, names)
    for k in rng.choice(1000, 8, replace=False):
        assert np.array_equal(got[k], host.retrieve(names[pick[k]])), k
    assert sum(len(g) for g in got) == int(hpi[pick].sum())            # every entry lies below depth

    ht.remove_batch([names[i] for i in pick])
    w_table, w_counts, w_hpi, w_names, w_removed = numpy_remove(table, counts, hpi, names, pick, mtb)
    assert np.array_equal(w_removed, hpi[pick])
    assert np.array_equal(ht.hashesperid, w_hpi) and ht.names == w_names
    assert np.array_equal(ht.counts, w_counts) and np.array_equal(ht.table, w_table)
    del w_table
    three = pick[:3]
    for i in three:
        host.remove(names[i])
    t3, c3, h3, n3, _ = numpy_remove(table, counts, hpi, names, three, mtb)
    assert np.array_equal(host.counts, c3) and np.array_equal(host.table, t3)
    assert np.array_equal(host.hashesperid, h3) and host.names == n3


@pytest.mark.parametrize("force_general", [False, True])
def test_matching_after_device_removal(force_general):
    """ingest_batch on the device, remove tracks on the device (the one with the smallest
    hashesperid among them), match: the rows equal those of a host-built table with host removes,
    and no removed id is ever reported."""
    sigs = [synth_track(9100 + i, 10.0 + (i % 5)) for i in range(20)]
    names = ["t%d" % i for i in range(20)]
    random.seed(21)
    dev = HashTable(hashbits=12, depth=20, maxtime=1 << 12)
    Analyzer().ingest_batch(dev, names, sigs)
    random.seed(21)
    host = HashTable(hashbits=12, depth=20, maxtime=1 << 12)
    Analyzer().ingest_batch(host, names, sigs, on_device=False)
    assert np.array_equal(dev.hashesperid, host.hashesperid)
    hpi = host.hashesperid.copy()
    smallest = np.nonzero(hpi == hpi.min())[0].tolist()
    gone = sorted(set(smallest) | {2, 7, 15})
    assert dev._dev_newer
    assert pruning_bound(dev) == hpi.min()
    dev.remove_batch([names[i] for i in gone])
    for i in gone:
        host.remove(names[i])
    assert dev._dev_newer
    # the fast kernel's pruning bound follows the removal: the smallest hashesperid left
    assert pruning_bound(dev) == np.delete(hpi, gone).min() > hpi.min()
    qan = Analyzer()
    qan.shifts = 4
    qs = qan.fingerprint_batch([synth_query(sigs[j], j, seconds=8.0, noise_sigma=0.01)[0] for j in (2, 3, 7, 11, 15, 19)])
    m = Matcher()
    m.force_general_kernel = force_general
    got = m.match_batch(dev, qs)
    want = m.match_batch(host, qs)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    assert not any(np.isin(r[:, 0], gone).any() for r in got)
    assert [int(got[k][0, 0]) for k in (1, 3, 5)] == [3, 11, 19]
    assert _same_state(dev, host)


def test_no_round_trip_after_store_batch(golden_match, capsys, monkeypatch):
    """After store_batch the per-name remove / retrieve run on the device copy: it stays the
    current one, nothing is downloaded or uploaded, and the results equal the host path."""
    gm = golden_match
    tracks = [gm["track%d/hashes" % i] for i in range(12)]
    names = ["t%d" % i for i in range(12)]
    random.seed(3)
    dev = HashTable(hashbits=10, depth=8, maxtime=1 << 12)
    dev.store_batch(names, tracks)
    random.seed(3)
    host = HashTable(hashbits=10, depth=8, maxtime=1 << 12)
    for n, t in zip(names, tracks):
        host.store(n, t)
    ctx = _lib.context(dev.device)
    key = ctx.table_key
    assert dev._dev_newer and key == dev._stamp()

    def no_download():
        raise AssertionError("the device copy was downloaded")
    monkeypatch.setattr(dev, "_pull_device", no_download)
    r = dev.retrieve("t4")
    assert ctx.table_key == key and dev._dev_newer
    assert np.array_equal(r, host.retrieve("t4"))
    capsys.readouterr()
    dev.remove("t4")
    out = capsys.readouterr().out
    assert dev._dev_newer and ctx.table_key == dev._stamp() == dev._dev_key
    host.remove("t4")
    assert capsys.readouterr().out == out
    monkeypatch.undo()
    assert _same_state(dev, host)


def test_errors_leave_everything_unchanged(golden_match):
    table, counts, hashbits, depth, mtb, hpi = expand_table(golden_match, "db2")
    ht = _table(table, counts, hashbits, depth, mtb, hpi)
    ht.remove_batch(["track1"])                           # the device copy now leads
    ctx = _lib.context(ht.device)
    key, names, hpi1 = ctx.table_key, list(ht.names), ht.hashesperid.copy()
    for bad in (["track2", "nosuch"], ["track2", "track2"], ["track2", 2], ["track2", len(hpi)], [-1]):
        with pytest.raises(ValueError):
            ht.remove_batch(bad)
        assert ctx.table_key == key and ht.names == names and np.array_equal(ht.hashesperid, hpi1)
    for bad in (["nosuch"], [len(hpi)], [-1]):
        with pytest.raises(ValueError):
            ht.retrieve_batch(bad)
    assert ht._dev_newer and ctx.table_key == key
    want = numpy_remove(table, counts, hpi, ht.names, [1], mtb)
    assert np.array_equal(ht.table, want[0]) and np.array_equal(ht.counts, want[1])
    # a pending store_batch_begin, then a shard of the device copy
    tok = ht.store_batch_begin(["new"], [golden_match["track0/hashes"]])
    with pytest.raises(AfpStateError):
        ht.remove_batch(["track3"])
    with pytest.raises(AfpStateError):
        ht.retrieve_batch(["track3"])
    ht.store_batch_finish(tok)
    _ = ht.table                                          # host arrays current again before the shard
    ht.restrict_device_ids(0, 10)
    with pytest.raises(AfpStateError):
        ht.remove_batch(["track3"])
    with pytest.raises(AfpStateError):
        ht.retrieve_batch(["track3"])
    assert ht.names[3] == "track3"
    # once another table has taken the device, the shard is gone: the whole table goes up again
    other = _table(table, counts, hashbits, depth, mtb, hpi)
    other.get_hits(np.zeros((1, 2), np.int32))
    want_rows = ht.retrieve(3)
    assert np.array_equal(ht.retrieve_batch(["track3"])[0], want_rows) and len(want_rows)
    ht.remove_batch(["track3"])
    assert ht.names[3] is None and ht._shard is None
    assert not ((ht.table >> np.uint32(mtb)) == 3 + 1).any()
