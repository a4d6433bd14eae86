"""One table from a multi-GPU ingest: per-rank tables exported to device snapshots
(HashTable.export_device, afp_table_export) and merged through merge_batch
(afp_table_merge_device), and dist.ingest_sharded end to end, against the statement of the
reference's multiproc_add (tests/ingest_merge_reference.py) and what the reference built
(tests/golden/ingest_merge.npz): table, counts, names, hashesperid, report lines, the next np.random
draw and the matcher's pruning bound."""
import datetime
import os
import random
import socket

import numpy as np
import pytest
import torch

from audfprint_b200 import Analyzer, HashTable, Matcher, _lib
from audfprint_b200 import dist as afd
from audfprint_b200.hash_table import DeviceTable
from audfprint_b200.synth import synth_table, synth_track
from tests import ingest_merge_reference as im
from tests import table_reference as ref
from tests.conftest import GOLDEN
from tests.test_gpu_table_merge import _same, pruning_bound

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden_ingest():
    return np.load(os.path.join(GOLDEN, "ingest_merge.npz"))


def rank_tables(files, ncores, hb, depth, mtb, seeds):
    """Worker r's table built on the device (store_batch) from random.seed(seeds[r])."""
    out = []
    for r, idx in enumerate(im.deal(len(files), ncores)):
        random.seed(seeds[r])
        w = HashTable(hashbits=hb, depth=depth, maxtime=1 << mtb)
        w.store_batch([files[i][0] for i in idx], [files[i][1] for i in idx])
        out.append(w)
    return out


def statement(base, files, ncores, seeds, np_seed):
    st = base.copy()
    np.random.seed(np_seed)
    lines = im.multiproc_add(st, files, ncores, seeds)
    return st, lines, np.random.random()


def check(ht, st, nxt):
    """ht equals the statement st, np.random continues with nxt, and the pruning bound the merge
    left on the device equals a fresh upload's and the statement's."""
    assert np.random.random() == nxt
    bound = pruning_bound(ht)
    assert _same(ht, st)
    fresh = ref.mirror(st)
    assert bound == pruning_bound(fresh) == ref.pruning_bound(st.table, st.counts, st.hashesperid, st.maxtimebits)


def device_state(ht):
    ctx = ht._sync_device()
    nb = 1 << int(ht.hashbits)
    t = np.empty((nb, int(ht.depth)), np.uint32)
    c = np.empty(nb, np.int32)
    ctx.check(ctx.lib.afp_table_download(ctx.h, t.ctypes.data, c.ctypes.data))
    return t, c


# ---- in one process: W per-rank tables, exported and merged -----------------------------------
@pytest.mark.parametrize("mode,ncores", im.CASES)
def test_snapshot_merge_equals_the_reference(golden_match, golden_ingest, mode, ncores):
    """W = 1, 2, 3, 5 per-rank tables (and 3 files on 5 ranks) merged as snapshots into an empty
    table (`new`) and into a loaded base with a freed name (`add`): the statement and the golden."""
    want = golden_ingest
    files = im.fixture_files(golden_match, mode)
    seeds = [im.SEED + r for r in range(ncores)]
    base = im.golden_base(want, mode)
    st, lines, nxt = statement(base, files, ncores, seeds, im.NP_SEED)
    key = "%s_%d" % (mode, ncores)
    assert lines == want[key + "/report"].tolist() and nxt == float(want[key + "/np_next"])
    ws = rank_tables(files, ncores, im.HASHBITS, im.DEPTH, im.MAXTIMEBITS, seeds)
    snaps = [w.export_device() for w in ws]
    for w, s in zip(ws, snaps):
        assert np.array_equal(s.table.cpu().numpy().view(np.uint32), w.table)
        assert np.array_equal(s.counts.cpu().numpy(), w.counts) and s.names == w.names
    ht = ref.mirror(base)
    ht.dirty = False
    np.random.seed(im.NP_SEED)
    ht.merge_batch(snaps)
    assert ht._dev_newer and ht.dirty
    check(ht, st, nxt)
    assert np.array_equal(ht.table, want[key + "/table"]) and np.array_equal(ht.counts, want[key + "/counts"])
    assert ht.names == im.golden_names(want, key)


def test_raw_counts_above_depth_are_clipped_by_the_first_merge(golden_match, golden_ingest):
    """A per-rank table keeps raw counts above depth; merged into an empty table they become depth,
    so the merged table is not the rank's table (the root cannot adopt it)."""
    files = im.fixture_files(golden_match)
    w, = rank_tables(files, 1, im.HASHBITS, im.DEPTH, im.MAXTIMEBITS, [im.SEED])
    assert (w.counts > im.DEPTH).any()
    ht = HashTable(hashbits=im.HASHBITS, depth=im.DEPTH, maxtime=1 << im.MAXTIMEBITS)
    np.random.seed(im.NP_SEED)
    ht.merge_batch([w.export_device()])
    assert np.array_equal(ht.counts, np.minimum(w.counts, im.DEPTH))
    assert np.array_equal(ht.counts, golden_ingest["new_1/counts"])


@pytest.mark.parametrize("depth", [1, 2])
def test_depth_one_and_two(golden_match, depth):
    """Depth 1 and 2: three files on four ranks (one without files)."""
    files = [("f%d" % i, np.asarray(golden_match["track%d/hashes" % (i + 10)], np.int32)[:300]) for i in range(3)]
    seeds = [7, 8, 9, 10]
    base = ref.State(8, depth, 12)
    st, _, nxt = statement(base, files, 4, seeds, 31)
    assert (st.counts > depth).any()
    snaps = [w.export_device() for w in rank_tables(files, 4, 8, depth, 12, seeds)]
    ht = ref.mirror(base)
    np.random.seed(31)
    ht.merge_batch(snaps)
    check(ht, st, nxt)


def test_mixed_list_of_host_tables_and_snapshots(golden_match, golden_ingest):
    """Host tables and snapshots in one list, into the loaded base with a freed name."""
    files = im.fixture_files(golden_match)
    seeds = [im.SEED + r for r in range(5)]
    base = im.golden_base(golden_ingest, "add")
    st, _, nxt = statement(base, files, 5, seeds, 5)
    ws = rank_tables(files, 5, im.HASHBITS, im.DEPTH, im.MAXTIMEBITS, seeds)
    mixed = [ws[0], ws[1].export_device(), ws[2], ws[3].export_device(), ws[4].export_device()]
    ht = ref.mirror(base)
    np.random.seed(5)
    ht.merge_batch(mixed)
    check(ht, st, nxt)


def test_bench_geometry_every_bucket_overflows():
    """Two 2^20 x 100 per-rank tables, every slot filled, counts above depth: merged into an empty
    table the first fits (counts clipped to 100), the second overflows every bucket.  Snapshots and
    host tables give the same table, counts and np.random state."""
    mtb, depth, nids = 14, 100, 100_000
    parts = [synth_table(20, depth, nids, mtb, seed=s) for s in (3, 4)]

    def host(k):
        t, c, h = parts[k]
        ht = HashTable(hashbits=20, depth=1, maxtime=1 << mtb)
        ht.table, ht.counts, ht.hashesperid, ht.depth = t, c, h, depth
        ht.names = ["r%d/%d" % (k, i) for i in range(nids)]
        return ht
    dev = torch.device("cuda", _lib.context().device)
    snaps = [DeviceTable(torch.from_numpy(t.view(np.int32)).to(dev), torch.from_numpy(c).to(dev),
                         host(k).names, h, 20, depth, mtb) for k, (t, c, h) in enumerate(parts)]
    np.random.seed(21)
    a = HashTable(hashbits=20, depth=depth, maxtime=1 << mtb)
    assert a.merge_batch(snaps) == 1 << 20
    nxt = np.random.random()
    np.random.seed(21)
    b = HashTable(hashbits=20, depth=depth, maxtime=1 << mtb)
    assert b.merge_batch([host(0), host(1)]) == 1 << 20
    assert np.random.random() == nxt
    assert np.array_equal(a.counts, np.minimum(parts[0][1], depth) + parts[1][1])
    assert np.array_equal(a.table, b.table) and np.array_equal(a.counts, b.counts)
    assert a.names == b.names and np.array_equal(a.hashesperid, b.hashesperid)
    assert pruning_bound(a) == pruning_bound(b)


# ---- errors are raised before anything changes ---------------------------------------------
def _snapshot_of(hb, depth, mtb, names, live=()):
    dev = torch.device("cuda", _lib.context().device)
    t = torch.zeros((1 << hb, depth), dtype=torch.int32, device=dev)
    c = torch.zeros(1 << hb, dtype=torch.int32, device=dev)
    for b in live:
        c[b] = 1
        t[b, 0] = (1 << mtb) + 3
    return DeviceTable(t, c, names, np.ones(len(names), np.uint32), hb, depth, mtb)


def test_errors_leave_everything_unchanged(golden_match, golden_ingest):
    """ValueError for a negative incoming count, IndexError for a live bucket outside the table,
    OverflowError for an id that does not fit - from merge_batch on a list whose first entry is
    valid, and from afp_table_merge_device itself: table, counts, names, hashesperid, the device
    copy and np.random are unchanged."""
    files = im.fixture_files(golden_match)
    good = rank_tables(files[:4], 1, im.HASHBITS, im.DEPTH, im.MAXTIMEBITS, [3])[0]
    ht = ref.mirror(im.golden_base(golden_ingest, "add"))
    ht.merge_batch([good.export_device()])                       # the device copy now leads
    np.random.seed(4)
    before = (ht.table.copy(), ht.counts.copy(), list(ht.names), ht.hashesperid.copy(), np.random.get_state()[1].copy())
    neg = good.export_device()
    neg.counts[17] = -1
    outside = _snapshot_of(im.HASHBITS + 1, im.DEPTH, im.MAXTIMEBITS, ["o"], live=[(1 << im.HASHBITS) + 5])
    over = _snapshot_of(im.HASHBITS, im.DEPTH, im.MAXTIMEBITS, ["x%d" % i for i in range(1 << 20)], live=[2])
    ok = good.export_device()
    cases_ = [(ValueError, neg), (IndexError, outside), (OverflowError, over)]

    def unchanged():
        after = (ht.table, ht.counts, ht.names, ht.hashesperid, np.random.get_state()[1])
        assert all(np.array_equal(x, y) for x, y in zip(before[:2] + before[3:], after[:2] + after[3:]))
        assert before[2] == after[2]
    for exc, bad in cases_:
        with pytest.raises(exc):
            ht.merge_batch([ok, bad])
        unchanged()
    # the library's own checks, without merge_batch's
    ctx = ht._sync_device()
    st = np.random.get_state()
    for exc, bad in cases_[:2]:
        state = np.empty(625, np.uint32)
        state[:624], state[624] = st[1], st[2]
        keep = state.copy()
        with pytest.raises(exc):
            ctx.check(ctx.lib.afp_table_merge_device(ctx.h, bad.table.data_ptr(), bad.counts.data_ptr(), bad.hashbits,
                                                     bad.depth, len(ht.names), state.ctypes.data, None, None))
        assert np.array_equal(state, keep)
        t, c = device_state(ht)
        assert np.array_equal(t, before[0]) and np.array_equal(c, before[1])
    unchanged()


# ---- dist.ingest_sharded end to end, from PCM ------------------------------------------------
DIST_GEOM = (8, 6, 12)            # hashbits, depth, maxtimebits: overflows in the ranks and the merge
DIST_FILES = 7


def dist_files():
    """(name, PCM) of the files, in command-line order; file 2 is too short to give hashes."""
    out = []
    for i in range(DIST_FILES):
        pcm = synth_track(700 + i, 8.0) if i != 2 else np.zeros(100, np.int16)
        out.append(("pcm%d" % i, pcm))
    return out


def dist_base():
    """A loaded base with a freed slot (its id offset counts the None)."""
    st = ref.State(*DIST_GEOM)
    rng = random.Random(5)
    for k in range(3):
        rows = np.stack([np.arange(200) * 3, np.arange(200) * 37 + k], axis=1)
        ref.store(st, ref.name_to_id(st, "base%d" % k), rows, rng)
    ref.remove(st, 1)
    return st


def _worker(rank, world, port, backend, device, replicate, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["AFP_DEVICE"] = str(device)
    torch.cuda.set_device(device)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        files = dist_files()
        an = Analyzer(device=device)
        mine = afd.shard_indices(len(files), rank, world)
        base = dist_base() if not replicate else ref.State(*DIST_GEOM)       # `add` and `new`
        ht = ref.mirror(base)
        ht.device = device
        random.seed(im.SEED + rank)
        np.random.seed(99)
        lines = []
        counts = afd.ingest_sharded(an, ht, [files[i][0] for i in mine], [files[i][1] for i in mine],
                                    replicate=replicate, report=lines.extend)
        nxt = np.random.random()
        hashes = [(n, h) for (n, _), h in zip(files, an.fingerprint_batch([p for _, p in files]))]
        ok = counts == [len(hashes[i][1]) for i in mine] and len(hashes[2][1]) == 0
        st, want_lines, want_nxt = statement(base, hashes, world, [im.SEED + r for r in range(world)], 99)
        w0 = im.worker_table([hashes[i] for i in afd.shard_indices(len(files), 0, world)], *DIST_GEOM,
                             random.Random(im.SEED))
        ok = ok and (w0.counts > DIST_GEOM[1]).any()            # the root's own table overflowed
        if rank == 0:
            ok = ok and lines == want_lines and nxt == want_nxt and _same(ht, st)
            ok = ok and (st.counts > DIST_GEOM[1]).any()
        else:
            ok = ok and lines == [] and nxt == np.random.RandomState(99).random_sample()
            ok = ok and (_same(ht, st) if replicate else _same(ht, base))
        if rank == 0 or replicate:
            qan = Analyzer(device=device)
            qan.shifts = 4
            qs = qan.fingerprint_batch([files[i][1][8000:8000 + 40000] for i in (0, 3, 6)])
            m = Matcher()
            got = m.match_batch(ht, qs)
            want = m.match_batch(ref.mirror(st), qs)
            ok = ok and all(np.array_equal(x, y) for x, y in zip(got, want)) and sum(len(r) for r in got) > 0
        out.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def _failing_worker(rank, world, port, device, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["AFP_DEVICE"] = str(device)
    torch.cuda.set_device(device)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=60))
    try:
        ht = HashTable(hashbits=10, depth=6, maxtime=1 << 12, device=device)
        sig = [synth_track(800 + rank, 4.0)]
        if rank == 1:
            sig = [np.zeros((2, 100), np.int16)]                 # not a 1-D signal: ValueError
        try:
            afd.ingest_sharded(Analyzer(device=device), ht, ["f%d" % rank], sig)
            out.put((rank, "no error", ""))
        except Exception as e:
            out.put((rank, type(e).__name__, str(e)))
        out.put((rank, "names", len(ht.names)))
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn(target, args_of, nput):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, 2, port) + args_of(r) + (out,)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(600)
            assert p.exitcode == 0
        return sorted(out.get(timeout=10) for _ in range(nput))
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)


@pytest.mark.parametrize("replicate", [False, True])
def test_ingest_sharded_world2_gloo_on_one_gpu(replicate):
    assert _spawn(_worker, lambda r: ("gloo", 0, replicate), 2) == [(0, True), (1, True)]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL at world size 2 needs two GPUs")
@pytest.mark.parametrize("replicate", [False, True])
def test_ingest_sharded_world2_nccl(replicate):
    assert _spawn(_worker, lambda r: ("nccl", r, replicate), 2) == [(0, True), (1, True)]


def test_a_failed_ingest_raises_on_every_rank():
    """Rank 1's ingest raises ValueError (a 2-D signal): rank 1 re-raises it, rank 0 raises a
    RuntimeError naming rank 1; no table moved and the root's table is unchanged."""
    got = _spawn(_failing_worker, lambda r: (0,), 4)
    assert got[0][:2] == (0, "RuntimeError") and "rank 1" in got[0][2]
    assert got[1] == (0, "names", 0)
    assert got[2][:2] == (1, "ValueError") and got[3] == (1, "names", 0)


def test_ingest_sharded_world_size_one(golden_match):
    """Without a process group: one rank, its table merged into `ht` (not adopted)."""
    an = Analyzer()
    files = dist_files()[:3]
    base = dist_base()
    hashes = [(n, h) for (n, _), h in zip(files, an.fingerprint_batch([p for _, p in files]))]
    st, want_lines, nxt = statement(base, hashes, 1, [im.SEED], 3)
    ht = ref.mirror(base)
    random.seed(im.SEED)
    np.random.seed(3)
    lines = []
    afd.ingest_sharded(an, ht, [n for n, _ in files], [p for _, p in files], report=lines.extend)
    assert lines == want_lines
    check(ht, st, nxt)
