"""exact_count / find_time_range on a table sharded by track-id range, on the device.

The shards are visited one after another on one GPU, as the ranks of a sharded match would run
them: pass 1 ranks every shard (afp_match_options_shard_rank) and keeps its per-query largest
qtime, the maxima are reduced, pass 2 ranks again, finishes (afp_match_options_shard_finish) and
packs (afp_shard_pack), and the record buffers are stacked as an all-gather delivers them for
afp_shard_merge.  Merged rows must be the whole table's (Matcher.match_batch, sort=False) bit for
bit, every record must be the host statement's (tests/shard_options_reference.py) field by field,
and the device merge must be dist.merge_shard_batch."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

from audfprint_b200 import dist as afd
from audfprint_b200 import HashTable, Matcher
from tests import cases
from tests import shard_options_reference as sor
from tests.conftest import expand_table, GOLDEN
from tests.test_gpu_match_long import DEPTH, LONG_HITS, shows  # noqa: F401  (fixture)
from tests.test_gpu_match_options import MODES, _build, _golden, _matcher

pytestmark = pytest.mark.gpu


def _pack_queries(qs):
    qoff = np.zeros(len(qs) + 1, np.int64)
    qoff[1:] = np.cumsum([len(q) for q in qs])
    packed = np.ascontiguousarray(np.concatenate(qs)) if qs else np.zeros((0, 2), np.int32)
    return packed.astype(np.int32), qoff


def _rcap(nshards):
    return (1024 // nshards) & ~1                 # the merge holds nshards * row_cap <= 1024 rows


def _shards(ht, m, qs, nshards, rcap=None, host=True):
    """The two passes and the device merge.  Returns (rows, offsets) of the merge, or the
    exception it raised, and the per-shard records {"dev", "host", "qmax_local"}."""
    rcap = rcap or _rcap(nshards)
    packed, qoff = _pack_queries(qs)
    nq, sd = len(qs), max(int(m.search_depth), 1)
    nids = len(ht.hashesperid)
    opts = (m.exact_count, m.find_time_range, m.time_quantile)
    ht._touch()
    full_hits = [ht.get_hits(q) if len(q) else np.zeros((0, 4), np.int32) for q in qs] if host else None
    full_qmax = [sor.query_qmax(h) for h in full_hits] if host else \
        [sor.query_qmax(ht.get_hits(q)) if len(q) else 0 for q in qs]
    info = []
    qmaxes = []
    for s in range(nshards):                      # pass 1: rank, keep the shard's maxima
        lo, hi = afd.id_range(nids, s, nshards)
        ctx = ht.restrict_device_ids(lo, hi)
        qm = torch.empty(max(nq, 1), dtype=torch.int32, device="cuda")
        m._run(ctx, m._params(), packed, nq, qoff, opts, shard_qmax=qm.data_ptr())
        got = qm.cpu().numpy()[:nq]
        want = [sor.query_qmax(ht.get_hits(q)) if len(q) else 0 for q in qs]       # the shard's own hits
        assert got.tolist() == want, s
        qmaxes.append(qm)
        info.append({"qmax_local": got})
    qmax = torch.stack(qmaxes).amax(dim=0).contiguous()
    assert qmax.cpu().numpy()[:nq].tolist() == full_qmax
    bits = [sor.key_bits(int(v)) for v in qmax.cpu().numpy()[:nq]]
    rb = int(ctx.lib.afp_shard_record_bytes(sd, rcap))
    bufs, hosts = [], []
    for s in range(nshards):                      # pass 2: rank, finish with the reduced maxima, pack
        lo, hi = afd.id_range(nids, s, nshards)
        ctx = ht.restrict_device_ids(lo, hi)
        m._run(ctx, m._params(), packed, nq, qoff, opts, shard_qmax=qmaxes[s].data_ptr())
        ctx.check(ctx.lib.afp_match_options_shard_finish(ctx.h, C.c_void_p(qmax.data_ptr()), None))
        buf = torch.empty((max(nq, 1), rb), dtype=torch.uint8, device="cuda")
        ctx.check(ctx.lib.afp_shard_pack(ctx.h, rcap, buf.data_ptr()))
        dev = buf.cpu().numpy().view(afd.record_dtype(sd, rcap)).reshape(-1)[:nq]
        info[s]["dev"] = dev
        if host:
            recs = [sor.shard_options_record(h, ht.hashesperid, lo, hi, m.window, m.threshcount, m.search_depth,
                                             m.exact_count, m.find_time_range, m.time_quantile, b)
                    for h, b in zip(full_hits, bits)]
            hrec = sor.pack_shard(recs, sd, rcap)
            for f in ("hdr", "w", "id", "raw", "rows"):
                assert np.array_equal(dev[f], hrec[f]), (s, f)
            info[s]["host"] = hrec
            hosts.append(hrec)
        bufs.append(buf[:nq] if nq else buf[:0])
    ht._touch()
    gathered = torch.cat(bufs, dim=0).contiguous()
    total = C.c_int64(0)
    try:
        ctx.check(ctx.lib.afp_shard_merge(ctx.h, gathered.data_ptr() if nq else None, nshards, nq, sd, rcap,
                                          C.byref(total)))
    except (IndexError, ValueError) as e:
        if host:
            with pytest.raises(type(e)):
                afd.merge_shard_batch(np.stack(hosts), m.search_depth, rcap)
        return e, info
    rows = np.empty((int(total.value), 7), np.int32)
    roff = np.zeros(nq + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_match_rows(ctx.h, rows.ctypes.data if len(rows) else None, 1,
                                           roff.ctypes.data_as(C.POINTER(C.c_int64))))
    if host:
        want_rows, want_off = afd.merge_shard_batch(np.stack(hosts), m.search_depth, rcap)
        assert np.array_equal(roff, want_off) and np.array_equal(rows, want_rows)
    return (rows, roff), info


def _single(m, ht, qs):
    ht._touch()
    try:
        return m.match_batch(ht, qs, sort=False)
    except IndexError as e:
        return e


def _check(m, ht, qs, nshards, **kw):
    """The sharded result == the whole table's, errors included; returns (single rows, info)."""
    single = _single(m, ht, qs)
    got, info = _shards(ht, m, qs, nshards, **kw)
    key = (nshards, m.exact_count, m.find_time_range, m.window, m.threshcount, m.search_depth, m.time_quantile)
    if isinstance(single, IndexError):
        assert isinstance(got, IndexError), key
        return single, info
    assert not isinstance(got, Exception), (key, got)
    rows, roff = got
    for i, s in enumerate(single):
        assert np.array_equal(rows[roff[i]:roff[i + 1]], s), (key, i)
    return single, info


# ---- golden databases -----------------------------------------------------------------------
@pytest.mark.parametrize("db", ["db", "db2"])
@pytest.mark.parametrize("nshards", [2, 3, 5])
def test_golden_databases(golden_match, db, nshards):
    ht, qs, _ = _golden(golden_match, db)
    quants = (0.0, 0.02, 0.05, 0.5, 0.99)
    k = nrows = 0
    # a shard finishes every candidate it publishes, so at threshcount 2 one shard of db2 can produce
    # more rows for a query than nshards * row_cap <= 1024 holds; threshcount 2 runs on db only
    low = (1, 2, 10) if db == "db" else (1, 3, 10)
    for window, thresh, sdepth in ((1, 5, 100), (2, 3, 100), (0, 3, 4), (2, 5, 1), low):
        for exact, trange in MODES:
            m = _matcher(exact, trange, window, thresh, sdepth, quants[k % len(quants)])
            k += 1
            single, _ = _check(m, ht, qs, nshards)
            nrows += sum(len(r) for r in single)
    assert nrows > 200
    m = _matcher(True, True, 2, 5, 100, 0.05)     # the general kernel on every shard
    m.force_general_kernel = True
    _check(m, ht, qs, nshards)
    assert Matcher.last_general_count(ht) > 0


# ---- constructed edges --------------------------------------------------------------------------
def test_power_of_two_key_width_across_shards():
    """(a) Track 0's largest qtime is 2^11 (11 key bits: two of its three pairs collide); track 1,
    on the other shard, holds the query's real largest time (13 bits: no collision)."""
    k, h = 11, 900
    col = [(1 << k, h, 5), (0, h + 1, 5), (100, h + 2, 5)]
    other = [(5000, 950, 1), (5001, 951, 1)]
    ht, q = _build([col, other], extra={1: 10})
    assert [afd.id_range(2, s, 2) for s in range(2)] == [(0, 1), (1, 2)]
    for sdepth in (1, 100):
        m = _matcher(True, False, 0, 1, sdepth, 0.0)
        single, info = _check(m, ht, [q], 2)
        assert info[0]["qmax_local"][0] == 1 << k and sor.key_bits(1 << k) == k
        assert sor.key_bits(int(info[1]["qmax_local"][0])) == 13
        assert single[0][single[0][:, 0] == 0][0, 1] == 3


def test_raw_equal_to_threshcount_across_shards():
    """(b) Track 0 (raw == threshcount, weight 1) is global rank 0 < D = 1, which track 1 (raw >
    threshcount, on the other shard) makes; on its own shard n_above is 0."""
    a = [(10, 100, 5), (20, 101, 5), (30, 102, 5)]
    b = [(40, 110, 7), (50, 111, 7), (60, 112, 7), (70, 113, 7)]
    ht, q = _build([a, b], extra={1: 60})
    for trange in (False, True):
        m = _matcher(True, trange, 0, 3, 100, 0.0)
        single, info = _check(m, ht, [q], 2)
        assert any(r[0] == 0 and r[4] == 0 and r[1] == 3 for r in single[0])
        hdr = info[0]["dev"]["hdr"][0]
        assert hdr[0] == 0 and hdr[1] == 1 and hdr[2] >= 1         # n_above 0, yet its row is there


def test_time_range_row_behind_a_heavier_below_threshold_id():
    """(c) On shard 1, id 2 (raw == threshcount, weight 1) outranks id 3 (raw 6 > threshcount): id 3
    is local rank 1 = the shard's n_above, and global rank 1 < D = 3 thanks to ids 0 and 1."""
    def one_offset(h0, n, d):
        return [(10 * i + 1, h0 + i, d) for i in range(n)]
    specs = [one_offset(100, 5, 3), one_offset(200, 5, 4), one_offset(300, 3, 5), one_offset(400, 6, 6)]
    ht, q = _build(specs, extra={0: 100, 1: 120, 3: 30})
    assert [afd.id_range(4, s, 2) for s in range(2)] == [(0, 2), (2, 4)]
    for quant in (0.0, 0.02, 0.5):
        m = _matcher(False, True, 1, 3, 100, quant)
        single, info = _check(m, ht, [q], 2)
        assert [tuple(r[[0, 4]]) for r in single[0]] == [(3, 1), (0, 2)]
        hdr = info[1]["dev"]["hdr"][0]
        rows = info[1]["dev"]["rows"][0][:hdr[2]]
        assert hdr[0] == 1 and rows[0, 0] == 3 and rows[0, 4] == 1     # local rank 1 >= local n_above 1


def test_empty_shards_empty_query_and_one_shard_query():
    """(d) Five shards over two tracks: three shards hold no id; an empty query; a query with hits
    on one shard only."""
    a = [(10, 100, 5), (20, 101, 5), (30, 102, 5), (35, 103, 5)]
    b = [(40, 110, 7), (50, 111, 7), (60, 112, 7), (70, 113, 7)]
    ht, q = _build([a, b], extra={1: 60})
    assert sum(afd.id_range(2, s, 5)[0] == afd.id_range(2, s, 5)[1] for s in range(5)) == 3
    qa = np.array([(t, h) for t, h, _ in a], np.int32)
    qs = [q, np.zeros((0, 2), np.int32), qa]
    for exact, trange in MODES:
        m = _matcher(exact, trange, 1, 2, 100, 0.02)
        single, _ = _check(m, ht, qs, 5)
        assert len(single[0]) > 0 and len(single[1]) == 0 and set(single[2][:, 0]) == {0}


def test_long_queries_across_shards(shows):
    """(e) The long-query path (rows * depth >= 2^24) on every shard."""
    ht, qs = shows
    assert all(len(q) * DEPTH >= LONG_HITS for q in qs)
    for exact, trange in MODES:
        m = _matcher(exact, trange, 2, 8, 10, 0.05)
        single, _ = _check(m, ht, [qs[0], qs[1][:3000]], 2, host=False)
        assert sum(len(r) for r in single) > 0


# ---- errors -------------------------------------------------------------------------------------
@pytest.mark.parametrize("db", ["db", "db2"])
def test_quantile_one_raises_where_the_single_table_does(golden_match, db):
    ht, qs, _ = _golden(golden_match, db)
    for exact in (True, False):
        m = _matcher(exact, True, 1, 2, 100, 1.0)
        single, _ = _check(m, ht, qs, 3)
        assert isinstance(single, IndexError)
        packed, qoff = _pack_queries(qs)
        ht.restrict_device_ids(0, len(ht.hashesperid))          # one shard holding every id
        with pytest.raises(IndexError):
            afd.match_sharded_batch(m, ht, (packed, qoff), row_cap=512)
        ht._touch()


def test_quantile_failure_past_the_global_depth_does_not_raise():
    """Id 1 (raw == threshcount, weight 1) is the only rank < D = 1 and yields no row; id 2, on the
    same shard, has a row whose quantile read fails - at global rank 2 >= D (id 0 outranks it)."""
    def one_offset(h0, n, d):
        return [(10 * i + 1, h0 + i, d) for i in range(n)]
    ht, q = _build([one_offset(100, 2, 3), one_offset(300, 3, 5), one_offset(400, 6, 6)], extra={0: 10, 2: 60})
    m = _matcher(False, True, 1, 3, 100, 1.0)
    single, info = _check(m, ht, [q], 2)
    assert not isinstance(single, Exception) and len(single[0]) == 0
    assert info[1]["dev"]["hdr"][0, 3] == (1 + 1) << 1             # local rank 1 failed on shard 1


def test_row_capacity_overflow_names_the_count(golden_match):
    ht, qs, _ = _golden(golden_match, "db")
    m = _matcher(True, True, 2, 1, 100, 0.02)
    got, info = _shards(ht, m, qs, 2, rcap=2)
    assert isinstance(got, ValueError)
    need = max(int(i["dev"]["hdr"][:, 2].max()) for i in info)
    assert need > 2 and ("produced %d rows" % need) in str(got)
    packed, qoff = _pack_queries(qs)
    with pytest.raises(ValueError, match=r"produced \d+ rows for one query, row_cap is 2"):
        afd.match_sharded_batch(m, ht, (packed, qoff), row_cap=2)
    with pytest.raises(ValueError, match="even"):
        afd.match_sharded_batch(m, ht, (packed, qoff), row_cap=3)


# ---- world size 1 --------------------------------------------------------------------------------
def test_world_size_one_equals_match_batch(golden_match):
    ht, qs, _ = _golden(golden_match, "db2")
    packed, qoff = _pack_queries(qs)
    for exact, trange in MODES + ((False, False),):
        for window, thresh, sdepth, quant in ((2, 5, 100, 0.02), (1, 3, 30, 0.5)):
            m = _matcher(exact, trange, window, thresh, sdepth, quant)
            ht._touch()
            rows, off = afd.match_sharded_batch(m, ht, (packed, qoff), row_cap=1024)
            single = m.match_batch(ht, qs, sort=False)
            for i, s in enumerate(single):
                assert np.array_equal(rows[off[i]:off[i + 1]], s), (exact, trange, i)
            per_query = afd.match_sharded(m, ht, qs, row_cap=1024)
            for p, s in zip(per_query, m.match_batch(ht, qs)):
                assert np.array_equal(p, s)


# ---- the real collectives: two processes ----------------------------------------------------------
def _worker(rank, world, port, backend, device, out):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["AFP_DEVICE"] = str(device)
    torch.cuda.set_device(device)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        gm = np.load(os.path.join(GOLDEN, "match.npz"))
        table, counts, hashbits, depth, mtb, hpi = expand_table(gm, "db")
        ht = HashTable(hashbits=hashbits, depth=depth, maxtime=1 << mtb)
        ht.table, ht.counts, ht.hashesperid = table, counts, hpi
        ht.device = device
        qs = [gm["q%d_%s/q" % (j, tag)] for j in range(cases.DB_QUERIES) for tag in ("clean", "noisy")]
        packed, qoff = _pack_queries(qs)
        ok = True
        for exact, trange in MODES:
            m = _matcher(exact, trange, 2, 2, 100, 0.05)
            single = m.match_batch(ht, qs, sort=False)
            ht.restrict_device_ids(*afd.id_range(len(hpi), rank, world))
            rows, off = afd.match_sharded_batch(m, ht, (packed, qoff), row_cap=512)
            ht._touch()
            ok = ok and all(np.array_equal(rows[off[i]:off[i + 1]], s) for i, s in enumerate(single))
        out.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn_world2(backend, devices):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, devices[r], out)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(600)
            assert p.exitcode == 0
        assert sorted(out.get(timeout=10) for _ in procs) == [(0, True), (1, True)]
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)


def test_world2_gloo_on_one_gpu():
    _spawn_world2("gloo", (0, 0))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL at world size 2 needs two GPUs")
def test_world2_nccl():
    _spawn_world2("nccl", (0, 1))
