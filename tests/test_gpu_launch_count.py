"""afp_launch_count of every entry point on small fixed inputs.

The count is public (bench.py reports it as gpu_launches), so each entry point's delta is pinned
here: a change that adds, drops or miscounts a launch shows up as a changed number.  Every case runs
on a context of its own, so that no state of an earlier case (a cached tile table, say) moves it."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from audfprint_b200 import _lib
from audfprint_b200 import analyzer as an_mod
from audfprint_b200.analyzer import Analyzer
from audfprint_b200.flac import parse
from audfprint_b200.matcher import timebits_breaks
from audfprint_b200.synth import synth_track
from tests import flac_writer

pytestmark = pytest.mark.gpu

I64 = C.POINTER(C.c_int64)

EXPECTED = {
    "fingerprint_device_pcm": (8, 7),        # the second batch of the same layout keeps its tile table
    "fingerprint_host_pcm": (8,),
    "fingerprint_chunked_host_pcm": (8,),
    "fetch_peaks": (6,),                     # two calls: the offsets, then the rows
    "from_peaks": (4, 5),                    # host rows, device rows
    "from_logs": (4,),
    "landmarks": (5,),
    "stft_mag_sgram": (2, 4),
    "pcm_frontend": (1, 1),
    "flac": (2, 1),
    "store_overflow_slots_patches": (12, 2, 1),
    "remove_retrieve": (4, 9),
    "merge_host_device": (7, 7),
    "get_hits": (3,),
    "match_fast_general_long": (6, 5, 14),   # the long path's candidate branch makes 3 launches and a scan
    "options_exact_trange": (23, 23),
    "shard_rank_finish_pack_merge": (7, 18, 1, 4),
}


def _ctx():
    ctx = _lib.Context(0)
    an = Analyzer()
    p = _lib.AnalyzerParams(an._a_dec(), an_mod.HPF_POLE ** (1 / an_mod.OVERSAMP), int(an.maxpksperframe),
                            int(an.maxpairsperpeak), int(an.targetdf), int(an.mindt), int(an.targetdt), 1, 0)
    ctx.check(ctx.lib.afp_set_analyzer(ctx.h, C.byref(p), None, None, float(an.f_sd)))
    return ctx


@pytest.fixture
def ctx():
    c = _ctx()
    yield c
    c.close()


def _delta(ctx, fn):
    n0 = ctx.launch_count()
    fn()
    ctx.sync()
    return ctx.launch_count() - n0


def _check(name, got):
    assert tuple(got) == EXPECTED[name], (name, tuple(got))


def _pcm(nfiles=3, seconds=4.0):
    tracks = [synth_track(700 + i, seconds) for i in range(nfiles)]
    off = np.zeros(nfiles + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in tracks])
    return np.ascontiguousarray(np.concatenate(tracks)), off


def _fingerprint(ctx, pcm, off, on_host):
    total = C.c_int64(0)
    ptr = pcm.ctypes.data if on_host else pcm.data_ptr()
    ctx.check(ctx.lib.afp_fingerprint_batch(ctx.h, ptr, 0, 1 if on_host else 0, len(off) - 1,
                                            off.ctypes.data_as(I64), None, C.byref(total)))
    return total.value


def _hashes(ctx, nfiles):
    off = np.zeros(nfiles + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, off.ctypes.data_as(I64)))
    rows = np.zeros((max(int(off[-1]), 1), 2), np.int32)
    ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, rows.ctypes.data, 1, None))
    return rows[:off[-1]], off


def _peaks(ctx, nfiles):
    off = np.zeros(nfiles + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, 0, None, 1, off.ctypes.data_as(I64)))
    rows = np.zeros((max(int(off[-1]), 1), 2), np.int32)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, 0, rows.ctypes.data, 1, None))
    return rows[:off[-1]], off


def test_fingerprint_device_pcm(ctx):
    pcm, off = _pcm()
    dev = torch.from_numpy(pcm).cuda()
    torch.cuda.synchronize()
    got = [_delta(ctx, lambda: _fingerprint(ctx, dev, off, False)) for _ in range(2)]
    _check("fingerprint_device_pcm", got)


def test_fingerprint_host_pcm(ctx):
    pcm, off = _pcm()
    _check("fingerprint_host_pcm", [_delta(ctx, lambda: _fingerprint(ctx, pcm, off, True))])


def test_fingerprint_chunked_host_pcm(ctx):
    # 64 MB or more of host PCM over several files takes the chunked copy / compute pipeline
    rng = np.random.default_rng(3)
    n = 9_000_000
    pcm = rng.integers(-3000, 3000, 4 * n, dtype=np.int16)
    off = np.arange(5, dtype=np.int64) * n
    _check("fingerprint_chunked_host_pcm", [_delta(ctx, lambda: _fingerprint(ctx, pcm, off, True))])


def test_fetch_peaks_and_from_peaks(ctx):
    pcm, off = _pcm()
    _fingerprint(ctx, pcm, off, True)
    ctx.sync()
    got = []
    box = {}
    got.append(_delta(ctx, lambda: box.setdefault("pk", _peaks(ctx, 3))))
    _check("fetch_peaks", got)
    rows, poff = box["pk"]
    status = np.zeros(3, np.int32)
    total = C.c_int64(0)

    def from_peaks(ptr, on_host):
        ctx.check(ctx.lib.afp_fingerprint_from_peaks(ctx.h, ptr, on_host, 3, poff.ctypes.data_as(I64),
                                                     status.ctypes.data, C.byref(total)))

    drows = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    got = [_delta(ctx, lambda: from_peaks(rows.ctypes.data, 1)), _delta(ctx, lambda: from_peaks(drows.data_ptr(), 0))]
    _check("from_peaks", got)


def test_from_logs(ctx):
    rng = np.random.default_rng(5)
    frames = np.array([120, 90], np.int32)
    logs = rng.normal(-3.0, 2.0, (int(frames.sum()), 256))
    stats = np.array([[-12.0, -3.0, 0.0], [-12.0, -3.0, 0.0]])
    total = C.c_int64(0)
    _check("from_logs", [_delta(ctx, lambda: ctx.check(ctx.lib.afp_fingerprint_from_logs(
        ctx.h, logs.ctypes.data, 1, 2, frames.ctypes.data, stats.ctypes.data, C.byref(total))))])


def test_landmarks(ctx):
    pcm, off = _pcm(1)
    _fingerprint(ctx, pcm, off, True)
    rows, _ = _peaks(ctx, 1)
    nlm = C.c_int64(0)
    _check("landmarks", [_delta(ctx, lambda: ctx.check(ctx.lib.afp_landmarks_from_peaks(
        ctx.h, rows.ctypes.data, len(rows), 1, C.byref(nlm))))])


def test_stft_mag_and_sgram(ctx):
    pcm, _ = _pcm(1, 2.0)
    n = len(pcm)
    T = 1 + n // 256
    mag = np.zeros((T, 257))
    sg = np.zeros((T, 256))
    got = [_delta(ctx, lambda: ctx.check(ctx.lib.afp_stft_mag(ctx.h, pcm.ctypes.data, 0, 1, n, mag.ctypes.data, 1))),
           _delta(ctx, lambda: ctx.check(ctx.lib.afp_sgram(ctx.h, pcm.ctypes.data, 0, 1, n, sg.ctypes.data, 1)))]
    _check("stft_mag_sgram", got)


def test_pcm_frontends(ctx):
    rng = np.random.default_rng(7)
    raw = rng.integers(-2000, 2000, (4000, 2), dtype=np.int16)
    taps = np.hanning(41)
    out = np.zeros(4000, np.float32)
    nout = C.c_int64(0)
    single = lambda: ctx.check(ctx.lib.afp_pcm_frontend(ctx.h, raw.ctypes.data, 1, 4000, 2, 1, 4, taps.ctypes.data,
                                                          41, out.ctypes.data, 1, C.byref(nout)))
    pcm = np.ascontiguousarray(np.concatenate([raw.ravel(), raw.ravel()]))
    poff = np.array([0, raw.size], np.int64)
    nfr = np.array([4000, 4000], np.int64)
    ch = np.array([2, 2], np.int32)
    up = np.array([1, 1], np.int32)
    down = np.array([4, 1], np.int32)
    rates = np.array([1, 4], np.int32)
    toff = np.array([0, 41], np.int64)
    dout = torch.zeros(9000, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    batch = lambda: ctx.check(ctx.lib.afp_pcm_frontend_batch(
        ctx.h, pcm.ctypes.data, 1, pcm.size, 2, poff.ctypes.data_as(I64), nfr.ctypes.data_as(I64), ch.ctypes.data,
        up.ctypes.data, down.ctypes.data, 1, rates.ctypes.data, toff.ctypes.data_as(I64), taps.ctypes.data,
        dout.data_ptr(), dout.numel(), None, None))
    _check("pcm_frontend", [_delta(ctx, single), _delta(ctx, batch)])


def test_flac_locate_and_decode(ctx):
    rng = np.random.default_rng(11)
    streams = [parse(flac_writer.stream(rng.integers(-3000, 3000, (n, 2)), 16, 44100)[0]) for n in (9000, 5000)]
    packed = np.ascontiguousarray(np.concatenate([s.frames for s in streams]))
    tab = (_lib.FlacStream * 2)()
    o = 0
    for k, s in enumerate(streams):
        tab[k] = _lib.FlacStream(o, len(s.frames), s.sample_rate, s.channels, s.bits_per_sample, s.max_blocksize)
        o += len(s.frames)
    ns = np.zeros(2, np.int64)
    st = np.zeros(2, np.int32)
    out = torch.zeros(2 * 14000, dtype=torch.int16, device="cuda")
    oo = np.array([0, 18000], np.int64)
    torch.cuda.synchronize()
    got = [_delta(ctx, lambda: ctx.check(ctx.lib.afp_flac_locate_batch(ctx.h, packed.ctypes.data, 1, o, 2, tab,
                                                                         ns.ctypes.data_as(I64), st.ctypes.data))),
           _delta(ctx, lambda: ctx.check(ctx.lib.afp_flac_decode_batch(ctx.h, out.data_ptr(), out.numel(),
                                                                         oo.ctypes.data_as(I64), st.ctypes.data)))]
    assert ns.tolist() == [9000, 5000]
    _check("flac", got)


def _small_table(ctx, hashbits=10, depth=8, mtb=16, nfiles=4, per=4000, seed=13):
    """afp_table_create, then one store of random rows that overflows many buckets."""
    ctx.check(ctx.lib.afp_table_create(ctx.h, hashbits, depth, mtb))
    rng = np.random.default_rng(seed)
    rows = np.stack([rng.integers(0, 1000, nfiles * per), rng.integers(0, 1 << hashbits, nfiles * per)], 1)
    rows = np.ascontiguousarray(rows.astype(np.int32))
    roff = np.arange(nfiles + 1, dtype=np.int64) * per
    ids = np.arange(nfiles, dtype=np.int64)
    novf = C.c_int64(0)
    store = lambda: ctx.check(ctx.lib.afp_table_store_batch(ctx.h, rows.ctypes.data, 1, roff.ctypes.data_as(I64),
                                                            nfiles, ids.ctypes.data_as(I64), C.byref(novf)))
    return store, novf, rows, roff


def test_store_with_overflow_then_slots_and_patches(ctx):
    store, novf, _, _ = _small_table(ctx)
    got = [_delta(ctx, store)]
    n = novf.value
    assert n > 0
    cnt = np.zeros(n, np.int32)
    ctx.check(ctx.lib.afp_table_fetch_overflow_counts(ctx.h, cnt.ctypes.data))
    state = np.array(random.Random(1).getstate()[1], dtype=np.uint32)
    slot = np.empty(n, np.int32)
    ctx.check(ctx.lib.afp_mt_randint_replay(state.ctypes.data, cnt.ctypes.data, n, slot.ctypes.data))
    got.append(_delta(ctx, lambda: ctx.check(ctx.lib.afp_table_apply_slots(ctx.h, slot.ctypes.data, n))))
    b = np.array([1, 2, 3], np.uint32)
    s = np.array([0, 1, 2], np.int32)
    v = np.array([7 << 16, 8 << 16, 9 << 16], np.uint32)
    got.append(_delta(ctx, lambda: ctx.check(ctx.lib.afp_table_apply_patches(ctx.h, b.ctypes.data, s.ctypes.data,
                                                                             v.ctypes.data, 3))))
    _check("store_overflow_slots_patches", got)


def test_remove_and_retrieve_repeated_ids(ctx):
    store, _, _, _ = _small_table(ctx, hashbits=12, depth=16, nfiles=6, per=2000)
    store()
    hpi = np.full(6, 2000, np.uint32)
    ctx.check(ctx.lib.afp_table_set_hashesperid(ctx.h, hpi.ctypes.data, 6))
    rm = np.array([1, 4], np.int64)
    removed = np.zeros(2, np.int64)
    rt = np.array([2, 0, 2, 5, 0], np.int64)
    total = C.c_int64(0)
    got = [_delta(ctx, lambda: ctx.check(ctx.lib.afp_table_remove_ids(ctx.h, rm.ctypes.data_as(I64), 2,
                                                                      removed.ctypes.data_as(I64)))),
           _delta(ctx, lambda: ctx.check(ctx.lib.afp_table_retrieve_ids(ctx.h, rt.ctypes.data_as(I64), 5,
                                                                        C.byref(total))))]
    assert total.value > 0
    _check("remove_retrieve", got)


def test_merge_host_and_device(ctx):
    store, _, _, _ = _small_table(ctx)
    store()
    rng = np.random.default_rng(17)
    hb, depth = 10, 8
    counts = rng.integers(0, 12, 1 << hb).astype(np.int32)
    table = ((rng.integers(1, 5, ((1 << hb), depth)) << 16) | rng.integers(0, 1000, ((1 << hb), depth)))
    table = np.ascontiguousarray(table.astype(np.uint32))
    state = np.zeros(625, np.uint32)
    state[:624] = np.random.RandomState(0).get_state()[1]
    state[624] = 624
    novf = C.c_int64(0)
    host = lambda: ctx.check(ctx.lib.afp_table_merge(ctx.h, table.ctypes.data, counts.ctypes.data, hb, depth, 8,
                                                     state.ctypes.data, C.byref(novf), None))
    dt, dc = torch.from_numpy(table.view(np.int32)).cuda(), torch.from_numpy(counts).cuda()
    torch.cuda.synchronize()
    dev = lambda: ctx.check(ctx.lib.afp_table_merge_device(ctx.h, dt.data_ptr(), dc.data_ptr(), hb, depth, 8,
                                                           state.ctypes.data, C.byref(novf), None))
    got = [_delta(ctx, host)]
    assert novf.value > 0
    got.append(_delta(ctx, dev))
    _check("merge_host_device", got)


class _Tracks:
    """Six tracks fingerprinted and stored on a table of depth 256, and query rows cut from them."""

    def __init__(self, ctx):
        pcm, off = _pcm(6, 6.0)
        _fingerprint(ctx, pcm, off, True)
        rows, roff = _hashes(ctx, 6)
        self.rows, self.roff = rows, roff
        ctx.check(ctx.lib.afp_table_create(ctx.h, 16, 256, 16))
        ids = np.arange(6, dtype=np.int64)
        novf = C.c_int64(0)
        ctx.check(ctx.lib.afp_table_store_batch(ctx.h, rows.ctypes.data, 1, roff.ctypes.data_as(I64), 6,
                                                ids.ctypes.data_as(I64), C.byref(novf)))
        hpi = np.diff(roff).astype(np.uint32)
        ctx.check(ctx.lib.afp_table_set_hashesperid(ctx.h, hpi.ctypes.data, 6))
        # queries: a stretch of tracks 1 and 4; the long one repeats every stored row until
        # rows * depth reaches 2^24
        q = [rows[roff[1]:roff[1] + 600], rows[roff[4] + 100:roff[4] + 700]]
        self.q, self.qoff = _lib.pack_rows(q)
        reps = -(-(1 << 16) // len(rows))
        self.lq, self.lqoff = _lib.pack_rows([np.tile(rows, (reps, 1))])


def _params(**kw):
    p = _lib.MatcherParams(1, 5, 100, 100, 0, 0, 0)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_get_hits(ctx):
    t = _Tracks(ctx)
    nh = C.c_int64(0)
    _check("get_hits", [_delta(ctx, lambda: ctx.check(ctx.lib.afp_get_hits(ctx.h, t.q.ctypes.data, len(t.q), 1,
                                                                           C.byref(nh))))])


def test_match_fast_general_long(ctx):
    t = _Tracks(ctx)
    total = C.c_int64(0)

    def match(q, qoff, p):
        ctx.check(ctx.lib.afp_match_batch(ctx.h, q.ctypes.data, 1, len(qoff) - 1, qoff.ctypes.data_as(I64),
                                          C.byref(p), C.byref(total)))

    got = [_delta(ctx, lambda: match(t.q, t.qoff, _params())),
           _delta(ctx, lambda: match(t.q, t.qoff, _params(force_general=1)))]
    got.append(_delta(ctx, lambda: match(t.lq, t.lqoff, _params())))
    assert total.value > 0
    _check("match_fast_general_long", got)


def test_options_exact_count_and_time_range(ctx):
    t = _Tracks(ctx)
    total = C.c_int64(0)
    br = timebits_breaks()

    def opts(exact, trange):
        ctx.check(ctx.lib.afp_match_options_batch(ctx.h, t.q.ctypes.data, 1, 2, t.qoff.ctypes.data_as(I64),
                                                  C.byref(_params()), exact, trange, 0.02,
                                                  br.ctypes.data_as(I64), C.byref(total)))

    got = [_delta(ctx, lambda: opts(1, 0))]
    assert total.value > 0
    got.append(_delta(ctx, lambda: opts(0, 1)))
    _check("options_exact_trange", got)


def test_shard_rank_finish_pack_merge(ctx):
    t = _Tracks(ctx)
    ranked = C.c_int64(0)
    total = C.c_int64(0)
    br = timebits_breaks()
    p = _params()
    qmax = torch.zeros(2, dtype=torch.int32, device="cuda")
    rb = int(ctx.lib.afp_shard_record_bytes(100, 256))
    rec = torch.zeros(2 * rb, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    got = [_delta(ctx, lambda: ctx.check(ctx.lib.afp_match_options_shard_rank(
               ctx.h, t.q.ctypes.data, 1, 2, t.qoff.ctypes.data_as(I64), C.byref(p), 1, 1, 0.02,
               br.ctypes.data_as(I64), C.c_void_p(qmax.data_ptr()), C.byref(ranked)))),
           _delta(ctx, lambda: ctx.check(ctx.lib.afp_match_options_shard_finish(ctx.h, C.c_void_p(qmax.data_ptr()),
                                                                                C.byref(total)))),
           _delta(ctx, lambda: ctx.check(ctx.lib.afp_shard_pack(ctx.h, 256, C.c_void_p(rec.data_ptr())))),
           _delta(ctx, lambda: ctx.check(ctx.lib.afp_shard_merge(ctx.h, C.c_void_p(rec.data_ptr()), 1, 2, 100, 256,
                                                                 C.byref(total))))]
    assert total.value > 0
    _check("shard_rank_finish_pack_merge", got)
