"""Stream order at the boundary between torch and the library.

The library runs its calls on the context's stream: its own non-blocking stream, or the stream
Context.set_stream names.  Torch runs on its current stream.  Every Python entry point that hands
torch CUDA memory to the library must order the two (Context.after_torch).  Each case here makes a
missing wait certain, then checks the result against the same call made from host memory, which the
rest of the suite pins to the reference:

- read after write: the buffer holds a valid input A and is complete; then, on torch's current
  stream, a sleep of SLEEP_MS and a write of another valid input B.  The call is made at once, while
  an event recorded after B's write is still pending.  A missing wait reads A: the case fails with
  "got input A's result", never on garbage, since every offset and count stays valid.
- write after read: a block is freed while a pending clone() (behind the sleep) still reads it, and
  the entry point's own allocation reuses that block (same data_ptr; otherwise the case fails,
  saying it tested nothing).  A missing wait lets the library's write overtake the clone.
- lifetime: a buffer the package allocates and drops while a call that returned without
  synchronising still reads it (Analyzer._fingerprint_pcm); the library's work is held behind a
  sleep, and a same-sized tensor is allocated and written right after.  The hashes must not change.
- afp_set_stream: a fetch=False fingerprint queued behind a sleep on the outgoing stream, a switch,
  a second batch of the same layout on the new stream: the workspace must end with the second one.

Each case runs once, in three stream modes: the library's own stream ("own"), the library on torch's
current stream ("current": Context.set_stream(torch.cuda.current_stream().cuda_stream)) and the
library on a side stream ("side").  Torch's current stream is a fresh non-default stream throughout,
so that the caching allocator's free blocks on it are the case's own.  (Torch's default stream has
the handle 0, which set_stream reads as "the library's own stream": bench.py, which passes the
current stream's handle from the default stream, runs in the "own" arrangement.)"""
import contextlib

import numpy as np
import pytest
import torch

from audfprint_b200 import Analyzer, HashTable, Matcher, _lib
from audfprint_b200 import analyzer as an_mod
from audfprint_b200 import dist as afd
from audfprint_b200.hash_table import DeviceTable
from audfprint_b200.synth import synth_track, pcm_to_float

pytestmark = pytest.mark.gpu

SLEEP_MS = 50                 # long against a host call (~0.1 ms), short against the suite
SR = 11025
GEOM = dict(hashbits=10, depth=2, maxtime=1 << 14)
MODES = ["own", "current", "side"]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def ctx(dev):
    return _lib.context(dev.index)


@pytest.fixture(scope="module")
def cycles(dev):
    """Device clock cycles of SLEEP_MS, measured with events around one torch.cuda._sleep."""
    n = 10 ** 7
    torch.cuda._sleep(n // 10)              # first launch out of the measurement
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(n)
    e1.record()
    torch.cuda.synchronize(dev)
    return int(n / e0.elapsed_time(e1) * SLEEP_MS)


@pytest.fixture(params=MODES)
def mode(request, ctx, dev):
    """Torch's current stream is a fresh stream; the context runs on its own stream, on torch's
    current stream or on a side stream.  The context is process-wide: its own stream comes back on
    teardown."""
    torch.cuda.synchronize(dev)
    cur = torch.cuda.Stream(dev)
    try:
        with torch.cuda.stream(cur):
            if request.param == "current":
                ctx.set_stream(cur.cuda_stream)
            elif request.param == "side":
                ctx.set_stream(torch.cuda.Stream(dev).cuda_stream)
            else:
                ctx.set_stream(None)
            yield request.param
    finally:
        torch.cuda.synchronize(dev)
        ctx.set_stream(None)


@pytest.fixture(scope="module")
def an():
    return Analyzer(device=0)


@pytest.fixture(scope="module")
def tracks():
    """Six 4 s tracks of equal length: inputs A and B of a case have the same layout."""
    return [synth_track(500 + i, 4.0) for i in range(6)]


# ---- helpers ----------------------------------------------------------------------------------
def _same(x, y):
    if isinstance(x, (list, tuple)):
        return isinstance(y, (list, tuple)) and len(x) == len(y) and all(_same(a, b) for a, b in zip(x, y))
    if isinstance(x, torch.Tensor):
        x = x.cpu().numpy()
    if isinstance(y, torch.Tensor):
        y = y.cpu().numpy()
    x, y = np.asarray(x), np.asarray(y)
    return x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()


def _check(got, ref_a, ref_b, what, stale="the library read the buffer before torch's write of B landed"):
    assert not _same(ref_a, ref_b), "%s: inputs A and B give the same result: the case cannot tell them apart" % what
    if _same(got, ref_a):
        pytest.fail("%s: got input A's result: %s" % (what, stale))
    assert _same(got, ref_b), "%s: the result is neither input A's nor input B's" % what


def _write_b_behind_sleep(cycles, write):
    """Sleep on torch's current stream, then `write()` there; returns the event after the write,
    checked to be pending."""
    torch.cuda._sleep(cycles)
    write()
    ev = torch.cuda.Event()
    ev.record()
    assert not ev.query(), "B's write finished before the call: the case tested nothing"
    return ev


@contextlib.contextmanager
def _freed_block_under_pending_read(cycles, like, monkeypatch):
    """A block the size of `like`, freed while a clone() behind a sleep still reads it.  Yields
    `allocs`, which collects the data_ptr of every torch.empty / torch.zeros the body makes; on exit
    the body must have reused the block, and the clone must have read the block's old content."""
    dev = like.device
    torch.cuda.synchronize(dev)
    torch.cuda.empty_cache()
    lo = torch.empty_like(like)               # neighbours: the freed block merges with nothing
    x = torch.empty_like(like)
    hi = torch.empty_like(like)
    x.view(torch.uint8).fill_(0x5a)
    old = x.clone()
    torch.cuda.synchronize(dev)
    torch.cuda._sleep(cycles)
    seen = x.clone()                          # pending behind the sleep
    ptr = x.data_ptr()
    del x
    allocs = []

    def recording(fn):
        def call(*a, **k):
            t = fn(*a, **k)
            allocs.append(t.data_ptr())
            return t
        return call
    with monkeypatch.context() as mp:
        mp.setattr(torch, "empty", recording(torch.empty))
        mp.setattr(torch, "zeros", recording(torch.zeros))
        yield allocs
    torch.cuda.synchronize(dev)
    assert ptr in allocs, "the entry point's allocation did not reuse the freed block: the case tested nothing"
    assert torch.equal(seen, old), "the library's write into a reused block overtook torch's pending read of it"
    del lo, hi


def _hashes(an, pcm_list):
    packed, starts, lens = an._pack(pcm_list)
    rows, roff = an.fingerprint_packed(packed, starts, sample_lengths=lens)
    return [rows[roff[i]:roff[i + 1]] for i in range(len(pcm_list))]


# ---- read after write ---------------------------------------------------------------------------
@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("dtype", ["int16", "float32"])
def test_fingerprint_packed_reads_after_torch_writes(mode, an, tracks, dev, cycles, where, dtype):
    conv = (lambda x: x) if dtype == "int16" else pcm_to_float
    a = np.concatenate([conv(t) for t in tracks[0:2]])
    b = np.concatenate([conv(t) for t in tracks[2:4]])
    off = np.array([0, len(tracks[0]), 2 * len(tracks[0])], np.int64)
    ref_a, ref_b = an.fingerprint_packed(a, off), an.fingerprint_packed(b, off)
    buf = torch.from_numpy(a).to(dev) if where == "device" else torch.from_numpy(a).pin_memory()
    src = torch.from_numpy(b).to(dev)
    torch.cuda.synchronize(dev)
    _write_b_behind_sleep(cycles, lambda: buf.copy_(src, non_blocking=True))
    got = an.fingerprint_packed(buf, off)
    _check(got, ref_a, ref_b, "fingerprint_packed(%s %s)" % (where, dtype))


@pytest.fixture(scope="module")
def match_setup(an, tracks):
    """A table of the six tracks and two two-query batches of equal layout: A from tracks 0-1,
    B from tracks 2-3 (each query a track's own hashes, cut to one length)."""
    hs = _hashes(an, tracks)
    ht = HashTable(hashbits=16, depth=20, maxtime=1 << 14, device=0)
    for i, h in enumerate(hs):
        ht.store("t%d" % i, h)
    n = min(len(h) for h in hs[:4])
    qa = np.ascontiguousarray(np.concatenate([hs[0][:n], hs[1][:n]]))
    qb = np.ascontiguousarray(np.concatenate([hs[2][:n], hs[3][:n]]))
    return ht, qa, qb, np.array([0, n, 2 * n], np.int64)


def _matcher(options):
    m = Matcher()
    m.exact_count = options == "exact_count"
    m.find_time_range = options == "find_time_range"
    return m


def _raw_device_rows(match_setup, dev, cycles, call, what):
    ht, qa, qb, qoff = match_setup
    ref_a, ref_b = call(qa), call(qb)
    buf = torch.from_numpy(qa).to(dev)
    src = torch.from_numpy(qb).to(dev)
    ht._sync_device()                     # the table upload is not part of the case
    torch.cuda.synchronize(dev)
    _write_b_behind_sleep(cycles, lambda: buf.copy_(src))
    _check(call(buf), ref_a, ref_b, what)


@pytest.mark.parametrize("options", ["plain", "exact_count", "find_time_range"])
def test_match_batch_reads_device_rows_after_torch_writes(mode, match_setup, dev, cycles, options):
    ht, _, _, qoff = match_setup
    m = _matcher(options)
    _raw_device_rows(match_setup, dev, cycles, lambda q: m.match_batch(ht, (q, qoff)), "match_batch(%s)" % options)


def test_match_batch_shard_packed_reads_device_rows_after_torch_writes(mode, match_setup, dev, cycles):
    ht, _, _, qoff = match_setup
    m = Matcher()
    _raw_device_rows(match_setup, dev, cycles, lambda q: m.match_batch_shard_packed(ht, (q, qoff)),
                     "match_batch_shard_packed")


@pytest.mark.parametrize("options", ["plain", "exact_count"])
def test_match_sharded_batch_reads_device_rows_after_torch_writes(mode, match_setup, dev, cycles, options):
    ht, _, _, qoff = match_setup
    m = _matcher(options)
    _raw_device_rows(match_setup, dev, cycles, lambda q: afd.match_sharded_batch(m, ht, (q, qoff), row_cap=64),
                     "dist.match_sharded_batch(%s)" % options)


@pytest.fixture(scope="module")
def tables(an, tracks):
    """Host tables A (tracks 0-2) and B (tracks 3-5) of one small geometry, buckets overflowing."""
    hs = _hashes(an, tracks)
    out = []
    for part in (range(0, 3), range(3, 6)):
        t = HashTable(device=0, **GEOM)
        for i in part:
            t.store("t%d" % i, hs[i])
        out.append(t)
    assert (out[1].counts > out[1].depth).any()
    return out


def _snapshot_rewritten(tables, dev, cycles):
    """DeviceTable tensors holding table A, then rewritten with table B behind a sleep."""
    ta, tb = tables
    tab = torch.from_numpy(ta.table.view(np.int32)).to(dev)
    cnt = torch.from_numpy(ta.counts).to(dev)
    tab_b = torch.from_numpy(tb.table.view(np.int32)).to(dev)
    cnt_b = torch.from_numpy(tb.counts).to(dev)
    torch.cuda.synchronize(dev)
    _write_b_behind_sleep(cycles, lambda: (tab.copy_(tab_b), cnt.copy_(cnt_b)))
    return DeviceTable(tab, cnt, tb.names, tb.hashesperid, tb.hashbits, tb.depth, tb.maxtimebits)


def test_merge_batch_reads_snapshot_after_torch_writes(mode, tables, dev, cycles):
    ref = {}
    for k, t in zip("ab", tables):
        h = HashTable(device=0, **GEOM)
        np.random.seed(7)
        h.merge(t)
        ref[k] = (h.table.copy(), h.counts.copy())
    snap = _snapshot_rewritten(tables, dev, cycles)
    got = HashTable(device=0, **GEOM)
    np.random.seed(7)
    got.merge_batch([snap])
    _check((got.table, got.counts), ref["a"], ref["b"], "merge_batch(DeviceTable)")


def test_install_device_reads_snapshot_after_torch_writes(mode, tables, dev, cycles):
    ref_a, ref_b = [(t.table.copy(), t.counts.copy()) for t in tables]
    snap = _snapshot_rewritten(tables, dev, cycles)
    got = HashTable(device=0, **GEOM)
    got._install_device(snap)
    _check((got.table, got.counts), ref_a, ref_b, "HashTable._install_device")


# ---- write after read ---------------------------------------------------------------------------
def test_pcm_frontend_to_device_writes_after_torch_reads(mode, tracks, dev, cycles, monkeypatch):
    raw = tracks[0]
    ref = an_mod.pcm_frontend(raw, 1, 2 * SR, SR)
    with _freed_block_under_pending_read(cycles, torch.empty(len(ref), dtype=torch.float32, device=dev),
                                         monkeypatch):
        got = an_mod.pcm_frontend(raw, 1, 2 * SR, SR, device=dev.index, to_host=False)
    assert np.array_equal(got.cpu().numpy(), ref)


def test_pcm_frontend_batch_writes_after_torch_reads(mode, tracks, dev, cycles, monkeypatch):
    raws = [tracks[0], np.stack([tracks[1], tracks[2]], axis=1).reshape(-1)]
    args = (raws, [1, 2], [SR, 2 * SR], SR)
    ref, off, lens = an_mod.pcm_frontend_batch(*args, device=dev.index)
    ref = ref.cpu()
    with _freed_block_under_pending_read(cycles, torch.empty_like(ref, device=dev), monkeypatch):
        got, off2, lens2 = an_mod.pcm_frontend_batch(*args, device=dev.index)
    assert np.array_equal(off, off2) and np.array_equal(lens, lens2)
    assert torch.equal(got.cpu(), ref)


def test_export_device_writes_after_torch_reads(mode, tables, dev, cycles, monkeypatch):
    t = tables[1]
    like = torch.empty(t.table.shape, dtype=torch.int32, device=dev)
    with _freed_block_under_pending_read(cycles, like, monkeypatch):
        snap = t.export_device()
    assert np.array_equal(snap.table.cpu().numpy().view(np.uint32), t.table)
    assert np.array_equal(snap.counts.cpu().numpy(), t.counts)


def test_collect_hashes_on_device_writes_after_torch_reads(mode, an, tracks, dev, cycles, monkeypatch):
    ref = _hashes(an, tracks[:3])
    packed, starts, lens = an._pack(tracks[:3])
    total = sum(len(h) for h in ref)
    an.fingerprint_packed(packed, starts, fetch=False, sample_lengths=lens)
    results = [None] * 3
    with _freed_block_under_pending_read(cycles, torch.empty((total, 2), dtype=torch.int32, device=dev),
                                         monkeypatch):
        an._collect_hashes([0, 1, 2], results, True, False)
    for r, h in zip(results, ref):
        assert np.array_equal(r.rows.cpu().numpy(), h)


@pytest.mark.parametrize("buffer", ["qmax", "records"])
def test_match_sharded_batch_writes_after_torch_reads(mode, match_setup, dev, cycles, monkeypatch, buffer):
    ht, qa, _, qoff = match_setup
    # qmax is the first allocation of an options call, the records buffer the first of a plain one
    m = _matcher("exact_count" if buffer == "qmax" else "plain")
    ref = afd.match_sharded_batch(m, ht, (qa, qoff), row_cap=64)
    nq = len(qoff) - 1
    if buffer == "qmax":
        like = torch.empty(nq, dtype=torch.int32, device=dev)
    else:
        rb = int(_lib.context(0).lib.afp_shard_record_bytes(int(m.search_depth), 64))
        like = torch.empty((nq, rb), dtype=torch.uint8, device=dev)
    with _freed_block_under_pending_read(cycles, like, monkeypatch):
        got = afd.match_sharded_batch(m, ht, (qa, qoff), row_cap=64)
    assert _same(got, ref)


# ---- lifetime -----------------------------------------------------------------------------------
def test_fingerprint_pcm_buffer_outlives_the_device_work(mode, an, ctx, tracks, dev, cycles, monkeypatch):
    """_fingerprint_pcm fingerprints the front-end's buffer with fetch=False and drops it on return.
    The library's work is held behind a sleep on its stream; right after the return a tensor of the
    buffer's size is allocated and filled with other audio.  The hashes must be those of the files."""
    items = [(i, (t, 1, SR), len(t), None) for i, t in enumerate(tracks[:3])]
    ref = [None] * 3
    an._fingerprint_pcm(items, 1, [0.0] * 3)
    an._collect_hashes([0, 1, 2], ref, False, False)

    sizes, pending = [], []
    frontend = an_mod.pcm_frontend_batch

    def frontend_hook(*a, **k):
        out, off, lens = frontend(*a, **k)
        sizes.append(out.numel())
        return out, off, lens
    fingerprint = an.fingerprint_packed

    def fingerprint_hook(*a, **k):
        lib_stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
        with torch.cuda.stream(lib_stream):
            torch.cuda._sleep(cycles)
        out = fingerprint(*a, **k)
        pending.append(lib_stream.record_event())
        return out
    monkeypatch.setattr(an_mod, "pcm_frontend_batch", frontend_hook)
    monkeypatch.setattr(an, "fingerprint_packed", fingerprint_hook)
    other = torch.from_numpy(pcm_to_float(np.concatenate(tracks[3:6]))).to(dev)
    torch.cuda.synchronize(dev)
    an._fingerprint_pcm(items, 1, [0.0] * 3)
    assert not pending[0].query(), "the library's work finished before the buffer was dropped: tested nothing"
    scribble = torch.empty(sizes[0], dtype=torch.float32, device=dev)
    scribble[:len(other)].copy_(other[:sizes[0]])
    got = [None] * 3
    an._collect_hashes([0, 1, 2], got, False, False)
    for g, r in zip(got, ref):
        assert np.array_equal(g, r), "a dropped front-end buffer was reused while the library still read it"


# ---- afp_set_stream ------------------------------------------------------------------------------
@pytest.mark.parametrize("to", ["stream", "null"])
def test_set_stream_waits_for_the_outgoing_stream(mode, an, ctx, tracks, dev, cycles, to):
    off = np.array([0, len(tracks[0]), 2 * len(tracks[0])], np.int64)
    a = torch.from_numpy(np.concatenate(tracks[0:2])).to(dev)
    b = torch.from_numpy(np.concatenate(tracks[2:4])).to(dev)
    ref_a, ref_b = an.fingerprint_packed(a, off), an.fingerprint_packed(b, off)   # also sizes the workspace
    torch.cuda.synchronize(dev)
    outgoing = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    with torch.cuda.stream(outgoing):
        torch.cuda._sleep(cycles)
    an.fingerprint_packed(a, off, fetch=False)
    ev = outgoing.record_event()
    assert not ev.query(), "the previous batch finished before the switch: the case tested nothing"
    ctx.set_stream(torch.cuda.Stream(dev).cuda_stream if to == "stream" else None)
    an.fingerprint_packed(b, off, fetch=False)
    torch.cuda.synchronize(dev)
    got = [None] * 2
    an._collect_hashes([0, 1], got, False, False)
    rows = np.concatenate(got)
    got = (rows, np.array([0, len(got[0]), len(rows)], np.int64))
    _check(got, ref_a, ref_b, "set_stream(%s) after a fetch=False batch" % to,
           "the previous batch's kernels ran after the next batch's, in the same workspace")
