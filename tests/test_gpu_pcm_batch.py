"""The batched PCM front-end (`afp_pcm_frontend_batch`, csrc/afp_pcm.cu): one call over a ragged list
of files gives, for every file, the bits `afp_pcm_frontend` gives on that file alone - every rate pair
of tests/exact_resample.py, 1 to 16 channels, lengths from 0 to 3 s, a repeated file and empty files
inside the list - in one launch, without touching the alignment gaps, from host or device PCM; and
every bad argument fails before anything is written."""
import ctypes as C

import numpy as np
import pytest
import torch

from audfprint_b200 import _lib
from audfprint_b200 import analyzer as an_mod
from tests.exact_resample import RATE_PAIRS, TARGET, check_rounded, downmix, n_out, noise_tone, reference, \
    taps_for, up_down

pytestmark = pytest.mark.gpu

GUARD = np.uint32(0x7FC0DEAD)          # a NaN payload no front-end output can have
P64 = C.POINTER(C.c_int64)


def _single(ctx, raw, ch, up, down):
    """afp_pcm_frontend on one file, host in, host out."""
    raw = np.ascontiguousarray(raw, np.int16).reshape(-1)
    nframes = len(raw) // ch
    taps = taps_for(up, down) if (up, down) != (1, 1) else None
    out = np.empty(max(n_out(nframes, up, down), 1), np.float32)
    n = C.c_int64(-1)
    ctx.check(ctx.lib.afp_pcm_frontend(ctx.h, raw.ctypes.data if nframes else None, 1, nframes, ch, up, down,
                                       taps.ctypes.data if taps is not None else None,
                                       len(taps) if taps is not None else 0, out.ctypes.data, 1, C.byref(n)))
    return out[:n.value]


class Batch:
    """The arguments of one afp_pcm_frontend_batch call over files [(raw (n, ch) int16, ch, up, down)]."""

    def __init__(self, files, lead=0):
        self.n = len(files)
        raws = [np.ascontiguousarray(f[0], np.int16).reshape(-1) for f in files]
        self.ch = np.array([f[1] for f in files], np.int32)
        self.up = np.array([f[2] for f in files], np.int32)
        self.down = np.array([f[3] for f in files], np.int32)
        self.nframes = np.array([len(r) // c for r, c in zip(raws, self.ch)], np.int64)
        self.inoff = lead + np.concatenate([[0], np.cumsum([len(r) for r in raws])])[:-1].astype(np.int64)
        self.pcm = np.concatenate([np.full(lead, 777, np.int16)] + raws + [np.full(3, -5, np.int16)])
        self.pcm_len = len(self.pcm) - 3
        self.rates, self.toff, self.taps = an_mod.taps_table(zip(self.up, self.down))

    def call(self, ctx, out, capacity, off=None, lens=None, pcm_ptr=None, on_host=1, **over):
        a = dict(pcm=pcm_ptr if pcm_ptr is not None else self.pcm.ctypes.data, pcm_len=self.pcm_len, n=self.n,
                 inoff=self.inoff, nframes=self.nframes, ch=self.ch, up=self.up, down=self.down,
                 npairs=len(self.rates), rates=self.rates, toff=self.toff, taps=self.taps)
        a.update(over)
        rates = np.ascontiguousarray(a["rates"], np.int32)
        return ctx.lib.afp_pcm_frontend_batch(
            ctx.h, a["pcm"], on_host, a["pcm_len"], a["n"], a["inoff"].ctypes.data_as(P64),
            a["nframes"].ctypes.data_as(P64), a["ch"].ctypes.data, a["up"].ctypes.data, a["down"].ctypes.data,
            a["npairs"], rates.ctypes.data, a["toff"].ctypes.data_as(P64), a["taps"].ctypes.data, out, capacity,
            off.ctypes.data_as(P64) if off is not None else None, lens.ctypes.data_as(P64) if lens is not None else None)

    def size(self, ctx):
        off, lens = np.zeros(self.n + 1, np.int64), np.zeros(self.n, np.int64)
        ctx.check(self.call(ctx, None, 0, off, lens))
        return off, lens

    def guarded_out(self, ctx, total):
        dev = torch.device("cuda", ctx.device)
        out = torch.full((total + 8,), int(GUARD.view(np.int32)), dtype=torch.int32, device=dev)
        torch.cuda.synchronize(dev)
        return out


def _ragged_files():
    """Every rate pair at 0, 1, down - 1, down, down + 1 and shorter-than-reach lengths plus one 3 s
    file, the channel counts spread over them; an empty file and a repeated file inside the list."""
    files, chs = [], (1, 2, 3, 6, 8, 16)
    k = 0
    for src, dst in RATE_PAIRS:
        up, down = up_down(src, dst)
        reach = ((len(taps_for(up, down)) - 1) // 2) // up
        for n in sorted({0, 1, down - 1, down, down + 1, max(1, reach // 2)}):
            ch = chs[k % len(chs)]
            files.append((noise_tone(n, ch, src, 100 + k), ch, up, down))
            k += 1
        files.append((noise_tone(3 * src, 2, src, 100 + k), 2, up, down))
        k += 1
    for ch in chs:                                      # down-mix only, and mono at the target rate
        files.append((noise_tone(TARGET // 3 + ch, ch, TARGET, ch), ch, 1, 1))
    files.insert(5, files[3])                           # a file repeated
    files.insert(9, (np.zeros((0, 3), np.int16), 3, 1, 4))   # an empty file between two others
    return files


@pytest.fixture(scope="module")
def ragged():
    return _ragged_files()


def test_one_call_bit_matches_each_file_alone(ragged):
    ctx = _lib.context()
    b = Batch(ragged, lead=5)
    off, lens = b.size(ctx)
    assert np.all(off[:-1] % 4 == 0) and np.all(np.diff(off) >= lens) and np.all(np.diff(off) - lens < 4)
    out = b.guarded_out(ctx, int(off[-1]))
    n0 = ctx.launch_count()
    ctx.check(b.call(ctx, out.data_ptr(), out.numel(), None, None))
    assert ctx.launch_count() - n0 == 1                 # one launch for the whole list
    got = out.cpu().numpy().view(np.uint32)
    written = np.zeros(len(got), bool)
    for i, (raw, ch, up, down) in enumerate(ragged):
        want = _single(ctx, raw, ch, up, down)
        assert lens[i] == len(want) == n_out(len(raw), up, down)
        seg = got[off[i]:off[i] + lens[i]]
        assert np.array_equal(seg, want.view(np.uint32)), (i, ch, up, down, len(raw))
        written[off[i]:off[i] + lens[i]] = True
    assert np.all(got[~written] == GUARD)               # alignment gaps and the tail untouched
    assert (~written[:off[-1]]).any()
    # mono at the target rate is exactly x / 32768
    for i, (raw, ch, up, down) in enumerate(ragged):
        if (ch, up, down) == (1, 1, 1):
            seg = got[off[i]:off[i] + lens[i]].view(np.float32)
            assert np.array_equal(seg, raw.reshape(-1).astype(np.float32) / np.float32(32768))


def test_a_subset_is_correctly_rounded(ragged):
    ctx = _lib.context()
    pick = [f for f in ragged if len(f[0]) and f[2] in (1, 147, 441) and len(f[0]) < 40000][:12]
    b = Batch(pick)
    off, lens = b.size(ctx)
    out = b.guarded_out(ctx, int(off[-1]))
    ctx.check(b.call(ctx, out.data_ptr(), out.numel()))
    got = out.cpu().numpy().view(np.float32)
    checked = 0
    for i, (raw, ch, up, down) in enumerate(pick):
        ref, S, m = reference(downmix(raw, ch), up, down)
        assert check_rounded(got[off[i]:off[i] + lens[i]], ref, S, m, "batch file %d" % i) <= 4
        checked += 1
    assert checked >= 6


def test_host_and_device_pcm_give_the_same_bits(ragged):
    ctx = _lib.context()
    files = ragged[:40]
    b = Batch(files, lead=3)                            # the PCM starts an odd number of samples in
    off, _ = b.size(ctx)
    host = b.guarded_out(ctx, int(off[-1]))
    ctx.check(b.call(ctx, host.data_ptr(), host.numel()))
    dev = torch.device("cuda", ctx.device)
    dpcm = torch.from_numpy(b.pcm.copy()).to(dev)
    torch.cuda.synchronize(dev)
    devout = b.guarded_out(ctx, int(off[-1]))
    ctx.check(b.call(ctx, devout.data_ptr(), devout.numel(), pcm_ptr=dpcm.data_ptr(), on_host=0))
    assert torch.equal(host, devout)
    # the Python wrapper: the same bits as pcm_frontend file by file
    raws = [f[0].reshape(-1) for f in files[:12]]
    chans = [f[1] for f in files[:12]]
    src = [8000] * len(raws)
    out, o2, l2 = an_mod.pcm_frontend_batch(raws, chans, src, TARGET)
    o = out.cpu().numpy()
    for i, (r, c) in enumerate(zip(raws, chans)):
        assert np.array_equal(o[o2[i]:o2[i] + l2[i]].view(np.uint32),
                              an_mod.pcm_frontend(r, c, 8000, TARGET).view(np.uint32))


def test_launches_do_not_grow_with_the_file_count():
    ctx = _lib.context()
    rng = np.random.default_rng(3)
    for nf in (64, 4096):
        files = []
        for k in range(nf):
            ch = (1, 2)[k % 2]
            up, down = ((1, 4), (147, 640), (1, 1))[k % 3]
            files.append((rng.integers(-3000, 3000, (int(rng.integers(0, 300)), ch)).astype(np.int16), ch, up, down))
        b = Batch(files)
        off, lens = b.size(ctx)
        out = b.guarded_out(ctx, int(off[-1]))
        n0 = ctx.launch_count()
        ctx.check(b.call(ctx, out.data_ptr(), out.numel()))
        assert ctx.launch_count() - n0 == 1, nf
        got = out.cpu().numpy().view(np.uint32)
        for i in range(0, nf, 97):
            raw, ch, up, down = files[i]
            assert np.array_equal(got[off[i]:off[i] + lens[i]], _single(ctx, raw, ch, up, down).view(np.uint32))


def test_bad_arguments_raise_before_anything_is_written():
    ctx = _lib.context()
    rng = np.random.default_rng(9)
    files = [(rng.integers(-100, 100, (300, 2)).astype(np.int16), 2, 1, 4),
             (rng.integers(-100, 100, (200, 1)).astype(np.int16), 1, 147, 640),
             (rng.integers(-100, 100, (50, 1)).astype(np.int16), 1, 1, 1)]
    b = Batch(files)
    off, _ = b.size(ctx)
    out = b.guarded_out(ctx, int(off[-1]))

    def bad(**over):
        with pytest.raises(ValueError):
            ctx.check(b.call(ctx, out.data_ptr(), over.pop("capacity", out.numel()), **over))

    def at(name, i, v):
        a = getattr(b, name).copy()
        a[i] = v
        return {name: a}

    bad(**at("nframes", 1, -1))                                   # a negative length
    bad(**at("ch", 0, 0))                                         # fewer than 1 channel
    bad(**at("up", 2, 0))                                         # up below 1
    bad(**at("down", 1, 0))                                       # down below 1
    bad(**at("down", 2, -4))
    bad(**at("up", 0, 3))                                         # (3, 4) has no taps
    bad(toff=np.array([0, b.toff[1] - 1, b.toff[2] - 1], np.int64))   # an even-length design
    bad(**at("inoff", 2, b.pcm_len - 49))                         # input past the buffer's end
    bad(**at("inoff", 0, -2))                                     # input before its start
    bad(**at("nframes", 0, b.pcm_len))                            # a length that does not fit
    bad(pcm_len=b.pcm_len - 1)
    bad(capacity=int(off[-1]) - 1)                                # output larger than the buffer
    bad(n=-1)
    torch.cuda.synchronize()
    assert np.all(out.cpu().numpy().view(np.uint32) == GUARD)     # untouched
    ctx.check(b.call(ctx, out.data_ptr(), out.numel()))           # the context is still usable
    got = out.cpu().numpy().view(np.uint32)
    assert np.array_equal(got[off[2]:off[2] + 50], _single(ctx, *files[2]).view(np.uint32))
    # nothing to compute: no launch, offsets still returned
    e = Batch([(np.zeros((0, 1), np.int16), 1, 1, 4)] * 3)
    n0 = ctx.launch_count()
    o, ln = e.size(ctx)
    ctx.check(e.call(ctx, out.data_ptr(), out.numel()))
    assert ctx.launch_count() == n0 and o.tolist() == [0, 0, 0, 0] and ln.tolist() == [0, 0, 0]
