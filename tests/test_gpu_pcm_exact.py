"""The device PCM front-end (`afp_pcm_frontend`, csrc/afp_pcm.cu) at every output sample: each output
is the correctly rounded float32 of the down-mix + polyphase FIR, outside a tie zone of a few samples
(tests/exact_resample.py), for every common source rate, lengths from 1 sample to 3 s and a 10.8-minute
file, impulses, full-scale DC, stopband tones, 1-LSB material, 1 to 16 channels, and PCM or output in
device memory."""
import ctypes as C

import numpy as np
import pytest

from audfprint_b200 import _lib
from audfprint_b200 import analyzer as an_mod
from tests.exact_resample import (RATE_PAIRS, TARGET, check_rounded, downmix, n_out, noise_tone, reference,
                                  taps_for, up_down)

pytestmark = pytest.mark.gpu

AFP_ERR_INVALID = -2           # include/afp.h
TIE_MAX = 4                    # tie-zone samples allowed in one case


def _check(raw, ch, src, dst, what, tie_max=TIE_MAX):
    """Host PCM in, host float32 out, checked at every output; returns (out, tie-zone count)."""
    raw = np.ascontiguousarray(raw, np.int16)
    got = an_mod.pcm_frontend(raw.reshape(-1), ch, src, dst)
    up, down = up_down(src, dst)
    ref, S, m = reference(downmix(raw, ch), up, down)
    ties = check_rounded(got, ref, S, m, what)
    print("ties %-40s %d of %d" % (what, ties, len(got)))
    assert ties <= tie_max, (what, ties)
    return got, ties


def _geometry(src, dst):
    up, down = up_down(src, dst)
    half = (len(taps_for(up, down)) - 1) // 2
    return up, down, half, half // up              # reach: input samples one output spans on each side


@pytest.mark.parametrize("src,dst", RATE_PAIRS)
def test_every_output_at_every_length(src, dst):
    """Noise plus tone at 1, 2, down - 1, down, down + 1 samples, shorter than the filter's reach,
    5 down and 5 down + 1 (n up % down zero and not) and 3 s: every output, both ends included."""
    up, down, half, reach = _geometry(src, dst)
    lengths = sorted({1, 2, max(1, reach // 2), down - 1, down, down + 1, 5 * down, 5 * down + 1, 3 * src})
    assert max(1, reach // 2) < reach
    for i, n in enumerate(lengths):
        assert (n * up % down == 0) == (n % down == 0)
        ch = 2 if n == 3 * src else 1
        got, _ = _check(noise_tone(n, ch, src, src + i), ch, src, dst, "%d->%d n=%d ch=%d" % (src, dst, n, ch))
        assert len(got) == n_out(n, up, down)


@pytest.mark.parametrize("src,dst", RATE_PAIRS)
def test_impulses_dc_stopband_and_lsb(src, dst):
    up, down, half, reach = _geometry(src, dst)
    taps = taps_for(up, down)
    n = 6 * reach + 2 * down + 1
    # an input sample where an output's position wraps to the next input sample
    j_wrap = next(j for j in range(n // 2, n) if (j * up) % down < up)
    for j0 in (0, n - 1, j_wrap):
        raw = np.zeros(n, np.int16)
        raw[j0] = -32768                                # mono -1.0: the output is -taps, exactly
        got, ties = _check(raw, 1, src, dst, "%d->%d impulse at %d" % (src, dst, j0))
        k = np.arange(len(got), dtype=np.int64) * down + half - j0 * up
        inside = (k >= 0) & (k < len(taps))
        want = np.where(inside, -taps[np.clip(k, 0, len(taps) - 1)], 0.0).astype(np.float32)
        assert ties == 0 and np.array_equal(got, want), (src, dst, j0)
    got, _ = _check(np.full(n, -32768, np.int16), 1, src, dst, "%d->%d DC" % (src, dst))
    nn = np.arange(len(got), dtype=np.int64)
    interior = (nn * down >= half) & ((nn * down + half) // up <= n - 1)
    assert np.count_nonzero(interior) > 0 and np.max(np.abs(got[interior] + 1.0)) < 0.01
    assert not np.all(interior)
    # full scale above the output's Nyquist rate (no stopband when upsampling): S is large and the
    # output small, down to where the worst-case float64 error reaches a float32 ulp, so this is
    # where the tie zone fills up; at least half the outputs must still be correctly rounded
    f = 0.5 * (dst / 2 + src / 2) if src > dst else 0.45 * src
    t = np.arange(n) / src
    tone = np.round(32767.0 * np.sin(2 * np.pi * f * t + 0.3)).astype(np.int16)
    got, _ = _check(tone, 1, src, dst, "%d->%d tone %.0f Hz" % (src, dst, f), tie_max=n_out(n, up, down) // 2)
    if f > 1.3 * dst / 2:                               # clear of the transition band
        assert np.max(np.abs(got[interior])) < 0.05
    lsb = np.random.default_rng(src + dst).integers(-1, 2, n).astype(np.int16)
    _check(lsb, 1, src, dst, "%d->%d 1 LSB" % (src, dst))


def _channel_signals(ch, n, seed):
    rng = np.random.default_rng(seed)
    full = rng.integers(-32768, 32768, (n, ch)).astype(np.int16)
    low = np.full((n, ch), -32768, np.int16)
    cancel = np.zeros((n, ch), np.int16)            # channel pairs that sum to 0 exactly
    v = rng.integers(-32767, 32768, (n, ch // 2)).astype(np.int16)
    cancel[:, 0:2 * (ch // 2):2], cancel[:, 1:2 * (ch // 2):2] = v, -v
    if ch % 2:
        cancel[:, -1] = rng.integers(-3, 4, n)      # odd count: a small remainder, mean not dyadic
    return {"full": full, "all -32768": low, "cancelling": cancel}


@pytest.mark.parametrize("ch", [1, 2, 3, 6, 8, 16])
def test_downmix_at_the_native_rate_is_the_rounded_mean(ch):
    """up = down = 1 (a multi-channel 11025 Hz file): bit-equal to RN32(sum / (32768 ch)), no tie zone."""
    for name, raw in _channel_signals(ch, 20011, ch).items():
        got = an_mod.pcm_frontend(raw.reshape(-1), ch, TARGET, TARGET)
        assert np.array_equal(got, downmix(raw, ch)), (ch, name)
        if name == "all -32768":
            assert np.all(got == -1.0)
        if name == "cancelling" and ch % 2 == 0:
            assert np.all(got == 0.0)


@pytest.mark.parametrize("src,ch", [(44100, 2), (48000, 6), (16000, 3), (22050, 8), (32000, 16), (96000, 3)])
def test_downmix_then_resample(src, ch):
    for name, raw in _channel_signals(ch, src // 2 + 5, src + ch).items():
        _check(raw, ch, src, TARGET, "%d ch=%d %s" % (src, ch, name))
    _check(noise_tone(src + 3, ch, src, ch), ch, src, TARGET, "%d ch=%d noise" % (src, ch))


def _frontend(ctx, pcm_ptr, pcm_on_host, nframes, ch, up, down, out_ptr, out_on_host):
    taps = taps_for(up, down) if (up, down) != (1, 1) else None
    n = C.c_int64(-1)
    rc = ctx.lib.afp_pcm_frontend(ctx.h, pcm_ptr, pcm_on_host, nframes, ch, up, down,
                                  taps.ctypes.data if taps is not None else None,
                                  len(taps) if taps is not None else 0, out_ptr, out_on_host, C.byref(n))
    return rc, n.value


@pytest.mark.parametrize("src,ch", [(44100, 2), (48000, 1), (TARGET, 3), (8000, 3)])
def test_device_pcm_and_device_output_give_the_same_bits(src, ch):
    """Host in / host out is checked against the statement; device PCM in (also starting an odd
    number of samples into its tensor) and device float32 out give the same bits."""
    import torch
    raw = noise_tone(src // 2 + 3, ch, src, 11 * ch)
    host, _ = _check(raw, ch, src, TARGET, "%d ch=%d host" % (src, ch))
    flat = raw.reshape(-1)
    dev_out = an_mod.pcm_frontend(flat, ch, src, TARGET, to_host=False)
    assert dev_out.is_cuda and np.array_equal(dev_out.cpu().numpy(), host)
    ctx = _lib.context()
    dev = torch.device("cuda", ctx.device)
    up, down = up_down(src, TARGET)
    nframes = len(raw)
    for skip in (0, 1, 3):
        buf = torch.full((skip + flat.size + 5,), 12345, dtype=torch.int16, device=dev)
        buf[skip:skip + flat.size] = torch.from_numpy(flat.copy()).to(dev)
        torch.cuda.synchronize(dev)
        ptr = buf.data_ptr() + 2 * skip
        out_h = np.full(len(host), np.nan, np.float32)
        assert _frontend(ctx, ptr, 0, nframes, ch, up, down, out_h.ctypes.data, 1) == (0, len(host))
        assert np.array_equal(out_h, host), skip
        out_d = torch.full((len(host),), float("nan"), dtype=torch.float32, device=dev)
        torch.cuda.synchronize(dev)
        assert _frontend(ctx, ptr, 0, nframes, ch, up, down, out_d.data_ptr(), 0) == (0, len(host))
        assert np.array_equal(out_d.cpu().numpy(), host), skip


def test_long_input_crosses_2_31_and_2_32_in_the_index_arithmetic():
    """10.8 minutes of 48 kHz mono (31 M samples): n*down + half and j*up pass 2^31 and 2^32.  The
    outputs on both sides of each crossing, the first and the last are checked."""
    src, nframes, w = 48000, 31_000_000, 8192
    up, down, half, _ = _geometry(src, TARGET)
    raw = np.random.default_rng(48).integers(-20000, 20001, nframes, dtype=np.int16)
    got = an_mod.pcm_frontend(raw, 1, src, TARGET)
    total = n_out(nframes, up, down)
    assert len(got) == total
    idx = [np.arange(w), np.arange(total - w, total)]
    for b in (2 ** 31, 2 ** 32):
        c = (b - half) // down
        assert c * down + half < b <= (c + 1) * down + half and c + w < total - w
        idx.append(np.arange(c - w, c + w))
    idx = np.concatenate(idx)
    assert (idx[-1] * down + half) > 2 ** 32 and (total - 1) * down + half > 2 ** 32
    ref, S, m = reference(downmix(raw, 1), up, down, idx)
    ties = check_rounded(got[idx], ref, S, m, "48000 long")
    print("ties %-40s %d of %d" % ("48000 long", ties, len(idx)))
    assert ties <= TIE_MAX


def test_argument_checks():
    ctx = _lib.context()
    raw = np.zeros(64, np.int16)
    out = np.empty(64, np.float32)
    taps = taps_for(1, 4)
    nout = C.c_int64(-1)

    def call(nframes=64, ch=1, up=1, down=4, t=taps, ntaps=len(taps), pcm=raw.ctypes.data, o=out.ctypes.data):
        nout.value = -1
        return ctx.lib.afp_pcm_frontend(ctx.h, pcm, 1, nframes, ch, up, down, t.ctypes.data if t is not None else None,
                                        ntaps, o, 1, C.byref(nout))

    assert call(ntaps=len(taps) - 1) == AFP_ERR_INVALID                  # even tap count
    assert call(t=None, ntaps=0) == AFP_ERR_INVALID                      # resampling without taps
    for ch in (0, -1):
        assert call(ch=ch) == AFP_ERR_INVALID
    assert call(up=0) == AFP_ERR_INVALID and call(up=-3) == AFP_ERR_INVALID
    assert call(down=0) == AFP_ERR_INVALID
    assert call(nframes=-1) == AFP_ERR_INVALID
    assert call(pcm=None) == AFP_ERR_INVALID and call(o=None) == AFP_ERR_INVALID
    assert call(nframes=0, pcm=None, o=None) == 0 and nout.value == 0
    assert call(nframes=0, up=1, down=1, t=None, ntaps=0, pcm=None, o=None) == 0 and nout.value == 0
    assert call() == 0 and nout.value == 16                              # the context is still usable
    assert np.all(out[:16] == 0.0)
