"""Extended-precision statement of the PCM front-end (csrc/afp_pcm.cu) and the bar it is held to.
TEST INFRASTRUCTURE, like tests/exact_stft.py.

The operation, for interleaved int16 PCM of `ch` channels resampled by up/down:

  mono[j] = RN32( (sum_c pcm[j][c]) / (32768 ch) )
  out[n]  = RN32( sum_j taps[n*down + half - j*up] * mono[j] ),   0 <= j < nframes,

with `taps` = analyzer.resample_taps(up, down) (2*half + 1 doubles, the very values the kernel
multiplies by) and len(out) = ceil(nframes * up / down).  RN32 is round-to-nearest-even to float32.

The channel sum is an integer below 2^24 in magnitude for ch <= 512, so the down-mix has one
rounding.  The polyphase sum is evaluated here in `np.longdouble` (64-bit mantissa): with m the most
terms of one output and S = sum_j |taps[.] * mono[j]|, it is within ref_err = (m + 1) 2^-64 S of the
exact sum.  The kernel accumulates in float64, within 1.01 m 2^-53 S of it.  So wherever the exact sum
is farther than delta = ref_err + 1.01 m 2^-53 S from a float32 rounding boundary, the kernel's
float32 output is the correctly rounded one; `check_rounded` asserts that, and allows one ulp in
the tie zone where it is not decided.
"""
from __future__ import annotations

import functools
from math import gcd

import numpy as np

from audfprint_b200.analyzer import resample_taps

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "np.longdouble must have a 64-bit mantissa (x86-64 extended precision)"

U53 = 2.0 ** -53
U64 = 2.0 ** -64
TARGET = 11025

# (source rate, target rate): every common rate into 11025 Hz, a source rate with gcd 1
# (44056: up 11025, down 44056, 881,121 taps) and two other targets
RATE_PAIRS = [(fs, TARGET) for fs in (8000, 12000, 16000, 22050, 24000, 32000, 37800, 44100, 48000,
                                      88200, 96000, 176400, 192000, 44056)] + [(44100, 22050), (48000, 8000)]


def up_down(src: int, dst: int) -> tuple[int, int]:
    g = gcd(int(src), int(dst))
    return int(dst) // g, int(src) // g


@functools.lru_cache(maxsize=None)
def taps_for(up: int, down: int) -> np.ndarray:
    t = resample_taps(up, down)
    t.setflags(write=False)
    return t


def n_out(nframes: int, up: int, down: int) -> int:
    return -(-int(nframes) * up // down)


def downmix(raw: np.ndarray, ch: int) -> np.ndarray:
    """mono float32: the exact integer channel sum, rounded once.  s / (32768 ch) is formed in
    float64 first; unless it is a float32 boundary itself it lies at least 2^-25 / ch (relative)
    away from one, far beyond float64's 2^-53, so the second rounding gives RN32 of the quotient."""
    s = np.asarray(raw, np.int16).reshape(-1, ch).astype(np.int64).sum(axis=1)
    return (s.astype(np.float64) / float(32768 * ch)).astype(np.float32)


def terms(mono: np.ndarray, up: int, down: int, taps: np.ndarray, n: np.ndarray, dtype=LD):
    """(t, x), both (len(n), m) in `dtype`: the taps and input samples of outputs n, term i using
    tap p + i*up and input sample floor(centre / up) - i (centre = n*down + half, p = centre mod up).
    Terms outside the taps or outside the input are 0 in both."""
    x = np.asarray(mono, np.float32)
    ntaps, nframes = len(taps), len(x)
    half = (ntaps - 1) // 2
    m = -(-ntaps // up)
    centre = np.asarray(n, np.int64) * down + half
    i = np.arange(m, dtype=np.int64)
    k = (centre % up)[:, None] + i[None, :] * up
    j = (centre // up)[:, None] - i[None, :]
    ok = (k < ntaps) & (j >= 0) & (j < nframes)
    t = np.where(ok, taps[np.minimum(k, ntaps - 1)], 0.0).astype(dtype)
    xv = np.where(ok, x[np.clip(j, 0, max(nframes - 1, 0))] if nframes else 0.0, 0.0).astype(dtype)
    return t, xv


def reference(mono: np.ndarray, up: int, down: int, n=None, chunk_terms: int = 1 << 21):
    """(ref longdouble, S float64, m) for outputs n (default: all of them).  up = down = 1 is the
    down-mix alone: ref is mono, m = 1."""
    x = np.asarray(mono, np.float32)
    total = n_out(len(x), up, down)
    n = np.arange(total, dtype=np.int64) if n is None else np.asarray(n, np.int64)
    assert n.size == 0 or (n.min() >= 0 and n.max() < total)
    if (up, down) == (1, 1):
        ref = x[n].astype(LD)
        return ref, np.abs(x[n]).astype(np.float64), 1
    taps = taps_for(up, down)
    m = -(-len(taps) // up)
    ref = np.empty(len(n), LD)
    S = np.empty(len(n), np.float64)
    step = max(1, chunk_terms // m)
    for s in range(0, len(n), step):
        t, xv = terms(x, up, down, taps, n[s:s + step])
        prod = t * xv
        ref[s:s + step] = prod.sum(axis=1)
        S[s:s + step] = np.abs(prod).sum(axis=1)
    return ref, S, m


def tie_delta(S, m: int):
    """Half-width of the tie zone: the reference's error plus the float64 accumulation's."""
    return ((m + 1) * U64 + 1.01 * m * U53) * np.asarray(S, np.float64)


def check_rounded(got, ref, S, m: int, what: str = "") -> int:
    """got == RN32(ref) at every sample whose ref is farther than tie_delta(S, m) from a float32
    rounding boundary, |got - ref| <= 1 ulp at the others.  Returns the number of the others."""
    got = np.asarray(got)
    assert got.dtype == np.float32 and got.shape == ref.shape, (what, got.dtype, got.shape, ref.shape)
    rn = ref.astype(np.float32)
    hi = (rn.astype(LD) + np.nextafter(rn, np.float32(np.inf)).astype(LD)) / 2
    lo = (rn.astype(LD) + np.nextafter(rn, np.float32(-np.inf)).astype(LD)) / 2
    dist = np.minimum(hi - ref, ref - lo)
    tie = dist <= tie_delta(S, m)
    bad = np.flatnonzero(~tie & (got != rn))
    assert bad.size == 0, "%s: %d samples not correctly rounded, first at %s: got %r want %r (ref %r)" % (
        what, bad.size, bad[:5].tolist(), got[bad[:5]].tolist(), rn[bad[:5]].tolist(),
        [float(v) for v in ref[bad[:5]]])
    ulp = np.spacing(np.maximum(np.abs(rn), np.abs(got))).astype(LD)
    far = np.flatnonzero(tie & (np.abs(got.astype(LD) - ref) > ulp))
    assert far.size == 0, "%s: %d tie-zone samples more than 1 ulp off, first at %s" % (
        what, far.size, far[:5].tolist())
    return int(np.count_nonzero(tie))


# ---- inputs -------------------------------------------------------------------------------------

def noise_tone(n: int, ch: int, fs: int, seed: int) -> np.ndarray:
    """(n, ch) int16: Gaussian noise (sigma 6000) plus a 997 Hz tone of amplitude 9000 on channel 0."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, ch)) * 6000.0
    x[:, 0] += 9000.0 * np.sin(2 * np.pi * 997.0 * np.arange(n) / fs)
    return np.round(x).clip(-32768, 32767).astype(np.int16)
