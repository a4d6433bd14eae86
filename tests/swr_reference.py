"""Statement of what `ffmpeg -i F -f s16le -ac 1 -ar 11025 -` does to 16-bit mono or stereo PCM: the
down-mix and resampling of libswresample (FFmpeg 8.0) with the library's defaults.  The reference
reads every file through that command (audio_read.py:196-203); the device front-end of
audfprint_b200/csrc/afp_swr.cu computes the same bits.

Equal rates: the library works in s16.  Stereo is mixed with Q15 weights, (16384 (l + r) + 16384) >> 15.

Different rates: the library works in float32.  The samples become x / 32768 and
  bank     P phases x L float32 taps: tap i of phase p weighs the input at offset i - (L-1)//2 - p/P
           from the output's position.  The taps are a Kaiser-windowed sinc (beta 9, cut-off 0.97 of
           the output band, 32 taps per output period, I0 by its power series) evaluated in double
           with math.sin / math.sqrt, divided by the sum of phase 0 and rounded to float32.
  position output n sits at input position n * D / P (D = in / g, P = out / g, P <= 1024: the
           exact-rational phases; other rates need interpolated phases and are refused, as are
           designs longer than 528 taps, i.e. rates above 176400 Hz).
  sum      the FMA3 kernel the library runs on x86: eight float32 lanes, lane k accumulating taps
           k, k+8, ... by fused multiply-add from zero, then lanes (k, k+4) added, then (k, k+2),
           then the last two.
  edges    x past its end is x mirrored around its end (x[N-1+k] = x[N-k]) for R samples and x
           before 0 is that extended x mirrored around sample 0 (x[-k] = x[k]).  Outputs run while
           their first input sample (n D // P) leaves the whole window in the extended input.  When N > L, R = (m + 1) // 2 with m the
           samples left in the library's buffer once every output whose window fits in x is made;
           otherwise R = (N + 1) // 2, and there are no outputs at all when N + R <= L.
  stereo   each channel is resampled, and the two results mixed as 0.5 l + 0.5 r in float32.
  output   lrintf(v * 32768) clipped to int16.

The module needs only NumPy and math.  The CPU tests hold it to the library's own output
(tests/golden/ffmpeg_frontend.npz) and the device front-end to it.
"""
from __future__ import annotations

import math

import numpy as np

OUT_RATE = 11025
FILTER_SIZE = 32
PHASE_COUNT = 1024
CUTOFF = 0.97
BETA = 9.0
LANES = 8
# 176400 Hz (528 taps) matches the library; 192000 Hz (575 taps) does not yet, so longer designs
# are refused
MAX_TAPS = 528


class Unsupported(ValueError):
    """An input this statement, like the device front-end, refuses."""


def bessel_i0(x):
    """I0(x) by its power series, summed in double until the terms stop changing the sum."""
    s, t, k, q = 1.0, 1.0, 1, x * x / 4.0
    while True:
        t *= q / (k * k)
        if s + t == s:
            return s
        s += t
        k += 1


def geometry(in_rate, out_rate=OUT_RATE):
    """(P phases, D phase step, L taps, factor) of the design for in_rate -> out_rate."""
    if in_rate < 1 or out_rate < 1:
        raise Unsupported("sample rate must be positive")
    g = math.gcd(in_rate, out_rate)
    P, D = out_rate // g, in_rate // g
    if P > PHASE_COUNT:
        raise Unsupported("%d Hz -> %d Hz needs interpolated phases" % (in_rate, out_rate))
    factor = min(out_rate * CUTOFF / in_rate, 1.0)
    L = max(int(math.ceil(FILTER_SIZE / factor)), 1)
    if L > MAX_TAPS:
        raise Unsupported("%d Hz -> %d Hz: %d taps, not yet matched to the library" % (in_rate, out_rate, L))
    return P, D, L, factor


def design(in_rate, out_rate=OUT_RATE):
    """float32 (P, L) bank."""
    P, _, L, factor = geometry(in_rate, out_rate)
    center = (L - 1) // 2
    bank = np.zeros((P, L), np.float32)
    norm = 0.0
    for ph in range(P if P % 2 else P // 2 + 1):
        s = math.sin(math.pi * ph / P) * (1 if center & 1 else -1) if factor == 1.0 else 0.0
        tab = []
        for i in range(L):
            x = math.pi * (float(i - center) - float(ph) / P) * factor
            if x == 0:
                y = 1.0
            elif factor == 1.0:
                y = s / x
            else:
                y = math.sin(x) / x
            w = 2.0 * x / (factor * L * math.pi)
            y *= bessel_i0(BETA * math.sqrt(max(1 - w * w, 0.0)))
            tab.append(y)
            s = -s
            if ph == 0:
                norm += y
        bank[ph] = np.array([t / norm for t in tab], np.float64).astype(np.float32)
        if P % 2 == 0 and ph > 0:
            bank[P - ph] = bank[ph][::-1]
    return bank


def out_length(n, in_rate, out_rate=OUT_RATE):
    """Number of samples the library yields for n input frames."""
    if in_rate == out_rate:
        return n
    return _edges(n, in_rate, out_rate)[0]


def _edges(n, in_rate, out_rate):
    """(outputs, R samples of reflection past the end) for n input frames."""
    P, D, L, _ = geometry(in_rate, out_rate)
    S = (L - 1) // 2 + n                                   # input samples past x[-(L-1)//2]
    if n <= L:
        R = (n + 1) // 2
        if n + R <= L:
            return 0, R
    else:
        made = ((S - L + 1) * P - 1) // D + 1              # outputs before the end is reflected
        R = (min(S - made * D // P, L) + 1) // 2
    return ((S + R - L + 1) * P - 1) // D + 1, R


def _fma(a, b, c):
    """float32 fused multiply-add, exact: round(a b + c) once to float32.

    a b is exact in float64 (48 significant bits).  s = RN64(a b + c) then rounds to the same float32
    as the exact sum unless s lands exactly on a float32 midpoint; there the float64 rounding error
    e (TwoSum, exact) says on which side of the midpoint the exact sum lies."""
    p = a.astype(np.float64) * b
    c = c.astype(np.float64)
    s = p + c
    z = s - p
    e = (p - (s - z)) + (c - z)                 # a b + c = s + e exactly
    r = s.astype(np.float32)
    other = np.nextafter(r, np.where(s > r, np.float32(np.inf), np.float32(-np.inf)))
    tie = (s != r) & (s == (r.astype(np.float64) + other) / 2) & (e != 0)
    if tie.any():
        up = np.where(e > 0, np.maximum(r, other), np.minimum(r, other))
        r = np.where(tie, up, r)
    return r


def resample_float(x, in_rate, out_rate=OUT_RATE, bank=None):
    """float32 mono samples -> float32 at out_rate, before the conversion to int16."""
    x = np.asarray(x, np.float32)
    P, D, L, _ = geometry(in_rate, out_rate)
    if bank is None:
        bank = design(in_rate, out_rate)
    n = len(x)
    nout, R = _edges(n, in_rate, out_rate)
    if nout == 0:
        return np.zeros(0, np.float32)
    A = -(-L // LANES) * LANES
    tail = np.concatenate([x, x[::-1][:R]])
    lead = L                                                 # mirrored samples before x[0]
    ext = np.concatenate([tail[1:L + 1][::-1], tail, np.zeros(A, np.float32)])
    taps = np.zeros((P, A), np.float32)
    taps[:, :L] = bank
    k = np.arange(nout, dtype=np.int64) * D
    start = k // P - (L - 1) // 2 + lead
    rows = taps[k % P]
    acc = np.zeros((nout, LANES), np.float32)
    lane = np.arange(LANES)
    for j in range(0, A, LANES):
        acc = _fma(ext[start[:, None] + j + lane[None, :]], rows[:, j:j + LANES], acc)
    acc = (acc[:, :4] + acc[:, 4:]).astype(np.float32)
    acc = (acc[:, :2] + acc[:, 2:]).astype(np.float32)
    return (acc[:, 0] + acc[:, 1]).astype(np.float32)


def to_s16(v):
    return np.clip(np.rint(np.asarray(v, np.float32) * np.float32(32768)), -32768, 32767).astype(np.int16)


def frontend(x, channels, in_rate, out_rate=OUT_RATE):
    """Interleaved int16 PCM of 1 or 2 channels -> the int16 mono the library yields."""
    if channels not in (1, 2):
        raise Unsupported("%d channels" % channels)
    x = np.asarray(x, np.int16).reshape(-1, channels)
    if in_rate == out_rate:
        if channels == 1:
            return x[:, 0].copy()
        return ((16384 * (x[:, 0].astype(np.int64) + x[:, 1]) + 16384) >> 15).astype(np.int16)
    f = x.astype(np.float32) * np.float32(1.0 / 32768)
    if channels == 1:
        return to_s16(resample_float(f[:, 0], in_rate, out_rate))
    half = np.float32(0.5)
    bank = design(in_rate, out_rate)
    l, r = (resample_float(f[:, c], in_rate, out_rate, bank) for c in (0, 1))
    return to_s16(l * half + r * half)
