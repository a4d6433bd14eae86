"""Statement of what `ffmpeg -i F -f s16le -ac 1 -ar 11025 -` does to 24-bit, 32-bit and float PCM and to
FLAC of 17-24 bits (FFmpeg 8.0, library defaults), on top of tests/swr_reference.py, which states the
16-bit case.  audfprint_b200/csrc/afp_swr.cu computes the same bits.

The decoders give s32 for 24-bit WAV (x << 8), 32-bit WAV (x) and b-bit FLAC (x << (32 - b)), and flt for
float WAV.  libswresample then makes s16 in one of three ways:
  mono, equal rates    s32 -> x >> 16 (floor); flt -> the s16 rule of v.
  stereo, equal rates  float32: each channel as a float (s32 as float(x) * 2^-31, flt as it is), then
                       0.5 l + 0.5 r, then the s16 rule.
  other rates          swr_reference.resample_float of those floats, per channel, mixed as above.
s16 rule: v * 32768 in float32, rounded half to even to int32, with NaN, +-Inf and anything outside
the int32 range giving INT32_MIN (x86 cvtps2dq), then saturated to int16 (packssdw).  The library
converts each buffer of n samples with that packed rule up to n & ~15 and the rest with its scalar
rule, av_clip_int16((int) lrintf(v * 32768)): rounded to int64 (NaN, +-Inf and anything outside the
int64 range give INT64_MIN), cut to its low 32 bits, then clipped.  The two differ only for NaN, +-Inf
and |v| >= 65536.  At equal rates a float WAV's buffers are the demuxer's 4096-byte packets, a multiple
of 16 frames, so the scalar rule takes the file's last n % 16 frames (scalar_tail).  At other rates the
buffers are the resampler's output per call; the statement takes the packed rule for all of them.

The default ('poly') front-end takes such a file as the int16 of the mono, equal-rate rule applied to
each sample (as_s16).

Sample formats are afp.h's AFP_PCM_* codes; the payload is the WAV data chunk's bytes as they are."""
from __future__ import annotations

import numpy as np

from tests import swr_reference as R

S16, F32, S24, S32 = 0, 1, 2, 3
WIDTH = {S16: 2, F32: 4, S24: 3, S32: 4}


def left_justified(payload, fmt):
    """Integer payload -> int32 samples holding x << (32 - bits), as the decoders give them."""
    b = np.frombuffer(bytes(payload), np.uint8)
    if fmt == S16:
        return b.view("<i2").astype(np.int32) << 16
    if fmt == S24:
        t = b[:len(b) // 3 * 3].reshape(-1, 3).astype(np.uint32)
        return ((t[:, 0] << 8) | (t[:, 1] << 16) | (t[:, 2] << 24)).view(np.int32)
    if fmt == S32:
        return b.view("<i4").astype(np.int32)
    raise ValueError("not an integer format: %r" % fmt)


def s16_rule(v):
    """float32 v -> int16: RNE(v * 32768) to int32, INT32_MIN for NaN, Inf or out of range, saturated."""
    t = np.asarray(v, np.float32) * np.float32(32768)
    ok = np.isfinite(t) & (t >= np.float32(-2.0 ** 31)) & (t < np.float32(2.0 ** 31))
    r = np.where(ok, np.rint(np.where(ok, t, 0)).astype(np.int64), -2 ** 31)
    return np.clip(r, -32768, 32767).astype(np.int16)


def scalar_s16_rule(v):
    """The library's scalar float -> s16 conversion (see the module's text)."""
    t = np.asarray(v, np.float32).astype(np.float64) * 32768.0
    ok = np.isfinite(t) & (np.abs(t) < 2.0 ** 63)
    r = np.rint(np.where(ok, t, 0)).astype(np.int64)             # INT64_MIN's low 32 bits are 0
    r = ((r & 0xFFFFFFFF) ^ 0x80000000) - 0x80000000
    return np.clip(r, -32768, 32767).astype(np.int16)


def scalar_tail(v):
    """s16 of float32 v converted as one equal-rate float stream: the last len % 16 by the scalar rule."""
    v = np.asarray(v, np.float32)
    out = s16_rule(v)
    k = len(v) - len(v) % 16
    out[k:] = scalar_s16_rule(v[k:])
    return out


def as_s16(payload, fmt):
    """Rule (1): the int16 of every sample."""
    if fmt == F32:
        return s16_rule(np.frombuffer(bytes(payload), "<f4"))
    return (left_justified(payload, fmt) >> 16).astype(np.int16)


def as_float(payload, fmt):
    """Rule (2): the float32 of every sample."""
    if fmt == F32:
        return np.frombuffer(bytes(payload), "<f4").astype(np.float32)
    return left_justified(payload, fmt).astype(np.float32) * np.float32(2.0 ** -31)


def frontend(payload, fmt, channels, in_rate, out_rate=R.OUT_RATE):
    """Interleaved payload of 1 or 2 channels -> the int16 mono the library yields."""
    if fmt == S16:
        return R.frontend(np.frombuffer(bytes(payload), "<i2"), channels, in_rate, out_rate)
    if channels not in (1, 2):
        raise R.Unsupported("%d channels" % channels)
    if in_rate == out_rate and channels == 1:
        return scalar_tail(as_float(payload, fmt)) if fmt == F32 else as_s16(payload, fmt)
    f = as_float(payload, fmt)
    f = f[:len(f) // channels * channels].reshape(-1, channels)
    if in_rate == out_rate:
        ch = [f[:, c] for c in range(channels)]
    else:
        bank = R.design(in_rate, out_rate)
        ch = [R.resample_float(f[:, c], in_rate, out_rate, bank) for c in range(channels)]
    if channels == 1:
        return s16_rule(ch[0])
    half = np.float32(0.5)
    v = ch[0] * half + ch[1] * half
    return scalar_tail(v) if fmt == F32 and in_rate == out_rate else s16_rule(v)
