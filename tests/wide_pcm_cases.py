"""Inputs of tests/golden/wide_pcm.npz, rebuilt from seeds: 24-bit, 32-bit and float WAV (plain and
WAVE_FORMAT_EXTENSIBLE) and 20- and 24-bit FLAC at the rates and edge lengths of
tests/ffmpeg_frontend_cases.py.  The library's output for each is stored there
(oracle/make_golden_wide_pcm.py), so the tests only need these bytes."""
from __future__ import annotations

import hashlib
import struct

import numpy as np

from tests import ffmpeg_frontend_cases as FC
from tests import wide_pcm_reference as W

RATES = (8000, 11025, 22050, 44100, 48000, 96000, 176400)
# (name, AFP_PCM_* code, WAVE format tag, container bits, extensible)
WAV_KINDS = (("s24", W.S24, 1, 24, False), ("s24x", W.S24, 1, 24, True), ("s32", W.S32, 1, 32, False),
             ("s32x", W.S32, 1, 32, True), ("f32", W.F32, 3, 32, False), ("f32x", W.F32, 3, 32, True))
FLAC_DEPTHS = (20, 24)
# 30 s songs: (name, rate, format); their oracle hashes are stored
SONGS = (("song_s24_48000", 48000, "s24"), ("song_f32_44100", 44100, "f32"))
# float specials: NaN, +-Inf, +-2e9, +-1.5, and the ties half an ulp of int16 either side of 1/32768
SPECIALS = np.array([np.nan, np.inf, -np.inf, 2e9, -2e9, 1.5, -1.5, 0.5 / 32768, 1.5 / 32768, 2.5 / 32768,
                     -0.5 / 32768, -1.5 / 32768, -2.5 / 32768, 32767.5 / 32768, -32768.5 / 32768, 1.0, -1.0,
                     65535.5 / 32768, -65536.5 / 32768, 0.0, -0.0], np.float32)

_GUID_TAIL = b"\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"


# outputs longer than this are stored as their first HEAD samples and a SHA-256 of the whole
HEAD = 4096


def store(out, key, pcm):
    """Put the library's int16 output under `key` of the golden dict (long ones as head + digest)."""
    pcm = np.ascontiguousarray(pcm, "<i2")
    if len(pcm) <= HEAD:
        out[key] = pcm
    else:
        out[key + "/head"] = pcm[:HEAD]
        out[key + "/sha256"] = np.frombuffer(hashlib.sha256(pcm.tobytes()).digest(), np.uint8)


def matches(g, key, pcm):
    """True when int16 `pcm` is what store() put under `key`."""
    pcm = np.ascontiguousarray(pcm, "<i2")
    if key in g.files:
        return np.array_equal(pcm, g[key])
    return (np.array_equal(pcm[:HEAD], g[key + "/head"]) and
            hashlib.sha256(pcm.tobytes()).digest() == g[key + "/sha256"].tobytes())


def wav_bytes(payload, rate, ch, tag, bits, extensible=False, valid_bits=None, mask=0, extra=b"", pad_chunk=None,
              fmt_size=None, data_size=None):
    """A RIFF WAVE file around `payload` (the data chunk's bytes).  extensible: WAVE_FORMAT_EXTENSIBLE with
    sub-format `tag`; fmt_size 18 adds a cbSize of 0 to a plain fmt chunk; pad_chunk: an unknown chunk of
    that many bytes (padded to even) before fmt; extra: bytes appended after the data chunk; data_size:
    the size the data chunk's header claims (default its length)."""
    width = (bits + 7) // 8
    if extensible:
        fmt = struct.pack("<HHIIHHHHI", 0xFFFE, ch, rate, rate * width * ch, width * ch, bits, 22,
                          valid_bits or bits, mask) + struct.pack("<I", tag) + _GUID_TAIL
    else:
        fmt = struct.pack("<HHIIHH", tag, ch, rate, rate * width * ch, width * ch, bits)
        if fmt_size == 18:
            fmt += b"\x00\x00"
    body = b"WAVE"
    if pad_chunk is not None:
        body += b"LIST" + struct.pack("<I", pad_chunk) + bytes(range(pad_chunk)) + b"\x00" * (pad_chunk & 1)
    body += b"fmt " + struct.pack("<I", len(fmt)) + fmt
    body += b"data" + struct.pack("<I", len(payload) if data_size is None else data_size) + bytes(payload)
    body += b"\x00" * (len(payload) & 1) + extra
    return b"RIFF" + struct.pack("<I", len(body)) + body


def payload_of(x, fmt):
    """int64 samples at the format's own depth (floats for F32) -> the data chunk's bytes."""
    if fmt == W.F32:
        return np.asarray(x, "<f4").tobytes()
    if fmt == W.S32:
        return np.asarray(x, np.int64).astype("<i4").tobytes()
    v = np.asarray(x, np.int64).astype("<i4").view(np.uint8).reshape(-1, 4)
    return v[:, :3].tobytes()


def signal(kind, n, ch, fmt, bits, rng, bank):
    """n x ch samples of `kind` at `bits` bits (floats in [-1, 1) for F32)."""
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    if kind == "noise":
        x = rng.integers(lo, hi + 1, (n, ch))
    elif kind == "square":
        t = np.sign(bank[0]) if bank is not None else np.ones(1)
        s = np.resize(np.where(t >= 0, hi, lo), n)
        x = np.stack([s, s[::-1]] if ch == 2 else [s], axis=1)
    elif kind == "impulse":
        x = np.zeros((n, ch), np.int64)
        if n:
            x[rng.integers(0, n), rng.integers(0, ch)] = lo
    else:
        x = np.zeros((n, ch), np.int64)
    if fmt == W.F32:
        x = x.astype(np.float64) / float(1 << (bits - 1))
        if kind == "noise":
            x = rng.uniform(-1.0, 1.0, (n, ch))
    return x


def cases():
    """(name, source, rate, channels, bytes, AFP_PCM_* code, payload) of every short case: source 'wav' or
    'flac'; payload is what the device reads (left-justified int32 for deep FLAC)."""
    out = []
    k = 0
    for rate in RATES:
        bank = None if rate == FC.R.OUT_RATE else FC.R.design(rate)
        for ch in (1, 2):
            for n in FC.lengths(rate):
                for name, fmt, tag, bits, ext in WAV_KINDS:
                    kind = FC.KINDS[k % len(FC.KINDS)] if n < rate else FC.KINDS[k % 2]
                    k += 1
                    x = signal(kind, n, ch, fmt, bits, np.random.default_rng(5000 + k), bank)
                    p = payload_of(x.reshape(-1), fmt)
                    data = wav_bytes(p, rate, ch, tag, bits, ext, mask=(0x4 if ch == 1 else 0x3) if ext else 0)
                    out.append(("%s_%d_%d_%d_%s" % (name, rate, ch, n, kind), "wav", rate, ch, data, fmt, p))
                if n < 16:
                    continue                  # FLAC blocks hold at least 16 samples
                for bits in FLAC_DEPTHS:
                    kind = FC.KINDS[k % len(FC.KINDS)] if n < rate else FC.KINDS[k % 2]
                    k += 1
                    x = signal(kind, n, ch, W.S32, bits, np.random.default_rng(5000 + k), bank)
                    data = flac_bytes(x, bits, rate)
                    p = (x.reshape(-1).astype(np.int64) << (32 - bits)).astype("<i4").tobytes()
                    out.append(("flac%d_%d_%d_%d_%s" % (bits, rate, ch, n, kind), "flac", rate, ch, data, W.S32, p))
    for rate in (11025, 44100):
        for ch in (1, 2):
            x = np.resize(SPECIALS, (len(SPECIALS) * 4 // ch, ch))
            x[:, -1] = x[::-1, 0] if ch == 2 else x[:, -1]
            p = payload_of(x.reshape(-1), W.F32)
            out.append(("special_%d_%d" % (rate, ch), "wav", rate, ch, wav_bytes(p, rate, ch, 3, 32), W.F32, p))
    return out


def flac_bytes(x, bits, rate):
    """FLAC of int64 samples (n, ch) at `bits` bits: verbatim subframes, independent channels."""
    from tests import flac_writer
    return flac_writer.stream(np.asarray(x, np.int64), bits, rate, specs=[{"kind": "verbatim"}] * x.shape[1])[0]


def song(rate, fmt_name, seconds=30.0):
    """-> (bytes of the file, AFP_PCM_* code, payload): tone bursts over noise, as FC.song, at full depth."""
    seed = {"s24": 21, "f32": 22}[fmt_name]
    rng = np.random.default_rng(seed)
    n = int(rate * seconds)
    t = np.arange(n) / rate
    x = rng.normal(0, 300 / 32768, (n, 2))
    for _ in range(120):
        f, a, t0, d = rng.uniform(150, 4500), rng.uniform(0.06, 0.28), rng.uniform(0, seconds), rng.uniform(0.1, 1.0)
        m = (t >= t0) & (t < t0 + d)
        x[m, 0] += a * np.sin(2 * np.pi * f * t[m])
        x[m, 1] += 0.7 * a * np.sin(2 * np.pi * f * t[m] + 1.0)
    if fmt_name == "s24":
        p = payload_of(np.clip(np.rint(x * (1 << 23)), -(1 << 23), (1 << 23) - 1).reshape(-1), W.S24)
        return wav_bytes(p, rate, 2, 1, 24), W.S24, p
    p = payload_of(x.reshape(-1), W.F32)
    return wav_bytes(p, rate, 2, 3, 32), W.F32, p


def chunk_cases():
    """(name, bytes, AFP_PCM_* code, channels, payload) of WAV files that pin the RIFF walk: fmt chunks of
    16, 18 and 40 bytes, an odd-size unknown chunk before fmt, a data size past the end of the file (whole
    frames present), wValidBitsPerSample below the container, bytes after the data chunk."""
    rng = np.random.default_rng(77)
    x24 = rng.integers(-(1 << 23), 1 << 23, 2 * 300)
    p24 = payload_of(x24, W.S24)
    xf = payload_of(rng.uniform(-1, 1, 2 * 300), W.F32)
    x32 = payload_of(rng.integers(-(1 << 31), 1 << 31, 300), W.S32)
    return [
        ("fmt16_s24", wav_bytes(p24, 44100, 2, 1, 24), W.S24, 2, p24),
        ("fmt18_s24", wav_bytes(p24, 44100, 2, 1, 24, fmt_size=18), W.S24, 2, p24),
        ("fmt40_s24", wav_bytes(p24, 44100, 2, 1, 24, extensible=True, mask=3), W.S24, 2, p24),
        ("fmt18_f32", wav_bytes(xf, 22050, 2, 3, 32, fmt_size=18), W.F32, 2, xf),
        ("odd_chunk_s32", wav_bytes(x32, 48000, 1, 1, 32, pad_chunk=13), W.S32, 1, x32),
        ("odd_chunk_f32x", wav_bytes(xf, 8000, 2, 3, 32, extensible=True, mask=3, pad_chunk=7), W.F32, 2, xf),
        ("past_eof_s24", wav_bytes(p24[:-42], 44100, 2, 1, 24, data_size=len(p24) + 600), W.S24, 2, p24[:-42]),
        ("past_eof_f32", wav_bytes(xf[:-20], 11025, 1, 3, 32, data_size=1 << 20), W.F32, 1, xf[:-20]),
        ("valid20_s24x", wav_bytes(p24, 48000, 2, 1, 24, extensible=True, valid_bits=20, mask=3), W.S24, 2, p24),
        ("trailing_list_s24", wav_bytes(p24, 96000, 1, 1, 24, extra=b"LIST\x05\x00\x00\x00abcde\x00"), W.S24, 1, p24),
    ]
