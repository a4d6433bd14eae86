"""Inputs of tests/golden/ffmpeg_frontend.npz, rebuilt from seeds: the library's output for each is
stored there (oracle/make_golden_ffmpeg_frontend.py), so the tests only need these arrays."""
from __future__ import annotations

import io
import wave

import numpy as np

from tests import swr_reference as R

RATES = (8000, 11025, 16000, 22050, 24000, 32000, 37800, 44100, 48000, 88200, 96000, 176400)
KINDS = ("noise", "square", "impulse", "silence")
# 30 s stereo files whose oracle hashes the golden file holds
SONGS = ((44100, 7), (48000, 8))


def lengths(rate):
    if rate == R.OUT_RATE:
        return (0, 1, 2, 100, rate)
    L = R.geometry(rate)[2]
    return (0, 1, 2, L // 2, L // 2 + 1, L - 1, L, L + 1, 2 * L, rate)


def cases():
    """(name, rate, channels, interleaved int16 pcm) of every short case."""
    out = []
    k = 0
    for rate in RATES:
        bank = None if rate == R.OUT_RATE else R.design(rate)
        for ch in (1, 2):
            for n in lengths(rate):
                kind = KINDS[k % len(KINDS)] if n < rate else KINDS[k % 2]
                k += 1
                rng = np.random.default_rng(1000 + k)
                if kind == "noise":
                    x = rng.integers(-32768, 32768, (n, ch))
                elif kind == "square":
                    # +-full scale with the sign of the taps it meets: the largest sums the FIR can make
                    t = np.sign(bank[0]) if bank is not None else np.ones(1)
                    s = np.resize(np.where(t >= 0, 32767, -32768), n)
                    x = np.stack([s, s[::-1]] if ch == 2 else [s], axis=1)
                elif kind == "impulse":
                    x = np.zeros((n, ch), np.int64)
                    if n:
                        x[rng.integers(0, n), rng.integers(0, ch)] = -32768
                else:
                    x = np.zeros((n, ch), np.int64)
                out.append(("%d_%d_%d_%s" % (rate, ch, n, kind), rate, ch, x.astype(np.int16).reshape(-1)))
    return out


def song(rate, seed, seconds=30.0):
    """Interleaved int16 stereo: tone bursts over noise, loud enough to clip now and then."""
    rng = np.random.default_rng(seed)
    n = int(rate * seconds)
    t = np.arange(n) / rate
    x = rng.normal(0, 300, (n, 2))
    for _ in range(120):
        f, a, t0, d = rng.uniform(150, 4500), rng.uniform(2000, 9000), rng.uniform(0, seconds), rng.uniform(0.1, 1.0)
        m = (t >= t0) & (t < t0 + d)
        x[m, 0] += a * np.sin(2 * np.pi * f * t[m])
        x[m, 1] += 0.7 * a * np.sin(2 * np.pi * f * t[m] + 1.0)
    return np.clip(np.rint(x), -32768, 32767).astype(np.int16).reshape(-1)


def wav_bytes(pcm, rate, ch):
    b = io.BytesIO()
    with wave.open(b, "wb") as w:
        w.setnchannels(ch)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes(np.asarray(pcm, "<i2").tobytes())
    return b.getvalue()


def flac_bytes(pcm, rate, ch):
    from tests import flac_writer
    return flac_writer.stream(np.asarray(pcm, np.int64).reshape(-1, ch), 16, rate)[0]


def wav_extensible_bytes(pcm, rate, ch, mask):
    """A 16-bit WAVE_FORMAT_EXTENSIBLE file with channel mask `mask`."""
    import struct
    data = np.asarray(pcm, "<i2").tobytes()
    guid = b"\x01\x00\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"     # KSDATAFORMAT_SUBTYPE_PCM
    fmt = struct.pack("<HHIIHHHHI", 0xFFFE, ch, rate, rate * 2 * ch, 2 * ch, 16, 22, 16, mask) + guid
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(data)) + data
    return b"RIFF" + struct.pack("<I", len(body)) + body
