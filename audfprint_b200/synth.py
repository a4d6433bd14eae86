"""Seeded synthetic 11025 Hz mono int16 PCM (SURVEY.md §8d).

Track i uses seed i; query j uses seed 10**9 + j.  The generator is plain
NumPy on the host so that the oracle, the golden fixtures and the GPU run all
see the very same samples.  It is bench/test input plumbing, not part of the
fingerprint path.
"""
from __future__ import annotations

import numpy as np

SR = 11025
QUERY_SEED_BASE = 10 ** 9


def synth_track(seed: int, seconds: float, sr: int = SR, nbursts_per_30s: int = 20) -> np.ndarray:
    """White Gaussian noise (sigma = 0.1 FS) plus Gaussian-windowed tone bursts
    (f ~ U[100, 5000] Hz, width 0.3 s, amplitude 3 sigma), normalised to 0.5 FS
    peak and rounded to int16."""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * sr))
    sigma = 0.1
    x = rng.standard_normal(n) * sigma
    nb = max(1, int(round(nbursts_per_30s * seconds / 30.0)))
    t = np.arange(n) / sr
    freqs = rng.uniform(100.0, 5000.0, nb)
    centres = rng.uniform(0.0, seconds, nb)
    phases = rng.uniform(0.0, 2 * np.pi, nb)
    width = 0.3
    for f, c, ph in zip(freqs, centres, phases):
        lo = max(0, int((c - 4 * width) * sr))
        hi = min(n, int((c + 4 * width) * sr) + 1)
        if hi <= lo:
            continue
        tt = t[lo:hi]
        x[lo:hi] += 3 * sigma * np.exp(-0.5 * ((tt - c) / width) ** 2) * np.sin(2 * np.pi * f * tt + ph)
    peak = np.max(np.abs(x)) if n else 1.0
    if peak > 0:
        x = x * (0.5 / peak)
    return np.round(x * 32768.0).clip(-32768, 32767).astype(np.int16)


def synth_query(track_pcm: np.ndarray, qseed: int, seconds: float = 10.0,
                noise_sigma: float = 0.02, sr: int = SR):
    """A `seconds`-long excerpt of `track_pcm` at a seeded random offset plus
    additive white noise, re-quantised to int16.  Returns (pcm, offset_samples)."""
    rng = np.random.default_rng(QUERY_SEED_BASE + qseed)
    n = int(round(seconds * sr))
    n = min(n, len(track_pcm))
    off = int(rng.integers(0, len(track_pcm) - n + 1))
    x = track_pcm[off:off + n].astype(np.float64) / 32768.0
    x = x + rng.standard_normal(n) * noise_sigma
    return np.round(x * 32768.0).clip(-32768, 32767).astype(np.int16), off


def synth_table(hashbits: int = 20, depth: int = 100, nids: int = 1_000_000, maxtimebits: int = 12,
                seed: int = 0, overflow: int = 50):
    """A hash table of the bench geometry with every slot filled: uniform-random ids in
    [0, nids) and times in [0, 2^maxtimebits), counts[b] = depth + U[0, overflow) (buckets that
    saw more inserts than they hold).  Returns (table, counts, hashesperid), hashesperid being
    the entries each id holds."""
    rng = np.random.default_rng(seed)
    shape = (1 << hashbits, depth)
    table = rng.integers(1, nids + 1, size=shape, dtype=np.uint32) << np.uint32(maxtimebits)
    table |= rng.integers(0, 1 << maxtimebits, size=shape, dtype=np.uint32)
    counts = (depth + rng.integers(0, overflow, size=shape[0])).astype(np.int32)
    hpi = np.bincount((table >> np.uint32(maxtimebits)).ravel(), minlength=nids + 1)[1:].astype(np.uint32)
    return table, counts, hpi


def pcm_to_float(pcm: np.ndarray) -> np.ndarray:
    """int16 -> float32 in [-1, 1), exactly what the reference's reader yields
    (audio_read.py:139-145: scale 1/32768 applied to '<i2' samples)."""
    return (pcm.astype(np.float32) * np.float32(1.0 / 32768.0)).astype(np.float32)
