"""Time the front-end call and wavfiles2hashes end to end for N x 30 s stereo 48 kHz files stored as s16,
s24 and f32 WAV, in both resampler modes.  Prints one JSON line per (format, mode) and writes them, with
the card's name and power limit, to profiles/wide_pcm_timing.json.

    python tools/wide_pcm_timing.py [--files 1024] [--seconds 30] [--reps 3]

The front-end time is one byte-form call (afp_pcm_frontend_batch_bytes / afp_swr_frontend_batch_bytes)
over the payloads already on the device, timed with a synchronise; end to end includes reading the files
and the host-to-device copy of their payloads.  Files are 8 distinct seeded signals linked under N names.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import Analyzer, _lib, analyzer as A  # noqa: E402
from tests import wide_pcm_cases as WC  # noqa: E402
from tests import wide_pcm_reference as W  # noqa: E402

RATE = 48000


def make_files(d, fmt, nfiles, seconds):
    rng = np.random.default_rng(1)
    base = []
    for k in range(8):
        x = rng.uniform(-0.5, 0.5, (int(RATE * seconds), 2))
        if fmt == "s16":
            data = WC.wav_bytes(np.rint(x * 32767).astype("<i2").tobytes(), RATE, 2, 1, 16)
        elif fmt == "s24":
            data = WC.wav_bytes(WC.payload_of(np.rint(x * (1 << 23)).reshape(-1), W.S24), RATE, 2, 1, 24)
        else:
            data = WC.wav_bytes(WC.payload_of(x.reshape(-1), W.F32), RATE, 2, 3, 32)
        p = os.path.join(d, "%s_base%d.wav" % (fmt, k))
        with open(p, "wb") as f:
            f.write(data)
        base.append(p)
    names = []
    for i in range(nfiles):
        p = os.path.join(d, "%s_%04d.wav" % (fmt, i))
        os.symlink(base[i % 8], p)
        names.append(p)
    return names


def frontend_ms(names, resampler, reps):
    import torch
    raws = [A._wav_read_raw(n) for n in names]
    pays = [A._as_payload(r, A._raw_format(r)) for r, _, _ in raws]
    packed, boff = A._pack_payloads([b for b, _ in pays])
    dev = torch.from_numpy(packed).to("cuda:0")
    fmts = [k for _, k in pays]
    nfr = [len(b) // A._WIDTH[k] // 2 for b, k in pays]
    ctx = _lib.context(0)
    args = (ctx, dev, boff[:-1], nfr, [2] * len(names), [RATE] * len(names), 11025, resampler, fmts)
    A._frontend_packed(*args)
    torch.cuda.synchronize()
    best = []
    for _ in range(reps):
        t = time.perf_counter()
        A._frontend_packed(*args)
        ctx.sync()
        best.append((time.perf_counter() - t) * 1e3)
    return float(np.median(best)), int(packed.nbytes)


def end_to_end_ms(names, resampler, reps):
    an = Analyzer(resampler=resampler, device=0)
    an.wavfiles2hashes(names[:8])
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        an.wavfiles2hashes(names)
        out.append((time.perf_counter() - t) * 1e3)
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rows = []
    with tempfile.TemporaryDirectory() as d:
        for fmt in ("s16", "s24", "f32"):
            names = make_files(d, fmt, a.files, a.seconds)
            for mode in ("poly", "ffmpeg"):
                fe, nbytes = frontend_ms(names, mode, a.reps)
                row = dict(format=fmt, resampler=mode, files=a.files, seconds=a.seconds, payload_bytes=nbytes,
                           frontend_ms=round(fe, 2), wavfiles2hashes_ms=round(end_to_end_ms(names, mode, a.reps), 1),
                           card=card)
                print(json.dumps(row), flush=True)
                rows.append(row)
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    with open(os.path.join(ROOT, "profiles", "wide_pcm_timing.json"), "w") as f:
        json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
