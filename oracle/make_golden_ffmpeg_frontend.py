"""Write tests/golden/ffmpeg_frontend.npz: what FFmpeg 8.0's libraries (oracle/ffdecode.py, which
drives them as `ffmpeg -i F -f s16le -ac 1 -ar 11025 -` does) make of every case of
tests/ffmpeg_frontend_cases.py, read from a WAV and from a FLAC file, and the reference
fingerprint (oracle/afp_oracle.py) of their output for the 30 s songs.  Runs on the CPU; rerunning
it on an x86 CPU with FMA3 gives the same file.

    python oracle/make_golden_ffmpeg_frontend.py
"""
from __future__ import annotations

import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import afp_oracle as orc  # noqa: E402
from oracle import ffdecode  # noqa: E402
from tests import ffmpeg_frontend_cases as FC  # noqa: E402


def library(data, suffix):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "x" + suffix)
        with open(p, "wb") as f:
            f.write(data)
        return ffdecode.decode(p)


def main():
    out = {}
    for name, rate, ch, pcm in FC.cases():
        w = library(FC.wav_bytes(pcm, rate, ch), ".wav")
        if len(pcm) >= 16 * ch:         # FLAC blocks hold at least 16 samples
            assert np.array_equal(w, library(FC.flac_bytes(pcm, rate, ch), ".flac")), name
        out["out_" + name] = w
    for rate, seed in FC.SONGS:
        pcm = FC.song(rate, seed)
        lib = library(FC.wav_bytes(pcm, rate, 2), ".wav")
        out["song_%d_hashes" % rate] = orc.fingerprint(lib.astype(np.float32) / np.float32(32768))
        out["song_%d_head" % rate] = lib[:4096]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ffmpeg_frontend.npz"), **out)


if __name__ == "__main__":
    main()
