"""Write tests/golden/wide_pcm.npz: what FFmpeg 8.0's libraries (oracle/ffdecode.py, which drives them as
`ffmpeg -i F -f s16le -ac 1 -ar 11025 -` does) make of every case of tests/wide_pcm_cases.py - 24-bit,
32-bit and float WAV, plain and WAVE_FORMAT_EXTENSIBLE, 20- and 24-bit FLAC, float specials and the RIFF
chunk cases - and the reference fingerprint (oracle/afp_oracle.py) of their output for the two 30 s
songs.  Runs on the CPU; rerunning it on an x86 CPU with FMA3 gives the same file.

    python oracle/make_golden_wide_pcm.py
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
from tests import wide_pcm_cases as WC  # noqa: E402


def library(data, suffix):
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "x" + suffix)
        with open(p, "wb") as f:
            f.write(data)
        return ffdecode.decode(p)


def main():
    out = {}
    for name, src, _, _, data, _, _ in WC.cases():
        WC.store(out, "out_" + name, library(data, "." + src))
    for name, data, _, _, _ in WC.chunk_cases():
        out["chunk_" + name] = library(data, ".wav")
    for name, rate, fmt in WC.SONGS:
        data = WC.song(rate, fmt)[0]
        lib = library(data, ".wav")
        out[name + "_hashes"] = orc.fingerprint(lib.astype(np.float32) / np.float32(32768))
        out[name + "_head"] = lib[:4096]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "wide_pcm.npz"), **out)


if __name__ == "__main__":
    main()
