"""SHA-256 digests of the conditioned spectrogram (Analyzer.conditioned_sgram, the afp_sgram entry
point: K1's logs, then the per-file floor and mean, then the high-pass) in FP64 and FP32 modes.

Inputs: the first 64 files of the bench batch (synth_track(seed, 30 s), seeds 0..63, as bench.py
generates them) and the adversarial cases of tests/cases.py (digital silence, a file whose floor
bites, files shorter than one frame, ragged lengths).  Two builds of K1 that compute the same
spectrogram print the same lines; run it on each and diff the output.

    python tools/k1_digest.py [--files N]
"""
import argparse
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from audfprint_b200 import Analyzer  # noqa: E402
from audfprint_b200.synth import synth_track  # noqa: E402
from tests import cases  # noqa: E402


def digest(an, signals):
    h = hashlib.sha256()
    for x in signals:
        s = np.ascontiguousarray(an.conditioned_sgram(x), np.float64)
        h.update(np.int64(s.shape[1]).tobytes())
        h.update(s.tobytes())
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=64, help="bench files (seeds 0..N-1, 30 s each)")
    a = ap.parse_args()
    bench = [synth_track(i, 30.0) for i in range(a.files)]
    adv = [(name, cases.adversarial_pcm(name)) for name in cases.ADVERSARIAL]
    for precision in ("fp64", "fp32"):
        an = Analyzer()
        an.precision = precision
        print("%s bench[0:%d] %s" % (precision, a.files, digest(an, bench)))
        for name, x in adv:
            print("%s %s %s" % (precision, name, digest(an, [x])))


if __name__ == "__main__":
    main()
