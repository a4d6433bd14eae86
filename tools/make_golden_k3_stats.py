"""Writes tests/golden/k3_stats.npz: the outputs the item statistics feed, for the mixed batch of
tests/test_gpu_k3_stats.py (stats_files), from a build of the project given by --root.

The fixture was recorded from the commit before the per-file K3 and the flagged-item statistics, so
that the test holds the new kernels to the three-launch statistics path and the landmark / merge K3
bit for bit: for fp64 and fp32 and shifts 1 and 4, every file's hashes in the batch, and the sha256 of
every file's conditioned spectrogram.  Needs a GPU.

    python tools/make_golden_k3_stats.py --root CHECKOUT --out tests/golden/k3_stats.npz
"""
import argparse
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--root", required=True, help="checkout whose library (built) computes the outputs")
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.root))
    spec = importlib.util.spec_from_file_location("k3_stats_cases", os.path.join(HERE, "tests", "test_gpu_k3_stats.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = {}
    for precision in ("fp64", "fp32"):
        for shifts in (1, 4):
            names, hashes, sg = mod.stats_outputs(precision, shifts)
            for name, h, d in zip(names, hashes, sg):
                out["%s_s%d_%s_hashes" % (precision, shifts, name)] = np.asarray(h, np.int32)
                out["%s_%s_sgram" % (precision, name)] = np.array(d)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    np.savez_compressed(a.out, **out)
    print("wrote", a.out, "from", os.path.abspath(a.root), {k: v.shape for k, v in out.items() if k.endswith("hashes")})


if __name__ == "__main__":
    main()
