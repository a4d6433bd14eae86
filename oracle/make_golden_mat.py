"""A Matlab-audfprint style .mat database and what the LIVE reference makes of it
(hash_table.py:248-285).  The .mat is written here with scipy.io.savemat in the layout the
reference's loader indexes (HT_params struct, HashTable depth x buckets, cell array of names);
tests/golden/matlab_db_arrays.npz holds the attributes of the reference object after loading it.

Needs a checkout of the reference (dpwe/audfprint) named by $AFP_REFERENCE:
    AFP_REFERENCE=<checkout> python oracle/make_golden_mat.py
"""
from __future__ import annotations

import os
import sys

import numpy as np
import scipy.io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["AFP_REFERENCE"])

import hash_table as ref_ht             # noqa: E402  (the reference)

OUT = os.path.join(ROOT, "tests", "golden")


def main():
    rng = np.random.default_rng(31)
    nbuckets, depth, maxtime, ntracks = 256, 4, 1024, 5
    counts = rng.integers(0, depth + 3, nbuckets).astype(np.int32)
    table = np.zeros((nbuckets, depth), np.uint32)
    for b in range(nbuckets):
        n = min(depth, counts[b])
        # Matlab ids are 1-based and stored as-is (the Python table also stores id + 1)
        table[b, :n] = (rng.integers(1, ntracks + 1, n) * maxtime + rng.integers(0, maxtime, n)).astype(np.uint32)
    names = np.empty((1, ntracks), dtype=object)
    for i in range(ntracks):
        names[0, i] = "mat_track_%d.mp3" % i
    names[0, 3] = np.zeros((0,), dtype="U1")           # a deleted entry: empty cell
    mat = {
        "HT_params": {"nhashes": float(nbuckets), "depth": float(depth), "maxtime": float(maxtime),
                      "hoptime": 0.02322, "targetsr": 11025.0, "nojenkins": 1.0, "version": 0.9},
        "HashTable": table.T.copy(),
        "HashTableCounts": counts.reshape(1, -1),
        "HashTableNames": names,
        "HashTableLengths": rng.integers(50, 900, (1, ntracks)).astype(np.float64),
    }
    fn = os.path.join(OUT, "matlab_db.mat")
    scipy.io.savemat(fn, mat)
    ht = ref_ht.HashTable(fn)
    np.savez_compressed(os.path.join(OUT, "matlab_db_arrays.npz"), table=ht.table, counts=ht.counts,
                        hashesperid=ht.hashesperid, names=np.array([n if isinstance(n, str) else "" for n in ht.names]),
                        geometry=np.array([ht.hashbits, ht.depth, ht.maxtimebits]),
                        params=np.array([ht.params["mat_version"], ht.params["hoptime"], ht.params["targetsr"],
                                         ht.params["nojenkins"]], np.float64))
    print("reference loaded:", ht.hashbits, ht.depth, ht.maxtimebits, ht.names, ht.params)


if __name__ == "__main__":
    main()
