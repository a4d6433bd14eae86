"""Golden vectors at the geometry of BASELINE configs[2] / configs[3] (VERDICT r1 "What's weak" #2):
180 s tracks (T = 7752 frames) through the LIVE reference, and a table with maxtimebits=12 whose
stored times alias (180 s > 2^12 frames = 95 s) built by the reference's own `store`, queried by
the reference's own `match_hashes`.

Needs a checkout of the reference (dpwe/audfprint) named by $AFP_REFERENCE:
    AFP_REFERENCE=<checkout> python oracle/make_golden_long.py
Stores only OUTPUT arrays of the reference in tests/golden/long.npz.
"""
from __future__ import annotations

import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ["AFP_REFERENCE"]
sys.path.insert(0, REF)

import audfprint_analyze as ref_an      # noqa: E402
import audfprint_match as ref_ma        # noqa: E402
import audio_read as ref_ar             # noqa: E402
import hash_table as ref_ht             # noqa: E402

from audfprint_b200.synth import synth_track, synth_query, pcm_to_float     # noqa: E402
from tests import cases                                                     # noqa: E402

_PCM = {}
ref_ar.audio_read = lambda filename, sr=None, channels=None: (pcm_to_float(_PCM[filename]), 11025)


def file_hashes(pcm, shifts):
    an = ref_an.Analyzer(20.0)
    an.shifts = shifts
    _PCM["x"] = pcm
    return np.asarray(an.wavfile2hashes("x"), dtype=np.int32).reshape(-1, 2)


def main():
    g = {}
    # ---- 180 s tracks, the configs[3] file length: shifts 1 for every seed, shifts 4 for one
    tracks = []
    for seed in cases.LONG_SEEDS:
        pcm = synth_track(seed, cases.LONG_SECONDS)
        h1 = file_hashes(pcm, 1)
        tracks.append(h1)
        g["t%d/wf2h_s1" % seed] = h1
        print("180 s seed", seed, "hashes", len(h1), "last time", int(h1[-1, 0]))
    g["t%d/wf2h_s4" % cases.LONG_SEEDS[0]] = file_hashes(synth_track(cases.LONG_SEEDS[0], cases.LONG_SECONDS), 4)
    # ---- a maxtimebits=12 table of those tracks (times alias mod 4096), reference store + match
    random.seed(4321)
    ht = ref_ht.HashTable(hashbits=cases.LONG_HASHBITS, depth=cases.LONG_DEPTH, maxtime=1 << cases.LONG_MAXTIMEBITS)
    for seed, h in zip(cases.LONG_SEEDS, tracks):
        ht.store("long%d" % seed, h)
    nz = np.nonzero(ht.counts)[0]
    g["db/params"] = np.array([cases.LONG_HASHBITS, cases.LONG_DEPTH, cases.LONG_MAXTIMEBITS], np.int32)
    g["db/buckets"] = nz.astype(np.int32)
    g["db/counts"] = ht.counts[nz]
    g["db/rows"] = ht.table[nz]
    g["db/hashesperid"] = np.asarray(ht.hashesperid)
    print("table: buckets", len(nz), "overfull", int(np.sum(ht.counts > ht.depth)))
    mt = ref_ma.Matcher()
    mt.window, mt.threshcount, mt.search_depth = 2, 5, 100
    for j, (k, secs) in enumerate(cases.LONG_QUERIES):
        pcm, off = synth_query(synth_track(cases.LONG_SEEDS[k], cases.LONG_SECONDS), 7000 + j, seconds=secs,
                               noise_sigma=0.01)
        q = file_hashes(pcm, 4)
        rows = mt.match_hashes(ht, q)
        hits = ht.get_hits(q)
        ids, raw = np.unique(hits[:, 0], return_counts=True)
        wtd = raw / ht.hashesperid[ids].astype(float)
        dep = min(int(np.count_nonzero(raw > 5)), 100)
        srt = np.sort(wtd)[::-1][:dep + 1]
        g["q%d/q" % j] = q
        g["q%d/rows" % j] = rows
        g["q%d/truth" % j] = np.array([k, off], np.int64)
        g["q%d/ties" % j] = np.array([bool(dep and np.any(srt[:-1] == srt[1:])),
                                      bool(len(np.unique(rows[:, 1])) != len(rows))])
        print("query", j, "track", k, "secs", secs, "nq", len(q), "rows", rows[:2].tolist(),
              "true dt", off // 256, "aliased", (off // 256) % (1 << cases.LONG_MAXTIMEBITS), g["q%d/ties" % j])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "long.npz"), **g)


if __name__ == "__main__":
    main()
