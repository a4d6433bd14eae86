"""tests/golden/live_reference.npz: what the reference (dpwe/audfprint) computes on seeds and
parameter settings that the other golden files do not cover.  tests/test_oracle_live_reference.py
compares the oracle with these outputs.

Needs a checkout of the reference (dpwe/audfprint) named by $AFP_REFERENCE:
    AFP_REFERENCE=<checkout> python -m oracle.make_golden_live

Each driver runs the reference in a subprocess, so that its module names (hash_table, ...) never
enter this process, and prints its outputs as one JSON line."""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "live_reference.npz")

SEEDS = [5101, 5102, 5103, 5104]
# (density, fanout, shifts, f_sd, maxpksperframe) and (window, threshcount, search_depth,
# max_alignments_per_id): the settings the GPU tests check against the oracle only
ANALYZER_PARAMS = [(20.0, 3, 2, 30.0, 5), (20.0, 3, 3, 30.0, 5), (20.0, 3, 8, 30.0, 5), (35.0, 5, 1, 20.0, 3),
                   (50.0, 6, 4, 30.0, 8), (10.0, 1, 1, 45.0, 1), (70.0, 8, 1, 30.0, 16)]
MATCHER_PARAMS = [(0, 5, 100, 100), (3, 0, 5, 100), (1, 5, 1, 100), (2, 1, 100, 0), (2, 5, 0, 100), (1, 2, 3, 1)]
SPREAD_CASES = [(256, 4.0), (256, 30.0), (64, 2.5), (17, 1.0), (300, 12.0), (1, 4.0)]

SEEDS_DRIVER = r'''
import json, random, sys
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(ref)r)
import audfprint_analyze as an, audfprint_match as ma, audio_read as ar, hash_table as htm
from audfprint_b200.synth import synth_track, synth_query, pcm_to_float
pcm = {}
ar.audio_read = lambda fn, sr=None, channels=None: (pcm_to_float(pcm[fn]), 11025)
out = {}
tracks = []
for seed in %(seeds)r:
    pcm["t"] = synth_track(seed, 14.0 + seed %% 5)
    for shifts in (1, 4):
        a = an.Analyzer(); a.shifts = shifts
        out["h_%%d_%%d" %% (seed, shifts)] = np.asarray(a.wavfile2hashes("t")).tolist()
    tracks.append(np.asarray(out["h_%%d_1" %% seed], np.int32))
random.seed(4)
ht = htm.HashTable(hashbits=14, depth=6, maxtime=1 << 12)
for i, h in enumerate(tracks):
    ht.store("s%%d" %% i, h)
m = ma.Matcher(); m.window = 2; m.threshcount = 3; m.search_depth = 4
for j, seed in enumerate(%(seeds)r):
    q, _ = synth_query(synth_track(seed, 14.0 + seed %% 5), 77 + j, seconds=6.0, noise_sigma=0.01)
    pcm["q"] = q
    a = an.Analyzer(); a.shifts = 4
    qh = np.asarray(a.wavfile2hashes("q"), np.int32)
    out["q_%%d" %% seed] = qh.tolist()
    out["hits_%%d" %% seed] = ht.get_hits(qh).tolist()
    out["rows_%%d" %% seed] = m.match_hashes(ht, qh).tolist()
out["table"] = ht.table.tolist(); out["counts"] = ht.counts.tolist(); out["hpi"] = np.asarray(ht.hashesperid).tolist()
print("JSON" + json.dumps(out))
'''

PARAM_DRIVER = r'''
import json, random, sys
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, %(ref)r)
import audfprint_analyze as an, audfprint_match as ma, audio_read as ar, hash_table as htm
from audfprint_b200.synth import synth_track, synth_query, pcm_to_float
pcm = {}
ar.audio_read = lambda fn, sr=None, channels=None: (pcm_to_float(pcm[fn]), 11025)
out = {}
for k, (density, fanout, shifts, f_sd, maxpks) in enumerate(%(aparams)r):
    for i in range(2):
        pcm["t"] = synth_track(6000 + 10 * k + i, 9.0 + i)
        a = an.Analyzer(density)
        a.maxpairsperpeak, a.shifts, a.f_sd, a.maxpksperframe = fanout, shifts, f_sd, maxpks
        out["h_%%d_%%d" %% (k, i)] = np.asarray(a.wavfile2hashes("t")).reshape(-1, 2).tolist()
        if shifts == 1:
            out["p_%%d_%%d" %% (k, i)] = np.asarray(a.wavfile2peaks("t")).reshape(-1, 2).tolist()
# matcher parameters on a small overflowing table
random.seed(9)
ht = htm.HashTable(hashbits=12, depth=8, maxtime=1 << 14)
trk = [synth_track(6500 + i, 12.0) for i in range(12)]
for i, t in enumerate(trk):
    pcm["t"] = t
    ht.store("s%%d" %% i, an.Analyzer().wavfile2hashes("t"))
out["table"] = ht.table.tolist(); out["counts"] = ht.counts.tolist(); out["hpi"] = np.asarray(ht.hashesperid).tolist()
qs = []
for j in range(4):
    q, _ = synth_query(trk[3 * j], 900 + j, seconds=7.0, noise_sigma=0.01)
    pcm["q"] = q
    a = an.Analyzer(); a.shifts = 4
    qs.append(np.asarray(a.wavfile2hashes("q"), np.int32).reshape(-1, 2))
    out["q_%%d" %% j] = qs[-1].tolist()
for k, (window, thresh, sdepth, maxal) in enumerate(%(mparams)r):
    m = ma.Matcher()
    m.window, m.threshcount, m.search_depth, m.max_alignments_per_id = window, thresh, sdepth, maxal
    for j, qh in enumerate(qs):
        out["rows_%%d_%%d" %% (k, j)] = np.asarray(m.match_hashes(ht, qh)).reshape(-1, 7).tolist()
print("JSON" + json.dumps(out))
'''

SPREAD_DRIVER = r'''
import json, sys
import numpy as np
sys.path.insert(0, %(ref)r)
import audfprint_analyze as an
rng = np.random.default_rng(12)
out = []
for n, width in %(cases)r:
    v = rng.standard_normal(n) * 3
    v[rng.integers(0, n, max(1, n // 9))] = 2.0          # plateaus / equal neighbours
    out.append([n, width, v.tolist(), an.Analyzer().spreadpeaksinvector(v, width).tolist()])
print("JSON" + json.dumps(out))
'''


def _run(code):
    run = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    if run.returncode != 0:
        raise RuntimeError(run.stderr[-2000:])
    return json.loads([ln for ln in run.stdout.splitlines() if ln.startswith("JSON")][0][4:])


def main(ref):
    out = {}
    seeds = _run(SEEDS_DRIVER % {"root": ROOT, "ref": ref, "seeds": SEEDS})
    params = _run(PARAM_DRIVER % {"root": ROOT, "ref": ref, "aparams": ANALYZER_PARAMS, "mparams": MATCHER_PARAMS})
    for prefix, d in (("seeds/", seeds), ("params/", params)):
        for k, v in d.items():
            dt = np.uint32 if k == "table" else np.int32
            out[prefix + k] = np.array(v, dt)
    for i, (n, width, v, want) in enumerate(_run(SPREAD_DRIVER % {"ref": ref, "cases": SPREAD_CASES})):
        out["spread/%d/in" % i] = np.array(v, np.float64)
        out["spread/%d/out" % i] = np.array(want, np.float64)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays)" % (OUT, len(out)))


if __name__ == "__main__":
    main(os.path.abspath(os.environ["AFP_REFERENCE"]))
