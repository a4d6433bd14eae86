"""How often does the opt-in FP32 spectrogram mode (Analyzer.precision = 'fp32') change a file's
hashes relative to the FP64 (reference-identical) path?  VERDICT r1 #6(b) asked for a study on
>= 1e5 files incl. the adversarial cases.  Tracks: seeds 2,000,000.. of the bench generator at
5 lengths, plus the adversarial inputs of tests/cases.py.  Writes profiles/r02_fp32_flip_study.json."""
import json, os, sys, time, multiprocessing as mp
import numpy as np
ROOT = __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__)))
sys.path.insert(0, ROOT)
from audfprint_b200.synth import synth_track
from tests import cases

def gen(args):
    seed, secs = args
    return synth_track(2_000_000 + seed, secs)

def main(total=100_000, chunk=4096):
    pool = mp.get_context("fork").Pool(int(sys.argv[1]) if len(sys.argv) > 1 else 16)
    from audfprint_b200 import Analyzer
    a64, a32 = Analyzer(), Analyzer()
    a32.precision = 'fp32'
    lens = [10.0, 20.0, 30.0, 45.0, 60.0]
    nfiles = nhash = ndiff_files = nsym = 0
    audio = 0.0
    t0 = time.time()
    worst = []
    for c0 in range(0, total, chunk):
        n = min(chunk, total - c0)
        sigs = pool.map(gen, [(c0 + i, lens[(c0 + i) % len(lens)]) for i in range(n)], chunksize=16)
        h64 = a64.fingerprint_batch(sigs)
        h32 = a32.fingerprint_batch(sigs)
        for i, (x, y) in enumerate(zip(h64, h32)):
            nfiles += 1; nhash += len(x); audio += len(sigs[i]) / 11025.0
            if not np.array_equal(x, y):
                ndiff_files += 1
                sx, sy = set(map(tuple, x.tolist())), set(map(tuple, y.tolist()))
                d = len(sx ^ sy); nsym += d
                worst.append((d, c0 + i))
    adv = {}
    for name in cases.ADVERSARIAL:
        pcm = cases.adversarial_pcm(name)
        x, y = a64.fingerprint_batch([pcm])[0], a32.fingerprint_batch([pcm])[0]
        adv[name] = {"hashes_fp64": int(len(x)), "identical": bool(np.array_equal(x, y))}
    out = {"files": nfiles, "audio_seconds": audio, "hashes_fp64": nhash, "files_with_any_difference": ndiff_files,
           "file_flip_rate": ndiff_files / max(1, nfiles), "hashes_in_symmetric_difference": nsym,
           "hash_flip_rate": nsym / max(1, nhash), "worst_files": sorted(worst, reverse=True)[:10],
           "adversarial": adv, "wall_s": time.time() - t0,
           "note": "FP32 STFT + MUFU log + float spectrogram (K1), K2 thresholds in FP64 either way"}
    os.makedirs(ROOT + '/profiles', exist_ok=True)
    json.dump(out, open(ROOT + '/profiles/r02_fp32_flip_study.json', 'w'), indent=1)
    print(json.dumps({k: out[k] for k in ("files", "files_with_any_difference", "file_flip_rate", "hash_flip_rate", "wall_s")}))
    print(adv)

if __name__ == "__main__":
    main()
