"""Timing of the reference's `new` / `add` and `precompute` over a file list: each per-file loop next
to its list form.

  ingest       Analyzer.ingest per file            vs  Analyzer.ingest_files
  precompute   precompute_file per file (hashes)   vs  precompute_files, at shifts 1 and 4
  peaks (-K)   precompute_file per file (peaks)    vs  precompute_files(type='peaks')
  .afpk table  Analyzer.ingest per .afpk file      vs  Analyzer.ingest_files of the .afpk files

Input: --files distinct seeded synthetic tracks of --seconds each, written as 11025 Hz mono WAVs and
as the same audio at 44.1 kHz stereo into a temporary directory; tables are 2^20 x 100.  Every pair
is warmed up on a few files of the same shape first (device buffers, table upload).  Times are host
wall clock around whole calls; the loop runs on the first --sample files and is reported per file,
the list form on all --files.  The split of the list-form ingest times its steps one after the other
on the same data, in rounds of 256 files: read (_wav_read_raw), front-end (pcm_frontend_batch),
fingerprint (fingerprint_packed + synchronise), store (store_batch from the workspace), and for
precompute the write of the hashes (fetch + files).  The card's name and power limit are printed
first, in the same run.

    python tools/ingest_precompute_timing.py [--files 1000] [--seconds 60] [--sample 100]
"""
import argparse
import contextlib
import ctypes as C
import io
import os
import random
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import Analyzer, HashTable  # noqa: E402
from audfprint_b200 import analyzer as an_mod  # noqa: E402
from audfprint_b200.synth import synth_track  # noqa: E402
from tools.long_query_timing import card  # noqa: E402
from tools.match_files_timing import write_wav  # noqa: E402


def write_inputs(d, n, seconds):
    from scipy.signal import resample_poly
    mono, stereo = [], []
    for j in range(n):
        x = synth_track(20000 + j, seconds)
        fn = os.path.join(d, "wav", "t%05d.wav" % j)
        os.makedirs(os.path.dirname(fn), exist_ok=True)
        write_wav(fn, x, 1, 11025)
        mono.append(fn)
        y = np.round(resample_poly(x.astype(np.float64), 4, 1)).clip(-32768, 32767).astype(np.int16)
        fn = os.path.join(d, "wav44", "t%05d.wav" % j)
        os.makedirs(os.path.dirname(fn), exist_ok=True)
        write_wav(fn, np.stack([y, y // 2], axis=1), 2, 44100)
        stereo.append(fn)
    return mono, stereo


def timed(fn):
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        out = fn()
    return time.perf_counter() - t0, out


def analyzer(shifts=1):
    an = Analyzer()
    an.shifts = shifts
    return an


def table():
    random.seed(1)
    return HashTable(hashbits=20, depth=100, maxtime=16384)


def _ingest_loop(files):
    an, ht = analyzer(), table()
    return [an.ingest(ht, f) for f in files]


def pair(label, loop, listed, files, sample):
    timed(lambda: loop(files[:2]))
    timed(lambda: listed(files[:8]))                            # warm-up of this shape
    t_loop, _ = timed(lambda: loop(files[:sample]))
    t_list, _ = timed(lambda: listed(files))
    per_loop, per_list = 1e3 * t_loop / sample, 1e3 * t_list / len(files)
    print("  %-34s loop %7.2f ms / file   list %7.2f ms / file (%d files)   %.1fx"
          % (label, per_loop, per_list, len(files), per_loop / per_list))


def split(files, outdir):
    """The list-form ingest's steps (and a precompute write) one after the other, rounds of 256."""
    an = analyzer()
    ht = table()
    ctx = an_mod._lib.context()
    ts = dict(read=0.0, frontend=0.0, fingerprint=0.0, store=0.0, write=0.0)
    for c0 in range(0, len(files), 256):
        chunk = files[c0:c0 + 256]
        t, raws = timed(lambda: [an_mod._wav_read_raw(fn) for fn in chunk])
        ts["read"] += t
        t, (out, off, lens) = timed(lambda: an_mod.pcm_frontend_batch(
            [r[0] for r in raws], [r[1] for r in raws], [r[2] for r in raws], 11025))
        ts["frontend"] += t
        t, _ = timed(lambda: (an.fingerprint_packed(out, off, 1, fetch=False, sample_lengths=lens), ctx.sync()))
        ts["fingerprint"] += t
        t0 = time.perf_counter()
        roff = np.empty(len(chunk) + 1, np.int64)
        ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, roff.ctypes.data_as(C.POINTER(C.c_int64))))
        rows = np.empty((int(roff[-1]), 2), np.int32)
        ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, rows.ctypes.data, 1, None))
        for k, fn in enumerate(chunk):
            an_mod._precompute_write(fn, an_mod.precompute_name(fn, outdir), True, rows[roff[k]:roff[k + 1]], 0.0)
        ts["write"] += time.perf_counter() - t0
        t, _ = timed(lambda: ht.store_batch(chunk, None))
        ts["store"] += t
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=1000)
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--sample", type=int, default=100)
    args = ap.parse_args()
    card()
    with tempfile.TemporaryDirectory() as d:
        mono, stereo = write_inputs(d, args.files, args.seconds)
        print("%d distinct %.0f s files of each kind; tables 2^20 x 100" % (args.files, args.seconds))
        out = os.path.join(d, "out")

        def fresh():
            shutil.rmtree(out, ignore_errors=True)
            return out

        for kind, files in (("11025 Hz mono", mono), ("44.1 kHz stereo", stereo)):
            print(kind)
            pair("ingest vs ingest_files", _ingest_loop, lambda fs: analyzer().ingest_files(table(), fs), files,
                 args.sample)
            for shifts in (1, 4):
                pair("precompute hashes, shifts %d" % shifts,
                     lambda fs: (lambda o: [analyzer(shifts).precompute_file(f, o) for f in fs])(fresh()),
                     lambda fs: analyzer(shifts).precompute_files(fs, fresh()), files, args.sample)
            pair("precompute peaks (-K)",
                 lambda fs: (lambda o: [analyzer().precompute_file(f, o, type="peaks") for f in fs])(fresh()),
                 lambda fs: analyzer().precompute_files(fs, fresh(), type="peaks"), files, args.sample)
            ts = split(files, fresh())
            print("  split of the list form over %d files: " % len(files) +
                  ", ".join("%s %.1f ms" % (k, 1e3 * v) for k, v in ts.items()))
        # the .afpk -> table route, from the mono files' peaks
        pk = os.path.join(d, "pk")
        with contextlib.redirect_stdout(io.StringIO()):
            analyzer().precompute_files(mono, pk, type="peaks")
        afpk = [an_mod.precompute_name(f, pk, False) for f in mono]
        print(".afpk files")
        pair(".afpk -> table", _ingest_loop, lambda fs: analyzer().ingest_files(table(), fs), afpk, args.sample)


if __name__ == "__main__":
    main()
