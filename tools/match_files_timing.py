"""Timing of matching a list of audio files: the per-file loop the reference's `match` runs
(Matcher.file_match_to_msgs per file) next to the list form (Matcher.files_match_to_msgs: batched
front-end, fingerprint and match per round of files).

Queries: seeded 10 s noisy excerpts of 64 synthetic 30 s tracks (BASELINE configs[2]-style),
written as 11025 Hz mono WAVs and as 44.1 kHz stereo WAVs into a temporary directory, against
bench.py's 2^20 x 100 table with 1 M ids, every bucket full.  --files distinct files of each kind are
written; longer lists repeat them (the files are in the page cache either way).  Matcher: window 2,
terse report lines, shifts 4.

Times are host wall clock around whole calls (each ends in a stream synchronise): the loop on the
first --sample files, reported per file; the list form at each --lists length after one warm-up
call at the same length (the first call at a length, which grows the device buffers, is reported
beside it).  The split of the list form (1,000 files) times its steps one after the other on the same
data: read (_wav_read_raw), front-end (pcm_frontend_batch), fingerprint (fingerprint_packed and
the fetch of the hashes into device memory), match (match_batch), format (the report lines).

    python tools/match_files_timing.py [--files 1000] [--sample 100] [--lists 1000,10000]
"""
import argparse
import os
import sys
import tempfile
import time
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from audfprint_b200 import Analyzer, HashTable, Matcher  # noqa: E402
from audfprint_b200 import analyzer as an_mod  # noqa: E402
from audfprint_b200.synth import synth_query, synth_track  # noqa: E402
from tools.long_query_timing import card  # noqa: E402


def write_wav(fn, pcm, nch, fs):
    with wave.open(fn, "wb") as w:
        w.setnchannels(nch)
        w.setsampwidth(2)
        w.setframerate(fs)
        w.writeframes(np.ascontiguousarray(pcm, np.int16).tobytes())


def make_table(tracks):
    an = Analyzer()
    th = an.fingerprint_batch(tracks)
    rows = np.concatenate(th)
    roff = np.concatenate([[0], np.cumsum([len(h) for h in th])]).astype(np.int64)
    table, counts, hashbits, depth, mtb, hpi, _ = bench.build_big_table(rows, roff, 1000000)
    ht = HashTable(hashbits=hashbits, depth=1, maxtime=1 << mtb)
    ht.table, ht.counts, ht.hashesperid, ht.depth = table, counts, hpi, depth
    ht.names = ["track%07d" % i for i in range(1000000)]
    return ht


def write_queries(d, tracks, n):
    from scipy.signal import resample_poly
    mono, stereo = [], []
    for j in range(n):
        q = synth_query(tracks[j % len(tracks)], j, seconds=10.0, noise_sigma=0.02)[0]
        fn = os.path.join(d, "q%05d.wav" % j)
        write_wav(fn, q, 1, 11025)
        mono.append(fn)
        x = np.round(resample_poly(q.astype(np.float64), 4, 1)).clip(-32768, 32767).astype(np.int16)
        fn = os.path.join(d, "q%05d_44k.wav" % j)
        write_wav(fn, np.stack([x, x // 2], axis=1), 2, 44100)
        stereo.append(fn)
    return mono, stereo


def analyzer():
    an = Analyzer()
    an.shifts = 4
    return an


def matcher():
    m = Matcher()
    m.window = 2
    return m


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def split(ht, names):
    """The list form's steps one after the other, in rounds of 256 files."""
    import torch
    an, mt = analyzer(), matcher()
    ts = dict(read=0.0, frontend=0.0, fingerprint=0.0, match=0.0, format=0.0)
    for c0 in range(0, len(names), 256):
        chunk = names[c0:c0 + 256]
        t, raws = timed(lambda: [an_mod._wav_read_raw(fn) for fn in chunk])
        ts["read"] += t
        t, (out, off, lens) = timed(lambda: an_mod.pcm_frontend_batch(
            [r[0] for r in raws], [r[1] for r in raws], [r[2] for r in raws], 11025))
        ts["frontend"] += t
        t0 = time.perf_counter()
        an.fingerprint_packed(out, off, 4, fetch=False, sample_lengths=lens)
        ctx = an_mod._lib.context()
        import ctypes as C
        roff = np.empty(len(chunk) + 1, np.int64)
        ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, roff.ctypes.data_as(C.POINTER(C.c_int64))))
        rows = torch.empty((max(int(roff[-1]), 1), 2), dtype=torch.int32, device=out.device)
        torch.cuda.current_stream(out.device).synchronize()          # the library writes it on its own stream
        ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, C.c_void_p(rows.data_ptr()), 0, None))
        ts["fingerprint"] += time.perf_counter() - t0
        t, res = timed(lambda: mt.match_batch(ht, (rows[:int(roff[-1])], roff)))
        ts["match"] += t
        t, _ = timed(lambda: [mt._msgs(an, ht, fn, r[:1], 0.0, 0) for fn, r in zip(chunk, res)])
        ts["format"] += t
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=1000)
    ap.add_argument("--sample", type=int, default=100)
    ap.add_argument("--lists", default="1000,10000")
    args = ap.parse_args()
    card()
    tracks = [synth_track(9000 + i, 30.0) for i in range(64)]
    ht = make_table(tracks)
    with tempfile.TemporaryDirectory() as d:
        mono, stereo = write_queries(d, tracks, args.files)
        print("table 2^20 x 100, 1 M ids; %d distinct 10 s queries of each kind" % args.files)
        for kind, files in (("11025 Hz mono", mono), ("44.1 kHz stereo", stereo)):
            mt = matcher()
            mt.files_match_to_msgs(analyzer(), ht, files[:8])           # warm-up: every shape, the table upload
            [mt.file_match_to_msgs(analyzer(), ht, fn) for fn in files[:4]]
            an = analyzer()
            t, want = timed(lambda: [mt.file_match_to_msgs(an, ht, fn, i) for i, fn in enumerate(files[:args.sample])])
            loop_ms = 1e3 * t / args.sample
            print("%s: per-file loop %.2f ms per file (first %d files)" % (kind, loop_ms, args.sample))
            for n in [int(x) for x in args.lists.split(",")]:
                names = [files[i % len(files)] for i in range(n)]
                # the first call at a size grows the device buffers (workspace, staging, torch's cache)
                t0, _ = timed(lambda: mt.files_match_to_msgs(analyzer(), ht, names))
                t, got = timed(lambda: mt.files_match_to_msgs(analyzer(), ht, names))
                assert got[:args.sample] == want
                print("  list form, %6d files: %8.1f ms, %7.3f ms per file, %.1f x the loop "
                      "(first call at this size: %.1f ms)" % (n, 1e3 * t, 1e3 * t / n, loop_ms / (1e3 * t / n), 1e3 * t0))
            ts = split(ht, files[:1000])
            print("  split over %d files: " % min(1000, len(files)) +
                  ", ".join("%s %.1f ms" % (k, 1e3 * v) for k, v in ts.items()))


if __name__ == "__main__":
    main()
