"""Timing of FLAC input: device decode alone, and files_match_to_msgs / ingest_files over lists of
FLAC files against the same lists as WAVs.

Audio: one seeded 30 s synthetic track per kind (11025 Hz mono, and 44.1 kHz stereo), written as a
WAV and as a FLAC file (FFmpeg's encoder at its default level through tools/make_golden_flac.py, or
the test bit writer's FIXED-order-2 frames when the FFmpeg libraries are absent), and --files links
to each, so every file is read from the page cache.

  decode     flac.locate + flac.decode_into of --files files in rounds of --round files (device
             events would split it further; this is host wall clock around calls that synchronise),
             reported in audio-seconds per second;
  split      one round of --round files step by step: read (the host parse: _wav_read_raw or
             flac.parse), decode + front-end (_frontend_sources), fingerprint (fingerprint_packed
             with fetch);
  lists      Matcher.files_match_to_msgs (shifts 4, terse) against an empty-ish table of 64 tracks, and
             Analyzer.ingest_files into a fresh table, over --files files, after one warm-up call.

    python tools/flac_timing.py [--files 1000] [--round 256]
"""
import argparse
import contextlib
import io
import os
import sys
import tempfile
import time
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import Analyzer, HashTable, Matcher, _lib, flac  # noqa: E402
from audfprint_b200 import analyzer as an_mod  # noqa: E402
from audfprint_b200.synth import synth_track  # noqa: E402
from tools.long_query_timing import card  # noqa: E402


def encode(pcm, rate):
    try:
        from tools.make_golden_flac import ff_encode
        return ff_encode(pcm, rate, 16), "FFmpeg level 5"
    except Exception:                      # no vendored FFmpeg: the bit writer's frames
        from tests import flac_writer as fw
        return fw.stream(pcm, 16, rate)[0], "bit writer, FIXED order 2"


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=1000)
    ap.add_argument("--round", type=int, default=256)
    args = ap.parse_args()
    print(card())
    mono = synth_track(7, 30.0)
    x44 = np.repeat(mono, 4)                                  # 44.1 kHz by sample repetition
    kinds = {"11025 Hz mono": (mono.reshape(-1, 1), 11025), "44.1 kHz stereo": (np.stack([x44, x44 // 2], 1), 44100)}
    ctx = _lib.context(0)
    tracks = [synth_track(900 + i, 30.0) for i in range(64)]
    ht0 = HashTable(hashbits=20, depth=100, maxtime=16384)
    an0 = Analyzer()
    for i, h in enumerate(an0.fingerprint_batch(tracks)):
        ht0.store("t%d" % i, h)
    with tempfile.TemporaryDirectory() as d:
        for kind, (pcm, rate) in kinds.items():
            data, how = encode(pcm, rate)
            wav, fl = os.path.join(d, "a.wav"), os.path.join(d, "a.flac")
            with wave.open(wav, "wb") as w:
                w.setnchannels(pcm.shape[1])
                w.setsampwidth(2)
                w.setframerate(rate)
                w.writeframes(np.ascontiguousarray(pcm, np.int16).tobytes())
            with open(fl, "wb") as f:
                f.write(data)
            names = {}
            for ext, src in (("wav", wav), ("flac", fl)):
                names[ext] = []
                for i in range(args.files):
                    p = os.path.join(d, "%s_%s_%d" % (kind[:2], ext, i))
                    os.symlink(src, p)
                    names[ext].append(p)
            secs = args.files * 30.0
            print("\n%s: FLAC %.2f MB (%s), WAV %.2f MB per file" % (kind, len(data) / 1e6, how,
                                                                     os.path.getsize(wav) / 1e6))
            # decode alone
            streams = [flac.read(names["flac"][0])] * args.round

            def decode_all():
                import torch
                for s in range(0, args.files, args.round):
                    m = min(args.round, args.files - s)
                    ns, _ = flac.locate(ctx, streams[:m])
                    out = torch.empty(int(ns.sum()) * pcm.shape[1], dtype=torch.int16, device="cuda:0")
                    off = np.concatenate([[0], np.cumsum(ns * pcm.shape[1])[:-1]])
                    with ctx.after_torch(out):
                        flac.decode_into(ctx, out, off)
            decode_all()
            t, _ = timed(decode_all)
            print("decode alone: %.3f s for %d files = %.0f audio-s/s" % (t, args.files, secs / t))
            # split of one round
            an = Analyzer()
            for ext in ("wav", "flac"):
                rnd = names[ext][:args.round]
                tr, raws = timed(lambda: [an_mod._audio_read_raw(fn) for fn in rnd])
                src = [r[0] for r in raws]
                tf, (out, off, lens, _) = timed(lambda: an_mod._frontend_sources(
                    src, [r[1] for r in raws], [r[2] for r in raws], 11025, device=0))
                tp, _ = timed(lambda: an.fingerprint_packed(out, off, 1, sample_lengths=lens))
                print("round of %d %s: read %.1f ms, decode + front-end %.1f ms, fingerprint %.1f ms" % (
                    len(rnd), ext.upper(), tr * 1e3, tf * 1e3, tp * 1e3))
            # list forms
            for ext in ("wav", "flac"):
                an = Analyzer()
                an.shifts = 4
                mt = Matcher()
                mt.verbose = False

                def match():
                    with contextlib.redirect_stdout(io.StringIO()):
                        return mt.files_match_to_msgs(an, ht0, names[ext])
                match()
                tm, _ = timed(match)
                ai = Analyzer()

                def ingest():
                    ht = HashTable(hashbits=20, depth=100, maxtime=16384)
                    return ai.ingest_files(ht, names[ext])
                ingest()
                ti, _ = timed(ingest)
                print("%s x %d: files_match_to_msgs %.2f s (%.0f audio-s/s), ingest_files %.2f s (%.0f audio-s/s)" % (
                    ext.upper(), args.files, tm, secs / tm, ti, secs / ti))


if __name__ == "__main__":
    main()
