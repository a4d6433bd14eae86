"""Golden vectors of the reference's `precompute` and of `new` / `merge` / `match` over precomputed
files, produced by the LIVE reference (dpwe/audfprint) on the PCM committed in
tests/golden/bundled.npz (the query and tracks 0, 4, 8, 12), written as 11025 Hz mono WAVs.

What runs is the reference's own code:
  * audfprint.file_precompute_peaks_or_hashes for every file: hashes at shifts 1 and 4, and peaks
    (the Makefile's `precompdir` / `precomppkdir` targets, Makefile:44-62);
  * audfprint.do_cmd('new') into two tables (two tracks each), HashTable.merge of the first into
    the second, and do_cmd('match') of the query's precomputed file - the sequence of the Makefile's
    `test_onecore_precomp` / `test_onecore_precomppk` scaled down to the four committed tracks, once
    from .afpt and once from .afpk files, with random.seed / np.random.seed fixed;
  * Analyzer.wavfile2hashes of every .afpk file it wrote.
The reader is replaced as in make_golden_bundled.py (here: a WAV parse standing where ffmpeg
stands), and `docopt`, which audfprint.py imports but the functions used never call, is a stub
module.

    AFP_REFERENCE=<checkout> python oracle/make_golden_precompute.py

Stored in tests/golden/precompute.npz: the bytes of every file written, the messages (without the
time.ctime lines), the tables (non-empty buckets, their rows and counts, names, hashesperid), the
`new` summary lines and the `match` report lines.  No reference source is copied.
"""
from __future__ import annotations

import os
import random
import sys
import tempfile
import types
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ["AFP_REFERENCE"]
sys.path.insert(0, REF)
sys.modules.setdefault("docopt", types.ModuleType("docopt"))

import audfprint as ref_cli             # noqa: E402  (the reference)
import audio_read as ref_ar             # noqa: E402
import hash_table as ref_ht             # noqa: E402

from oracle.make_golden_bundled import PCM_TRACKS, make_analyzer, make_matcher   # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "precompute.npz")
BUNDLED = os.path.join(ROOT, "tests", "golden", "bundled.npz")
DENSITY = 100.0                          # the Makefile's --density 100
TABLE = dict(hashbits=20, depth=100, maxtime=16384)   # the command line's defaults


def _reader(filename, sr=None, channels=None):
    """Stands where the reference's ffmpeg pipe stands (audio_read.py:56-99): 16-bit mono WAV."""
    with wave.open(filename, "rb") as w:
        assert w.getnchannels() == 1 and w.getsampwidth() == 2 and w.getframerate() == 11025
        x = np.frombuffer(w.readframes(w.getnframes()), "<i2")
    return x.astype(np.float32) / 32768.0, 11025


ref_ar.audio_read = _reader


def wav_names(gb):
    """Relative names of the WAVs, in the reference's layout: Nine_Lives/<track>.wav and query.wav."""
    names = [str(n) for n in gb["names"]]
    tracks = [os.path.splitext(names[k])[0] + ".wav" for k in PCM_TRACKS]
    return tracks, os.path.splitext(str(gb["query_name"]))[0] + ".wav"


def write_wavs(gb, where):
    tracks, query = wav_names(gb)
    for nm, pcm in list(zip(tracks, [gb["track%d/pcm" % k] for k in PCM_TRACKS])) + [(query, gb["query/pcm"])]:
        fn = os.path.join(where, nm)
        os.makedirs(os.path.dirname(fn) or ".", exist_ok=True)
        with wave.open(fn, "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(11025)
            w.writeframes(np.ascontiguousarray(pcm, np.int16).tobytes())
    return tracks, query


def table_arrays(g, key, ht):
    b = np.nonzero(ht.counts)[0]
    g[key + "/buckets"] = b.astype(np.int32)
    g[key + "/rows"] = np.asarray(ht.table[b], np.uint32)
    g[key + "/counts"] = np.asarray(ht.counts[b], np.int32)
    g[key + "/names"] = np.array(ht.names)
    g[key + "/hashesperid"] = np.asarray(ht.hashesperid, np.uint32)


def main():
    gb = np.load(BUNDLED)
    g = {}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as where:
        os.chdir(where)
        try:
            tracks, query = write_wavs(gb, ".")
            g["tracks"], g["query"] = np.array(tracks), np.array(query)
            # precompute: (kind, shifts) -> precompdir
            runs = (("hashes", 1, "precompdir"), ("hashes", 4, "precompdir_s4"), ("peaks", 1, "precomppkdir"))
            for kind, shifts, pdir in runs:
                an = make_analyzer(DENSITY, shifts)
                key = "%s_s%d" % (kind, shifts)
                msgs, outs = [], []
                for fn in tracks + [query]:
                    m = ref_cli.file_precompute_peaks_or_hashes(an, fn, pdir, hashes_not_peaks=kind == "hashes")
                    msgs += m
                    op = m[0].split(" ")[1]
                    outs.append(op)
                    g["%s/%s" % (key, op)] = np.frombuffer(open(op, "rb").read(), np.uint8)
                    print(m[0])
                g[key + "/msgs"] = np.array(msgs)
                g[key + "/outputs"] = np.array(outs)
            # .afpk -> hashes, as wavfile2hashes forms them
            an = make_analyzer(DENSITY, 1)
            for op in g["peaks_s1/outputs"]:
                g["afpk_hashes/" + str(op)] = np.asarray(an.wavfile2hashes(str(op)), np.int32).reshape(-1, 2)
            # new (two tracks) + new (two tracks) + merge + match, from .afpt and from .afpk files
            for route, pdir, ext in (("precomp", "precompdir", ".afpt"), ("precomppk", "precomppkdir", ".afpk")):
                files = [os.path.join(pdir, os.path.splitext(t)[0] + ext) for t in tracks]
                qfile = os.path.join(pdir if ext == ".afpk" else "precompdir_s4", os.path.splitext(query)[0] + ext)
                random.seed(2015)
                np.random.seed(2015)
                lines = []
                report = lambda msgs: lines.extend(msgs)
                tabs = []
                for part in (files[:2], files[2:]):
                    an = make_analyzer(DENSITY, 1)
                    ht = ref_ht.HashTable(**TABLE)
                    ref_cli.do_cmd("new", an, ht, iter(part), None, None, None, report)
                    tabs.append(ht)
                for k, ht in enumerate(tabs):
                    table_arrays(g, "%s/new%d" % (route, k), ht)
                tabs[1].merge(tabs[0])
                table_arrays(g, route + "/merged", tabs[1])
                g[route + "/new_lines"] = np.array([ln for ln in lines if not ln.endswith(" ...")])
                g[route + "/qfile"] = np.array(qfile)
                an = make_analyzer(DENSITY, 4)        # `match` runs at 4 shifts
                mlines = []
                ref_cli.do_cmd("match", an, tabs[1], iter([qfile]), make_matcher(), None, None,
                               lambda msgs: mlines.extend(msgs))
                g[route + "/match_lines"] = np.array(mlines)
                print(route, lines, mlines)
        finally:
            os.chdir(cwd)
    np.savez_compressed(OUT, **g)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
