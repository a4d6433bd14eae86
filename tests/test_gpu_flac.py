"""FLAC decoding on the device (afp_flac_locate_batch / afp_flac_decode_batch) and FLAC files through
every file entry point.

- Every fixture of tests/golden/flac.npz (FFmpeg-encoded and bit-writer files) decodes to FFmpeg's
  decode bit for bit, in one batched call and through the per-file reader; each damaged file gets its
  status, and nothing outside the good files' output ranges is written.
- 4,096 short files decode in one call.
- Device-resident input respects stream order (a torch.cuda._sleep holds torch's write back).
- FLAC against WAV of the same PCM: the per-file and list forms of hashes, peaks, matching (shifts 1
  and 4, exact count and time range), ingest and precompute, and dist.match_files_sharded at world 2
  over gloo give identical results, on lists that mix WAV, FLAC, .afpk and unreadable files.
- query.flac against the bundled database prints the reference's golden report line."""
import contextlib
import io
import os
import random
import wave

import numpy as np
import pytest
import torch

from audfprint_b200 import Analyzer, HashTable, _lib, flac
from audfprint_b200 import analyzer as an_mod
from tests import flac_writer
from tests.test_gpu_match_files import _spawn
from tests.test_gpu_zz_bundled import MATCH_CONFIGS, golden_table, make_matcher

pytestmark = pytest.mark.gpu
DENS = 100.0
TAG = "d100"
SENTINEL = 0x5A5A


@pytest.fixture(scope="module")
def gf():
    from tests.conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "flac.npz"))


@pytest.fixture(scope="module")
def gb():
    from tests.conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "bundled.npz"))


def _expected(gf, gb, name):
    """FFmpeg's decode of fixture `name` (the bundled query's is its PCM in bundled.npz)."""
    if name == "bundled_query":
        return gb["query/pcm"]
    if name + "/pcm_of" in gf.files:
        name = str(gf[name + "/pcm_of"])
    return gf[name + "/pcm"]


def _streams(gf, names):
    return [flac.parse(gf[n + "/flac"].tobytes()) for n in names]


def test_every_fixture_decodes_in_one_call(gf, gb):
    names = [str(n) for n in gf["names"]]
    ctx = _lib.context(0)
    nsamples, status = flac.locate(ctx, _streams(gf, names))
    meta = {n: gf[n + "/meta"] for n in names}
    # gaps of 37 int16 between the files: every value outside the good files' ranges stays the sentinel
    off, pos = [], 5
    for n, ns in zip(names, nsamples):
        off.append(pos)
        pos += int(ns) * int(meta[n][1]) + 37
    out = torch.full((pos,), SENTINEL, dtype=torch.int16, device="cuda:0")
    with ctx.after_torch(out):
        st = flac.decode_into(ctx, out, off)
    got = out.cpu().numpy()
    keep = np.zeros(pos, bool)
    for n, o, ns, s0, s in zip(names, off, nsamples, status, st):
        assert int(s) == int(meta[n][3]), (n, int(s))
        if s:
            # refused by the locate step: no samples; by the decode step: its own range may be written
            assert s0 == 0 or ns == 0, n
            keep[o:o + int(ns) * int(meta[n][1])] = True
            continue
        want = _expected(gf, gb, n)
        assert np.array_equal(got[o:o + len(want)], want), n
        keep[o:o + len(want)] = True
    assert np.all(got[~keep] == SENTINEL)


def test_the_per_file_reader_decodes_each_fixture(gf, gb, tmp_path):
    for n in [str(n) for n in gf["names"]]:
        fn = str(tmp_path / n)
        with open(fn, "wb") as f:
            f.write(gf[n + "/flac"].tobytes())
        status = int(gf[n + "/meta"][3])
        if status:
            with pytest.raises(IOError):
                an_mod._wav_reader(fn, device=0)
            continue
        rate, nch = int(gf[n + "/meta"][0]), int(gf[n + "/meta"][1])
        raw = flac.decode(flac.parse(gf[n + "/flac"].tobytes()), 0)
        assert np.array_equal(raw, _expected(gf, gb, n)), n
        d, sr = an_mod._wav_reader(fn, sr=None, device=0)
        assert sr == rate and len(d) == len(raw) // nch


def test_4096_short_files_in_one_call(gf, gb):
    names = ["ff_short", "w_variable", "w_depth8", "w_codes_bs6_sr12"]
    base = _streams(gf, names)
    pick = [k % len(names) for k in range(4096)]
    ctx = _lib.context(0)
    nsamples, status = flac.locate(ctx, [base[k] for k in pick])
    assert not status.any()
    lens = [int(ns) * base[k].channels for ns, k in zip(nsamples, pick)]
    off = np.concatenate([[0], np.cumsum(lens)[:-1]])
    out = torch.empty(int(sum(lens)), dtype=torch.int16, device="cuda:0")
    with ctx.after_torch(out):
        assert not flac.decode_into(ctx, out, off).any()
    got = out.cpu().numpy()
    for o, ln, k in zip(off, lens, pick):
        assert np.array_equal(got[o:o + ln], _expected(gf, gb, names[k]))


@pytest.fixture(scope="module")
def cycles():
    n = 10 ** 7
    torch.cuda._sleep(n // 10)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(n)
    e1.record()
    torch.cuda.synchronize()
    return int(n / e0.elapsed_time(e1) * 50)          # 50 ms


def _behind_sleep(cycles, write):
    torch.cuda._sleep(cycles)
    write()
    ev = torch.cuda.Event()
    ev.record()
    assert not ev.query(), "the write finished before the call: the case tested nothing"


def test_device_bytes_respect_stream_order(gf, gb, cycles):
    """Bytes in device memory, written on torch's stream behind a sleep, are read after the write."""
    import ctypes as C
    names = ["w_variable", "ff_level8"]
    streams = _streams(gf, names)
    packed, nbytes, tab = flac._table(streams)
    ctx = _lib.context(0)
    dev = torch.zeros(len(packed), dtype=torch.uint8, device="cuda:0")
    src = torch.from_numpy(packed).pin_memory()
    nsamples, status = np.zeros(2, np.int64), np.zeros(2, np.int32)
    torch.cuda.synchronize()
    _behind_sleep(cycles, lambda: dev.copy_(src, non_blocking=True))
    with ctx.after_torch(dev):
        rc = ctx.lib.afp_flac_locate_batch(ctx.h, dev.data_ptr(), 0, nbytes, 2, tab,
                                           nsamples.ctypes.data_as(C.POINTER(C.c_int64)), status.ctypes.data)
    assert rc == 0 and not status.any()
    lens = [int(n) * s.channels for n, s in zip(nsamples, streams)]
    out = torch.empty(sum(lens), dtype=torch.int16, device="cuda:0")
    with ctx.after_torch(out, dev):
        assert not flac.decode_into(ctx, out, [0, lens[0]]).any()
    got = out.cpu().numpy()
    assert np.array_equal(got[:lens[0]], _expected(gf, gb, "w_variable"))
    assert np.array_equal(got[lens[0]:], _expected(gf, gb, "ff_level8"))


def test_round_buffer_respects_stream_order(gf, gb, cycles):
    """The round's int16 buffer: torch copies the WAV samples behind a sleep, the library decodes the
    FLAC files after them and reads both; the result is the one without the sleep."""
    s = _streams(gf, ["ff_chmode_mid_side"])[0]
    wav = _expected(gf, gb, "ff_level3")
    args = ([wav, s], [2, 2], [11025, 44100], 11025)
    ref = an_mod._frontend_sources(*args, device=0)[0].cpu().numpy()
    torch.cuda.synchronize()
    torch.cuda._sleep(cycles)
    got = an_mod._frontend_sources(*args, device=0)[0].cpu().numpy()
    assert np.array_equal(got, ref)


# ---- FLAC against WAV of the same PCM ------------------------------------------------------------
def _wav(fn, pcm, nch, fs):
    with wave.open(fn, "wb") as w:
        w.setnchannels(nch)
        w.setsampwidth(2)
        w.setframerate(fs)
        w.writeframes(np.ascontiguousarray(pcm, np.int16).tobytes())


@pytest.fixture(scope="module")
def dirs(gf, gb, tmp_path_factory):
    """Two directories with the same file names: one holds FLAC files, the other WAVs of their decoded
    PCM.  Both hold the same .afpk file and the same unreadable file; the FLAC directory's `bad` is a
    damaged FLAC, the WAV directory's an unreadable WAV.  Besides fixtures, the FLAC directory holds the
    bundled tracks and, built from them, a 44.1 kHz mid/side stereo file, a 48 kHz 6-channel file and a
    24-bit stereo file, encoded here with the test bit writer, long enough to give hashes."""
    root = tmp_path_factory.mktemp("flac_vs_wav")
    d_fl, d_wav = root / "flac", root / "wav"
    d_fl.mkdir()
    d_wav.mkdir()
    t = {k: gb["track%d/pcm" % k].astype(np.int64) for k in (0, 4, 8, 12)}
    x44 = np.repeat(t[4][:5 * 11025], 4)
    built = {"stereo44k": (np.stack([x44, x44 // 2], 1), 16, 44100, {"chmode": 10}),
             "ch6_48k": (np.stack([np.roll(t[8], 97 * c)[:3 * 48000] >> (c % 3) for c in range(6)], 1), 16, 48000, {}),
             "s24": (np.stack([t[12] * 256 + 77, t[0] * 256 - 3], 1), 24, 44100, {"specs": [{"method": 1}] * 2})}
    built.update({"t%d" % k: (t[k].reshape(-1, 1), 16, 11025, {}) for k in t})
    for fn, (pcm, bps, rate, kw) in built.items():
        (d_fl / fn).write_bytes(flac_writer.stream(pcm, bps, rate, **kw)[0])
        _wav(str(d_wav / fn), pcm >> (bps - 16), pcm.shape[1], rate)
    files = {"query.flac": "bundled_query", "mid_side": "ff_chmode_mid_side", "ch8": "ff_ch8", "s24_short": "ff_s24_stereo",
             "variable": "w_variable", "total0": "w_total0", "lpc32": "w_lpc32", "short": "ff_short"}
    for fn, key in files.items():
        (d_fl / fn).write_bytes(gf[key + "/flac"].tobytes())
        rate, nch = int(gf[key + "/meta"][0]), int(gf[key + "/meta"][1])
        _wav(str(d_wav / fn), _expected(gf, gb, key), nch, rate)
    (d_fl / "bad").write_bytes(gf["c_residual_bit/flac"].tobytes())
    (d_wav / "bad").write_bytes(b"RIFF\x00\x00\x00\x00WAVEjunk")
    for d in (d_fl, d_wav):
        (d / "broken").write_bytes(b"not audio at all")
    cwd = os.getcwd()
    os.chdir(d_wav)
    try:
        an_mod.peaks_save(str(d_fl / "q.afpk"), Analyzer(density=DENS).wavfile2peaks("query.flac"))
        an_mod.peaks_save(str(d_wav / "q.afpk"), Analyzer(density=DENS).wavfile2peaks("query.flac"))
    finally:
        os.chdir(cwd)
    names = ["query.flac", "t0", "stereo44k", "q.afpk", "bad", "ch6_48k", "t4", "broken", "s24", "variable", "t8",
             "mid_side", "total0", "ch8", "lpc32", "short", "s24_short", "t12", "query.flac"]
    return str(d_fl), str(d_wav), names


@contextlib.contextmanager
def _in(d):
    cwd = os.getcwd()
    os.chdir(d)
    try:
        yield
    finally:
        os.chdir(cwd)


def _analyzer(shifts, fail=False):
    an = Analyzer(density=DENS)
    an.shifts = shifts
    an.fail_on_error = fail
    return an


def _run(d, fn):
    """fn() in directory d with stdout captured -> (result, output lines).  A refused FLAC file is
    reported when its round runs, an unreadable WAV when it is read, so callers compare the lines
    as sets."""
    buf = io.StringIO()
    with _in(d), contextlib.redirect_stdout(buf):
        res = fn()
    return res, buf.getvalue().splitlines()


def _same(a, b):
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype == b.dtype and \
            np.array_equal(a, b)
    return a == b


def _strip_times(lines):
    return [ln.split(" Analyzed ", 1)[-1] for ln in lines]


@pytest.mark.parametrize("shifts", [1, 4])
def test_hashes_and_peaks_equal_the_wavs(dirs, shifts):
    d_fl, d_wav, names = dirs
    for call in (lambda an: [an.wavfile2hashes(n) for n in names], lambda an: an.wavfiles2hashes(names),
                 lambda an: [an.wavfile2peaks(n, shifts) for n in names], lambda an: an.wavfiles2peaks(names, shifts)):
        an_f, an_w = _analyzer(shifts), _analyzer(shifts)
        got, out_f = _run(d_fl, lambda: call(an_f))
        want, out_w = _run(d_wav, lambda: call(an_w))
        assert _same(got, want) and sorted(out_f) == sorted(out_w)
        assert (an_f.soundfiledur, an_f.soundfiletotaldur, an_f.soundfilecount) == \
            (an_w.soundfiledur, an_w.soundfiletotaldur, an_w.soundfilecount)


@pytest.mark.parametrize("shifts", [1, 4])
@pytest.mark.parametrize("cfg", ["default", "exact", "range"])
def test_matching_equals_the_wavs(gb, dirs, cfg, shifts):
    d_fl, d_wav, names = dirs
    ht = golden_table(gb, TAG)
    for form in ("loop", "list"):
        res = []
        for d in (d_fl, d_wav):
            an, mt = _analyzer(shifts), make_matcher(**MATCH_CONFIGS[cfg])
            if form == "loop":
                msgs, out = _run(d, lambda: [mt.file_match_to_msgs(an, ht, n, i) for i, n in enumerate(names)])
            else:
                msgs, out = _run(d, lambda: mt.files_match_to_msgs(an, ht, names))
            res.append((msgs, sorted(_strip_times(out)), an.soundfiletotaldur, an.soundfilecount))
        assert res[0] == res[1], form


def test_query_flac_prints_the_golden_report_line(gb, dirs):
    d_fl, _, _ = dirs
    an, mt = _analyzer(4), make_matcher()
    msgs, _ = _run(d_fl, lambda: mt.file_match_to_msgs(an, golden_table(gb, TAG), "query.flac"))
    want = [str(m).replace("query.mp3", "query.flac") for m in gb[TAG + "/query_s4/default/msgs"]]
    assert msgs == want


def test_a_damaged_flac_raises_like_an_unreadable_wav(dirs):
    d_fl, d_wav, names = dirs
    for call in (lambda an: an.wavfiles2hashes(names), lambda an: an.wavfile2hashes("bad")):
        for d in (d_fl, d_wav):
            an = _analyzer(1, fail=True)
            with pytest.raises(IOError, match="Error reading bad"):
                _run(d, lambda: call(an))
            assert an.soundfilecount == 0


@pytest.mark.parametrize("fail", [False, True])
def test_ingest_equals_the_wavs(dirs, fail):
    d_fl, d_wav, names = dirs
    res = []
    for d in (d_fl, d_wav):
        an, ht = _analyzer(1, fail), HashTable(hashbits=18, depth=20, maxtime=16384)
        random.seed(7)
        try:
            out, lines = _run(d, lambda: an.ingest_files(ht, names))
        except IOError as e:
            out, lines = "IOError " + str(e), []
        res.append((out, sorted(lines), ht.names, np.asarray(ht.table).tobytes(), np.asarray(ht.counts).tobytes(),
                    list(ht.hashesperid), an.soundfilecount, random.random()))
    assert res[0] == res[1]


@pytest.mark.parametrize("kind", ["hashes", "peaks"])
def test_precompute_equals_the_wavs(dirs, tmp_path, kind):
    d_fl, d_wav, names = dirs
    res = []
    for d, tag in ((d_fl, "f"), (d_wav, "w")):
        an = _analyzer(1)
        out = str(tmp_path / tag)
        msgs, _ = _run(d, lambda: an.precompute_files(names, out, type=kind))
        files = {}
        for r, _, fs in os.walk(out):
            for f in fs:
                files[os.path.relpath(os.path.join(r, f), out)] = open(os.path.join(r, f), "rb").read()
        res.append(([[m.replace(out, "OUT") for m in ms] for ms in msgs], files))
    assert res[0] == res[1] and len(res[0][1]) >= 10


def test_match_files_sharded_world2_gloo_equals_the_wavs(dirs):
    d_fl, d_wav, names = dirs
    got = _spawn("gloo", d_fl, names, "ok")
    want = _spawn("gloo", d_wav, names, "ok")
    assert got[0][1] == "ok" and got == want
