"""The list forms of match_file / file_match_to_msgs (Matcher.match_files, files_match_to_msgs over
Analyzer.wavfiles2hashes) and their multi-GPU form (dist.match_files_sharded): for every matcher
option of the bundled-audio tests, verbose and terse, at shifts 1 and 4, they return what the
per-file calls return - rows, seconds, hash counts, report lines, "Analyzed" lines and the
analyzer's counters - on a list that mixes 11025 Hz mono WAVs, the same audio at 44.1 kHz stereo and
48 kHz mono, an 8 kHz file, empty and 100-sample WAVs, .afpt / .afpk files, an unreadable file and a
query over an hour (the long matching path)."""
import contextlib
import datetime
import io
import os
import socket
import wave

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

from audfprint_b200 import Analyzer, Matcher
from audfprint_b200 import analyzer as an_mod
from audfprint_b200 import dist as afd
from tests.test_gpu_zz_bundled import MATCH_CONFIGS, PCM_TRACKS, golden_table, make_matcher

pytestmark = pytest.mark.gpu
DENS = 100.0
TAG = "d100"


def _wav(fn, pcm, nch, fs):
    with wave.open(fn, "wb") as w:
        w.setnchannels(nch)
        w.setsampwidth(2)
        w.setframerate(fs)
        w.writeframes(np.ascontiguousarray(pcm, np.int16).tobytes())


def _resampled(pcm, fs):
    x = resample_poly(pcm.astype(np.float64), fs // np.gcd(fs, 11025), 11025 // np.gcd(fs, 11025))
    return np.round(x).clip(-32768, 32767).astype(np.int16)


@pytest.fixture(scope="module")
def gb():
    from tests.conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "bundled.npz"))


@pytest.fixture(scope="module")
def files(gb, tmp_path_factory):
    """The mixed list, written into a directory the tests chdir into, so that the query's report
    lines carry the name the golden lines carry."""
    d = tmp_path_factory.mktemp("mf")
    q = gb["query/pcm"]
    qn = str(gb["query_name"])
    _wav(str(d / qn), q, 1, 11025)
    for k in PCM_TRACKS:
        _wav(str(d / ("excerpt%d" % k)), gb["track%d/pcm" % k][3 * 11025:8 * 11025], 1, 11025)
    x44 = _resampled(q, 44100)
    _wav(str(d / "q44k_stereo.wav"), np.stack([x44, (x44 * 0.5).astype(np.int16)], axis=1), 2, 44100)
    _wav(str(d / "q48k.wav"), _resampled(q, 48000), 1, 48000)
    _wav(str(d / "q8k.wav"), _resampled(gb["track4/pcm"], 8000), 1, 8000)
    _wav(str(d / "empty.wav"), np.zeros(0, np.int16), 1, 11025)
    _wav(str(d / "tiny.wav"), np.arange(100, dtype=np.int16) * 50, 1, 11025)
    (d / "broken.wav").write_bytes(b"RIFF\x00\x00\x00\x00WAVEjunk")
    from tests.test_match_files_cpu import _zero_rate_wav
    _zero_rate_wav(str(d / "rate0.wav"))            # parses; the front-end has no rate to resample from
    hour = np.tile(np.concatenate([gb["track%d/pcm" % k] for k in PCM_TRACKS]), 91)       # 3640 s
    _wav(str(d / "hour.wav"), hour, 1, 11025)
    an = Analyzer(density=DENS)
    cwd = os.getcwd()
    os.chdir(d)
    try:
        an_mod.hashes_save("q.afpt", an.wavfile2hashes(qn))
        an_mod.peaks_save("q.afpk", an.wavfile2peaks(qn))
    finally:
        os.chdir(cwd)
    mixed = [qn, "excerpt0", "q44k_stereo.wav", "empty.wav", "q48k.wav", "excerpt4", "q.afpt", "q8k.wav",
             "tiny.wav", "broken.wav", "excerpt8", "rate0.wav", "q.afpk", "hour.wav", "excerpt12", qn]
    return d, mixed


@pytest.fixture
def indir(files, monkeypatch):
    monkeypatch.chdir(files[0])
    return files[1]


def _analyzer(shifts, **kw):
    an = Analyzer(density=DENS)
    an.shifts = shifts
    an.fail_on_error = False
    for k, v in kw.items():
        setattr(an, k, v)
    return an


def _counters(an):
    return an.soundfiledur, an.soundfiletotaldur, an.soundfilecount


def _strip(text):
    """Captured output: the "Analyzed" lines without their time stamps, then the other lines (the
    "skipping" report of an unreadable file comes when the file is read, which the list form does
    before it reports the round's files)."""
    lines = text.splitlines()
    return ([ln.split(" Analyzed ", 1)[1] for ln in lines if " Analyzed " in ln] +
            [ln for ln in lines if " Analyzed " not in ln])


def _loop(mt, an, ht, names, start=0):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        msgs = [mt.file_match_to_msgs(an, ht, fn, start + i) for i, fn in enumerate(names)]
    return msgs, _strip(buf.getvalue())


def _batch(mt, an, ht, names, start=0):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        msgs = mt.files_match_to_msgs(an, ht, names, start)
    return msgs, _strip(buf.getvalue())


@pytest.fixture(scope="module")
def table(gb):
    return golden_table(gb, TAG)


def test_the_hour_takes_the_long_path(indir, table):
    an = _analyzer(4)
    q = an.wavfile2hashes("hour.wav")
    mt = make_matcher()
    mt.match_batch(table, [q])
    assert Matcher.last_status(table, 1)[0, 0] == 6


@pytest.mark.parametrize("shifts", [1, 4])
@pytest.mark.parametrize("cfg", list(MATCH_CONFIGS))
def test_list_forms_equal_the_per_file_calls(gb, indir, table, cfg, shifts):
    names = indir
    qn = str(gb["query_name"])
    for verbose in (True, False):
        mt = make_matcher(**MATCH_CONFIGS[cfg])
        mt.verbose = verbose
        a_loop, a_batch = _analyzer(shifts), _analyzer(shifts)
        want, out_loop = _loop(mt, a_loop, table, names, start=3)
        got, out_batch = _batch(mt, a_batch, table, names, start=3)
        assert got == want, (cfg, shifts, verbose)
        assert out_batch == out_loop
        assert _counters(a_batch) == _counters(a_loop)
        assert len(a_batch.last_batch_durations) == len(names)
        key = "%s/query_s%d/%s/%s" % (TAG, shifts, cfg, "msgs" if verbose else "msgs_terse")
        golden = [str(s) for s in gb[key]]
        assert got[0] == golden and got[-1] == golden
        if verbose:
            assert sum(ln.startswith("#%d " % (3 + i)) for i, ln in enumerate(
                [ln for ln in out_batch if not ln.startswith("wavfile2peaks")])) == len(names)
    # the tuples of match_files
    a_loop, a_batch = _analyzer(shifts), _analyzer(shifts)
    mt.verbose = False
    want = [mt.match_file(a_loop, table, fn, i) for i, fn in enumerate(names)]
    got = mt.match_files(a_batch, table, names)
    for (r1, s1, n1), (r2, s2, n2) in zip(want, got):
        assert np.array_equal(r1, r2) and s1 == s2 and n1 == n2
    assert _counters(a_batch) == _counters(a_loop)


def test_wavfiles2hashes_equals_wavfile2hashes(indir):
    for shifts in (1, 4):
        a1, a2 = _analyzer(shifts), _analyzer(shifts)
        want = [a1.wavfile2hashes(fn) for fn in indir]
        got = a2.wavfiles2hashes(indir)
        for w, g in zip(want, got):
            assert type(w) is type(g) and np.array_equal(np.asarray(w), np.asarray(g))
        assert _counters(a1) == _counters(a2)
        assert sum(isinstance(g, list) and g == [] for g in got) >= 3      # empty.wav, broken.wav, rate0.wav


def test_per_file_results_and_bookkeeping(indir, table):
    """The per-file calls' own results, whatever the list forms return: [] for audio without
    samples, for an unreadable file and, at shifts < 2, for a WAV without hashes (at shifts >= 2 an
    empty (0, 2) array); `shifts` empty peak lists for audio without samples; .afpt hashes and .afpk
    peaks as loaded, and an .afpt read as audio by wavfile2peaks.  Each call counts its file once and
    leaves `last_batch_durations`, which is list-form output, as it was."""
    def empty_list(x):
        return type(x) is list and x == []
    for shifts in (1, 4):
        an = _analyzer(shifts)
        an.last_batch_durations = mark = [7.0]
        with contextlib.redirect_stdout(io.StringIO()):
            assert all(empty_list(an.wavfile2hashes(f)) for f in ("empty.wav", "broken.wav", "rate0.wav"))
            tiny = an.wavfile2hashes("tiny.wav")
            assert empty_list(tiny) if shifts < 2 else (type(tiny) is np.ndarray and tiny.shape == (0, 2))
            assert an.wavfile2hashes("q.afpt") == an_mod.hashes_load("q.afpt")
            assert an.wavfile2peaks("q.afpk", shifts) == an_mod.peaks_load("q.afpk")
            assert an.wavfile2peaks("empty.wav", shifts) == ([[]] * shifts if shifts >= 2 else [])
            assert an.wavfile2peaks("q.afpt", 3) == [[], [], []]
            rows, sec, nh = make_matcher().match_file(an, table, "empty.wav")
            assert rows.shape == (0, 7) and sec == 0.0 and nh == 0
        assert an.soundfilecount == 9 and an.last_batch_durations is mark


def test_tiny_caps_give_the_same_result(indir, table):
    mt = make_matcher(**MATCH_CONFIGS["exact_range_time"])
    want, out_w = _batch(mt, _analyzer(4), table, indir)
    for frames, nbytes, per_call in ((1, 1, 1), (1 << 40, 200000, 3), (2000, 1 << 40, 5)):
        an = _analyzer(4, max_frames_per_call=frames, max_pcm_bytes_per_call=nbytes)
        mt.max_files_per_call = per_call
        got, out_g = _batch(mt, an, table, indir)
        assert got == want and out_g == out_w, (frames, nbytes, per_call)


def test_a_read_error_raises_and_changes_nothing(indir, table):
    mt = make_matcher()
    a_loop = _analyzer(1, fail_on_error=True)
    with pytest.raises(IOError) as e_loop, contextlib.redirect_stdout(io.StringIO()):
        _loop(mt, a_loop, table, indir)
    an = _analyzer(1, fail_on_error=True)
    an.soundfiletotaldur, an.soundfilecount = 12.5, 2
    before = _counters(an)
    with pytest.raises(IOError) as e_batch, contextlib.redirect_stdout(io.StringIO()):
        mt.files_match_to_msgs(an, table, indir)
    assert str(e_batch.value) == str(e_loop.value) == "wavfile2peaks: Error reading broken.wav"
    assert _counters(an) == before
    with pytest.raises(IOError), contextlib.redirect_stdout(io.StringIO()):
        an.wavfiles2hashes(indir)
    assert _counters(an) == before
    mt.illustrate = True
    with pytest.raises(NotImplementedError):
        mt.match_files(an, table, indir[:2])


def test_a_custom_reader(gb, table):
    pcm = {"query": gb["query/pcm"], "ex4": gb["track4/pcm"][3 * 11025:8 * 11025], "short": gb["query/pcm"][:50],
           "none": gb["query/pcm"][:0], "int16": gb["track8/pcm"][:40000]}

    def reader(fn, sr=None, channels=None):
        if fn == "int16":
            return pcm[fn], 11025
        return pcm[fn].astype(np.float32) / 32768.0, 11025

    names = ["query", "ex4", "none", "short", "int16", "query"]
    for cfg in ("top5", "exact"):
        mt = make_matcher(**MATCH_CONFIGS[cfg])
        a1, a2 = _analyzer(4, reader=reader), _analyzer(4, reader=reader)
        want, o1 = _loop(mt, a1, table, names)
        got, o2 = _batch(mt, a2, table, names)
        assert got == want and o1 == o2 and _counters(a1) == _counters(a2)


# ---- multi-GPU: world 2 ------------------------------------------------------------------------
def _worker(rank, world, port, backend, device, where, names, mode, out):
    import torch.distributed as dist
    from tests.conftest import GOLDEN
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["AFP_DEVICE"] = str(device)
    torch.cuda.set_device(device)
    os.chdir(where)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        gb = np.load(os.path.join(GOLDEN, "bundled.npz"))
        ht = golden_table(gb, TAG)
        ht.device = device
        if mode == "mismatch" and rank == 1:
            ht.names = ht.names + ["extra"]
        an = Analyzer(density=DENS, device=device)
        an.shifts = 4
        an.fail_on_error = mode == "read_error"
        mt = make_matcher(**MATCH_CONFIGS["exact_range_time"])
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                got = afd.match_files_sharded(mt, an, ht, names)
            out.put((rank, "ok", got, an.soundfilecount))
        except Exception as e:
            out.put((rank, type(e).__name__, str(e), an.soundfilecount))
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _spawn(backend, where, names, mode):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, r if backend == "nccl" else 0, str(where), names,
                                               mode, out)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = sorted((out.get(timeout=600) for _ in range(2)), key=lambda t: t[0])
        for p in procs:
            p.join(600)
            assert p.exitcode == 0
        return res
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(30)


def _single_gpu_lines(files, names):
    cwd = os.getcwd()
    os.chdir(files[0])
    try:
        an = _analyzer(4)
        from tests.conftest import GOLDEN
        ht = golden_table(np.load(os.path.join(GOLDEN, "bundled.npz")), TAG)
        with contextlib.redirect_stdout(io.StringIO()):
            return make_matcher(**MATCH_CONFIGS["exact_range_time"]).files_match_to_msgs(an, ht, names)
    finally:
        os.chdir(cwd)


def _readable(files):
    return [fn for fn in files[1] if fn not in ("broken.wav", "rate0.wav", "hour.wav")]


def test_match_files_sharded_world2_gloo(files):
    names = _readable(files)
    want = _single_gpu_lines(files, names)
    res = _spawn("gloo", files[0], names, "ok")
    assert res[0][1] == "ok" and res[0][2] == want
    assert res[1][1] == "ok" and res[1][2] is None
    assert res[0][3] + res[1][3] == len(names) and res[0][3] == (len(names) + 1) // 2


def test_failures_raise_on_both_ranks(files):
    names = _readable(files)
    names = names[:3] + ["broken.wav"] + names[3:]        # index 3: rank 1's file
    res = _spawn("gloo", files[0], names, "read_error")
    assert [r[1] for r in res] == ["OSError", "OSError"]
    assert res[0][2] == res[1][2] == "wavfile2peaks: Error reading broken.wav"
    res = _spawn("gloo", files[0], _readable(files), "mismatch")
    assert [r[1] for r in res] == ["ValueError", "ValueError"] and res[0][3] == res[1][3] == 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL at world size 2 needs two GPUs")
def test_match_files_sharded_world2_nccl(files):
    names = _readable(files)
    want = _single_gpu_lines(files, names)
    res = _spawn("nccl", files[0], names, "ok")
    assert res[0][2] == want and res[1][2] is None
