"""Analyzer.ingest_files, the list form of the reference's `new` / `add` loop, against that loop
(Analyzer.ingest per file): returned (duration, hashes), table, counts, names, hashesperid, the
counters and the next random.random() must be equal, on a list that mixes mono, stereo, 48 kHz and
8 kHz WAVs, empty, unreadable and 0 Hz files, .afpt / .afpk files and repeated names; also under
tiny caps, with a read failure under fail_on_error, and for dist.ingest_files_sharded at world 1."""
import os
import random
import wave

import numpy as np
import pytest
from scipy.signal import resample_poly

from audfprint_b200 import Analyzer, HashTable
from audfprint_b200 import analyzer as an_mod
from audfprint_b200 import dist as afd
from audfprint_b200.synth import synth_track

pytestmark = pytest.mark.gpu


def _wav(fn, pcm, nch, fs):
    with wave.open(fn, "wb") as w:
        w.setnchannels(nch)
        w.setsampwidth(2)
        w.setframerate(fs)
        w.writeframes(np.ascontiguousarray(pcm, np.int16).tobytes())


def _resampled(pcm, fs):
    g = np.gcd(fs, 11025)
    return np.round(resample_poly(pcm.astype(np.float64), fs // g, 11025 // g)).clip(-32768, 32767).astype(np.int16)


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("ingf")
    tr = [synth_track(900 + i, 8.0 + i) for i in range(6)]
    names = []
    for i, x in enumerate(tr):
        fn = str(d / ("t%d.wav" % i))
        _wav(fn, x, 1, 11025)
        names.append(fn)
    x44 = _resampled(tr[1], 44100)
    _wav(str(d / "st44.wav"), np.stack([x44, (x44 // 2).astype(np.int16)], axis=1), 2, 44100)
    _wav(str(d / "m48.wav"), _resampled(tr[2], 48000), 1, 48000)
    _wav(str(d / "m8.wav"), _resampled(tr[3], 8000), 1, 8000)
    _wav(str(d / "empty.wav"), np.zeros(0, np.int16), 1, 11025)
    (d / "broken.wav").write_bytes(b"RIFF\x00\x00\x00\x00WAVEjunk")
    from tests.test_match_files_cpu import _zero_rate_wav
    _zero_rate_wav(str(d / "rate0.wav"))
    an = Analyzer(density=100.0)
    an_mod.hashes_save(str(d / "h4.afpt"), an.wavfile2hashes(names[4]))
    an_mod.peaks_save(str(d / "p5.afpk"), an.wavfile2peaks(names[5]))
    an_mod.peaks_save(str(d / "one.afpk"), [(7, 30)])
    p = lambda s: str(d / s)
    mixed = [names[0], p("st44.wav"), p("empty.wav"), p("m48.wav"), p("h4.afpt"), names[1], p("p5.afpk"),
             p("one.afpk"), p("m8.wav"), p("broken.wav"), names[2], p("rate0.wav"), names[3], names[0],
             p("p5.afpk"), names[4], names[5]]
    return d, names, mixed


def _an(shifts=1, **kw):
    an = Analyzer(density=100.0)
    an.shifts = shifts
    an.fail_on_error = False
    for k, v in kw.items():
        setattr(an, k, v)
    return an


def _state(ht, an, ret):
    return dict(table=np.array(ht.table), counts=np.array(ht.counts), names=list(ht.names),
                hpi=np.array(ht.hashesperid), ret=ret, rnd=random.random(),
                cnt=(an.soundfiledur, an.soundfiletotaldur, an.soundfilecount))


def _loop(lst, geom, shifts=1, seed=5, **kw):
    an = _an(shifts, **kw)
    ht = HashTable(hashbits=geom[0], depth=geom[1], maxtime=geom[2])
    random.seed(seed)
    ret, err = [], None
    try:
        for f in lst:
            ret.append(an.ingest(ht, f))
    except Exception as e:
        err = e
    return _state(ht, an, ret), err


def _listed(lst, geom, shifts=1, seed=5, **kw):
    an = _an(shifts, **kw)
    ht = HashTable(hashbits=geom[0], depth=geom[1], maxtime=geom[2])
    random.seed(seed)
    ret, err = [], None
    try:
        ret = an.ingest_files(ht, lst)
    except Exception as e:
        err = e
    return _state(ht, an, ret), err


def _same(a, b, raised=False):
    for k in ("table", "counts", "hpi"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    assert a["names"] == b["names"]
    if not raised:                 # a raising list form returns nothing; the loop returned the earlier files
        assert a["ret"] == b["ret"]
    assert a["rnd"] == b["rnd"]
    assert a["cnt"] == b["cnt"]


@pytest.mark.parametrize("geom", [(10, 6, 1 << 14), (20, 100, 1 << 14)])
@pytest.mark.parametrize("shifts", [1, 4])
def test_ingest_files_equals_loop(files, geom, shifts):
    _, _, mixed = files
    want, e1 = _loop(mixed, geom, shifts)
    got, e2 = _listed(mixed, geom, shifts)
    assert e1 is None and e2 is None, (e1, e2)
    _same(want, got)


def test_tiny_caps(files):
    _, _, mixed = files
    want, _ = _loop(mixed, (10, 6, 1 << 14), 4)
    got, err = _listed(mixed, (10, 6, 1 << 14), 4, max_frames_per_call=3000, max_pcm_bytes_per_call=200000)
    assert err is None
    _same(want, got)


@pytest.mark.parametrize("at", [0, 4, 5, 16])
def test_read_failure_keeps_loop_state(files, at):
    """fail_on_error: the failing file raises the loop's exception, after the files before it were
    stored: at the first file, inside a chunk and at a chunk's last file (tiny caps)."""
    d, names, _ = files
    good = [names[i % len(names)] for i in range(16)]
    lst = good[:at] + [str(d / "broken.wav")] + good[at:]
    kw = dict(fail_on_error=True, max_frames_per_call=2500)
    want, e1 = _loop(lst, (10, 6, 1 << 14), 1, **kw)
    got, e2 = _listed(lst, (10, 6, 1 << 14), 1, **kw)
    assert type(e1) is type(e2) is IOError and str(e1) == str(e2)
    _same(want, got, raised=True)


def test_malformed_afpk_keeps_loop_state(files, tmp_path):
    d, names, _ = files
    bad = str(tmp_path / "bad.afpk")
    an_mod.peaks_save(bad, [(5, 3), (2, 4)])                  # not column-major
    empty = str(tmp_path / "empty.afpk")
    an_mod.peaks_save(empty, [])
    for extra in (bad, empty):
        lst = [names[0], str(d / "p5.afpk"), extra, str(d / "one.afpk"), names[1]]
        want, e1 = _loop(lst, (10, 6, 1 << 14), 1, fail_on_error=True)
        got, e2 = _listed(lst, (10, 6, 1 << 14), 1, fail_on_error=True)
        assert e1 is not None and type(e1) is type(e2)
        _same(want, got, raised=True)


def test_ingest_files_sharded_world1(files):
    d, names, _ = files
    wavs = names + [str(d / "m48.wav")]
    an = _an()
    ht = HashTable(hashbits=14, depth=20, maxtime=1 << 14)
    random.seed(8)
    np.random.seed(8)
    lines = []
    afd.ingest_files_sharded(an, ht, wavs, report=lines.append)
    an2 = _an()
    ht2 = HashTable(hashbits=14, depth=20, maxtime=1 << 14)
    random.seed(8)
    np.random.seed(8)
    sigs = [an2._read(f)[0] for f in wavs]
    afd.ingest_sharded(an2, ht2, wavs, sigs, report=lines.append)
    np.testing.assert_array_equal(ht.table, ht2.table)
    np.testing.assert_array_equal(ht.counts, ht2.counts)
    assert list(ht.names) == list(ht2.names)
    np.testing.assert_array_equal(ht.hashesperid, ht2.hashesperid)
    assert lines[0] == lines[1]


def test_store_batch_of_empty_tracks_stores_nothing(files):
    """store_batch(names, hashes) with every hash list empty takes the names and stores no entry,
    whatever the workspace holds (it once stored the last fingerprint batch instead)."""
    _, names, _ = files
    an = _an()
    an.wavfiles2hashes(names[:3])                     # a fingerprint batch of 3 files in the workspace
    ht = HashTable(hashbits=10, depth=6, maxtime=1 << 14)
    assert ht.store_batch(["a", "b", "c"], [[], np.zeros((0, 2), np.int32), []]) == [0, 0, 0]
    assert list(ht.names) == ["a", "b", "c"] and not np.asarray(ht.counts).any()
    assert not np.asarray(ht.table).any() and not np.asarray(ht.hashesperid).any()


# ---- world 2 over gloo, spawned on one GPU -------------------------------------------------------
GEOM = dict(hashbits=12, depth=8, maxtime=1 << 14)


def _worker(rank, world, port, names, fail, out):
    import contextlib
    import datetime
    import io
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    os.environ["AFP_DEVICE"] = "0"
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        an = _an(1, device=0, fail_on_error=fail)
        ht = HashTable(device=0, **GEOM)
        random.seed(1000 + rank)
        np.random.seed(7)
        lines = []
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                ret = afd.ingest_files_sharded(an, ht, names, report=lines.extend)
            out.put((rank, "ok", (np.array(ht.table), np.array(ht.counts), list(ht.names),
                                  np.array(ht.hashesperid), lines, ret)))
        except Exception as e:
            out.put((rank, type(e).__name__, str(e)))
    finally:
        dist.destroy_process_group()


def _spawn(names, fail):
    import socket
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, 2, port, names, fail, out)) for r in range(2)]
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


def test_ingest_files_sharded_world2_gloo(files):
    d, names, mixed = files
    lst = [f for f in mixed if not f.endswith("rate0.wav")]
    res = _spawn(lst, False)
    assert res[0][1] == "ok" and res[1][1] == "ok", res
    # what the reference's multiproc_add builds for the same per-worker seeds: worker r's table from
    # files r, r + 2, ..., then the merge of both in worker order
    tabs = []
    for r in range(2):
        t = HashTable(**GEOM)
        random.seed(1000 + r)
        rets = _an(1).ingest_files(t, lst[r::2])
        assert res[r][2][5] == rets
        tabs.append(t)
    ht = HashTable(**GEOM)
    np.random.seed(7)
    ht.merge_batch(tabs)
    table, counts, nm, hpi, lines, _ = res[0][2]
    np.testing.assert_array_equal(table, ht.table)
    np.testing.assert_array_equal(counts, ht.counts)
    assert nm == list(ht.names)
    np.testing.assert_array_equal(hpi, ht.hashesperid)
    assert lines == ["hash_table %d has %d files %d hashes" % (r, len(t.names), int(np.sum(t.hashesperid)))
                     for r, t in enumerate(tabs)]
    assert res[1][2][2] == [] and res[1][2][4] == []          # the other rank's table is unchanged


def test_ingest_files_sharded_read_failure_on_one_rank(files):
    d, names, _ = files
    lst = names[:3] + [str(d / "broken.wav")] + names[3:]      # index 3: rank 1's file
    res = _spawn(lst, True)
    assert [r[1] for r in res] == ["OSError", "OSError"], res
    assert res[0][2] == res[1][2] == "wavfile2peaks: Error reading " + str(d / "broken.wav")
