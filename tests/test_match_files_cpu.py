"""CPU: the host side of the list forms of wavfile2hashes / match_file and of their multi-GPU form -
the raw WAV parse split out of the default reader, the chunk planning, the per-(up, down) taps table,
read errors of files that never reach the device, and the reassembly of per-rank results in list
order over gloo."""
import os
import socket
import struct
import wave

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from audfprint_b200 import Analyzer
from audfprint_b200 import analyzer as an_mod
from audfprint_b200 import dist as afd


def _write_wav(fn, pcm, nch, fs, width=2):
    with wave.open(fn, "wb") as w:
        w.setnchannels(nch)
        w.setsampwidth(width)
        w.setframerate(fs)
        w.writeframes(pcm.tobytes())


def _zero_rate_wav(fn, nframes=100):
    """A WAV whose header says 0 frames per second (the wave module reads it; its writer refuses it)."""
    data = np.arange(nframes, dtype="<i2").tobytes()
    body = (b"WAVEfmt " + struct.pack("<IHHIIHH", 16, 1, 1, 0, 0, 2, 16) + b"data" + struct.pack("<I", len(data))
            + data)
    with open(fn, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", len(body)) + body)


def _raised(fn, *args, **kw):
    try:
        fn(*args, **kw)
    except Exception as e:          # noqa: BLE001 - the point is to compare what is raised
        return type(e), str(e)
    return None


def test_raw_parse_accepts_and_rejects_what_the_reader_does(tmp_path):
    rng = np.random.default_rng(1)
    mono = rng.integers(-32768, 32768, 1001).astype(np.int16)
    stereo = rng.integers(-32768, 32768, (777, 2)).astype(np.int16)
    _write_wav(str(tmp_path / "m.wav"), mono, 1, 11025)
    _write_wav(str(tmp_path / "s.wav"), stereo, 2, 44100)
    _write_wav(str(tmp_path / "e.wav"), np.zeros(0, np.int16), 1, 11025)
    raw, nch, fs = an_mod._wav_read_raw(str(tmp_path / "m.wav"))
    assert raw.dtype == np.dtype("<i2") and nch == 1 and fs == 11025 and np.array_equal(raw, mono)
    d, sr = an_mod._wav_reader(str(tmp_path / "m.wav"), sr=11025)      # mono at the target rate: host only
    assert sr == 11025 and np.array_equal(d, raw.astype(np.float32) * np.float32(1.0 / 32768.0))
    raw, nch, fs = an_mod._wav_read_raw(str(tmp_path / "s.wav"))
    assert nch == 2 and fs == 44100 and np.array_equal(raw, stereo.reshape(-1))
    raw, nch, fs = an_mod._wav_read_raw(str(tmp_path / "e.wav"))
    assert len(raw) == 0 and nch == 1
    # rejects: 8-bit samples, not a WAV, a missing file - same type and message from both
    _write_wav(str(tmp_path / "b8.wav"), np.zeros(100, np.uint8), 1, 11025, width=1)
    (tmp_path / "junk.wav").write_bytes(b"this is not a RIFF file at all")
    for name in ("b8.wav", "junk.wav", "missing.wav"):
        fn = str(tmp_path / name)
        got = _raised(an_mod._wav_read_raw, fn)
        assert got is not None and got == _raised(an_mod._wav_reader, fn, sr=11025, channels=1), name
    assert _raised(an_mod._wav_read_raw, str(tmp_path / "b8.wav")) == \
        (OSError, "only 16-bit PCM WAV is supported, got 1-byte samples")


def test_unreadable_files_never_reach_the_device(tmp_path, capsys):
    """A list of only unreadable files is decided on the host: skipped and counted as empty without
    fail_on_error, the reader's IOError with the counters unchanged with it."""
    names = [str(tmp_path / n) for n in ("a.wav", "b.wav", "c.wav")]
    (tmp_path / "b.wav").write_bytes(b"RIFF junk")
    _zero_rate_wav(names[2])                  # parses, but no rate to resample from
    assert an_mod._wav_read_raw(names[2])[2] == 0
    an = Analyzer()
    an.fail_on_error = False
    an.soundfiletotaldur, an.soundfilecount, an.soundfiledur = 7.5, 3, 2.5
    assert an.wavfiles2hashes(names) == [[], [], []]
    assert (an.soundfiledur, an.soundfiletotaldur, an.soundfilecount) == (0.0, 7.5, 6)
    assert an.last_batch_durations == [0.0, 0.0, 0.0]
    out = capsys.readouterr().out.splitlines()
    assert out == ["wavfile2peaks: Error reading %s skipping" % n for n in names]
    loop = Analyzer()
    loop.fail_on_error = False
    assert [loop._read(n)[0] for n in names] == [[], [], []]
    assert capsys.readouterr().out.splitlines() == out
    an.fail_on_error = True
    with pytest.raises(IOError) as e:
        an.wavfiles2hashes(names)
    assert str(e.value) == "wavfile2peaks: Error reading " + names[0]
    assert (an.soundfiledur, an.soundfiletotaldur, an.soundfilecount) == (0.0, 7.5, 6)
    assert an.wavfiles2hashes([]) == [] and an.soundfilecount == 6


def test_chunk_planning_keeps_list_order_under_both_caps():
    rng = np.random.default_rng(5)
    frames = rng.integers(1, 50, 200).tolist()
    nbytes = rng.integers(1, 900, 200).tolist()
    for mf, mb in ((100, 10 ** 9), (10 ** 9, 2000), (120, 1500), (1, 1), (10 ** 9, 10 ** 9)):
        ch = an_mod.plan_chunks(frames, nbytes, mf, mb)
        assert ch[0][0] == 0 and ch[-1][1] == len(frames)
        assert all(a[1] == b[0] for a, b in zip(ch, ch[1:])) and all(e > s for s, e in ch)
        for s, e in ch:
            f, b = sum(frames[s:e]), sum(nbytes[s:e])
            assert e - s == 1 or (f <= mf and b <= mb)
            if e < len(frames):      # greedy: the next file would have broken a cap
                assert f + frames[e] > mf or b + nbytes[e] > mb
    # a file over a cap goes alone, and the files around it are unaffected
    assert an_mod.plan_chunks([10, 10, 500, 10, 10], [1] * 5, 100, 10 ** 9) == [(0, 2), (2, 3), (3, 5)]
    assert an_mod.plan_chunks([1] * 5, [10, 10, 5000, 10, 10], 10 ** 9, 100) == [(0, 2), (2, 3), (3, 5)]
    assert an_mod.plan_chunks([500], [1], 100, 100) == [(0, 1)]
    assert an_mod.plan_chunks([], [], 100, 100) == []
    assert an_mod.plan_chunks([1] * 4, [1] * 4, 1, 1) == [(0, 1), (1, 2), (2, 3), (3, 4)]


def test_taps_are_designed_once_per_pair():
    pairs = [(1, 1), (1, 4), (147, 640), (1, 4), (1, 1), (147, 640), (441, 320), (1, 4)]
    rates, off, taps = an_mod.taps_table(pairs)
    assert rates.dtype == np.int32 and rates.tolist() == [[1, 4], [147, 640], [441, 320]]
    assert off.dtype == np.int64 and off[0] == 0 and len(off) == 4 and off[-1] == len(taps)
    for (u, d), a, b in zip(rates.tolist(), off[:-1], off[1:]):
        want = an_mod.resample_taps(u, d)
        assert np.array_equal(taps[a:b], want) and (b - a) % 2 == 1
    rates, off, taps = an_mod.taps_table([(1, 1)] * 3)
    assert rates.shape == (0, 2) and off.tolist() == [0]


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ok = True
        for n in (0, 1, world - 1, world, 7, 11):
            for root in range(world):
                mine = [["msg %d" % int(j), "line 2 of %d" % int(j)] for j in afd.shard_indices(n, rank, world)]
                got = afd.gather_in_list_order(mine, n, root=root)
                want = [["msg %d" % j, "line 2 of %d" % j] for j in range(n)]
                ok = ok and (got == want if rank == root else got is None)
        out.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 3])
def test_results_come_back_in_list_order_over_gloo(world):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    assert sorted(out.get(timeout=10) for _ in range(world)) == [(r, True) for r in range(world)]


def test_single_process_reassembly():
    assert afd.gather_in_list_order([["a"], ["b"]], 2) == [["a"], ["b"]]
