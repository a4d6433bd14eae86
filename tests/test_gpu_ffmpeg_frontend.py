"""The device's ffmpeg front-end (afp_swr_frontend_batch) against FFmpeg's output and the statement
(tests/golden/ffmpeg_frontend.npz, tests/swr_reference.py), through every entry point."""
import os

import numpy as np
import pytest

from tests import ffmpeg_frontend_cases as FC
from tests import swr_reference as R

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ffmpeg_frontend.npz"))


def _as_s16(v):
    v = np.asarray(v, np.float32) * np.float32(32768)
    assert np.array_equal(v, np.rint(v))
    return v.astype(np.int16)


def test_batch_host_and_device_input():
    import torch
    from audfprint_b200 import analyzer as A
    cs = FC.cases()
    raws, chs, rates = [c[3] for c in cs], [c[2] for c in cs], [c[1] for c in cs]
    for src in ("host", "device"):
        if src == "host":
            out, off, lens = A.pcm_frontend_batch(raws, chs, rates, R.OUT_RATE, resampler='ffmpeg')
        else:
            inoff = np.zeros(len(raws) + 1, np.int64)
            inoff[1:] = np.cumsum([len(r) for r in raws])
            pcm = torch.from_numpy(np.concatenate(raws)).cuda()
            from audfprint_b200 import _lib
            out, off, lens = A._frontend_packed(_lib.context(None), pcm, inoff[:-1],
                                                [len(r) // c for r, c in zip(raws, chs)], chs, rates, R.OUT_RATE,
                                                'ffmpeg')
        host = out.cpu().numpy()
        for k, (name, _, _, _) in enumerate(cs):
            got = _as_s16(host[off[k]:off[k] + lens[k]])
            assert np.array_equal(got, GOLD["out_" + name]), (src, name)


@pytest.mark.parametrize("suffix", [".wav", ".flac"])
def test_per_file_reader(tmp_path, suffix):
    from audfprint_b200 import analyzer as A
    for name, rate, ch, pcm in FC.cases():
        if len(pcm) < 16 * ch or rate not in (8000, 22050, 44100, 48000, 37800, 11025):
            continue
        p = str(tmp_path / ("x" + suffix))
        with open(p, "wb") as f:
            f.write(FC.wav_bytes(pcm, rate, ch) if suffix == ".wav" else FC.flac_bytes(pcm, rate, ch))
        d, sr = A._wav_reader(p, sr=R.OUT_RATE, channels=1, resampler='ffmpeg')
        assert sr == R.OUT_RATE
        assert np.array_equal(_as_s16(d), GOLD["out_" + name]), (suffix, name)


def test_songs_give_the_reference_hashes(tmp_path):
    from audfprint_b200 import Analyzer
    files = []
    for rate, seed in FC.SONGS:
        for suffix in (".wav", ".flac"):
            pcm = FC.song(rate, seed)
            p = str(tmp_path / ("s%d%s" % (rate, suffix)))
            with open(p, "wb") as f:
                f.write(FC.wav_bytes(pcm, rate, 2) if suffix == ".wav" else FC.flac_bytes(pcm, rate, 2))
            files.append((p, GOLD["song_%d_hashes" % rate]))
    an = Analyzer(resampler='ffmpeg')
    listed = an.wavfiles2hashes([p for p, _ in files])
    for (p, want), got in zip(files, listed):
        assert np.array_equal(np.asarray(got), want), p
        assert np.array_equal(np.asarray(an.wavfile2hashes(p)), want), p
    # the default front-end is a different resampler: not the same hashes
    assert not np.array_equal(np.asarray(Analyzer().wavfile2hashes(files[0][0])), files[0][1])


def test_refusals():
    from audfprint_b200 import analyzer as A, _lib
    with pytest.raises(_lib.AfpError):
        A.pcm_frontend_batch([np.zeros(300, np.int16)], [3], [44100], R.OUT_RATE, resampler='ffmpeg')
    with pytest.raises(_lib.AfpError):
        A.pcm_frontend_batch([np.zeros(300, np.int16)], [1], [44099], R.OUT_RATE, resampler='ffmpeg')
    with pytest.raises(ValueError):
        A.pcm_frontend(np.zeros(300, np.int16), 1, 44100, R.OUT_RATE, resampler='sox')


def test_refused_files_in_lists_are_read_failures(tmp_path, capsys):
    from audfprint_b200 import Analyzer
    rng = np.random.default_rng(9)
    files = []
    for k, (rate, mask) in enumerate([(44100, None), (192000, None), (48000, 0x30), (44099, None), (48000, None)]):
        pcm = (rng.normal(0, 3000, 2 * rate)).astype(np.int16)
        p = tmp_path / ("f%d.wav" % k)
        p.write_bytes(FC.wav_bytes(pcm, rate, 2) if mask is None else FC.wav_extensible_bytes(pcm, rate, 2, mask))
        files.append(str(p))
    an = Analyzer(resampler='ffmpeg')
    an.fail_on_error = False
    per_file = [an.wavfile2hashes(f) for f in files]
    listed = an.wavfiles2hashes(files)
    for k, (a, b) in enumerate(zip(per_file, listed)):
        assert np.array_equal(np.asarray(a), np.asarray(b)), k
    assert [len(x) > 0 for x in listed] == [True, False, False, False, True]
    assert capsys.readouterr().out.count("skipping") == 6
    an.fail_on_error = True
    for f in files[1:4]:
        with pytest.raises(IOError):
            an.wavfile2hashes(f)
        with pytest.raises(IOError):
            an.wavfiles2hashes([files[0], f])
