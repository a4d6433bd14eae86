"""The device PCM front-end (csrc/afp_pcm.cu, SURVEY.md §8f-2): down-mix + polyphase resampling
against scipy.signal.resample_poly, and through the WAV reader to fingerprints.  The reference
delegates this step to ffmpeg (audio_read.py:196-203), whose resampler no other implementation
reproduces bit for bit; the front-end's own output is held to its correctly rounded statement at
every sample by tests/test_gpu_pcm_exact.py."""
import wave

import numpy as np
import pytest
from scipy.signal import resample_poly

from audfprint_b200 import Analyzer
from audfprint_b200 import analyzer as an_mod
from audfprint_b200.synth import synth_track
from oracle import afp_oracle as orc
from tests.exact_resample import TARGET, check_rounded, downmix, reference, up_down

pytestmark = pytest.mark.gpu


def _host_statement(raw, nch, fs, sr):
    x = raw.reshape(-1, nch).astype(np.float32) * np.float32(1.0 / 32768.0)
    mono = x.mean(axis=1).astype(np.float32) if nch > 1 else x[:, 0]
    if sr is None or sr == fs:
        return mono
    from math import gcd
    g = gcd(sr, fs)
    return resample_poly(mono.astype(np.float64), sr // g, fs // g).astype(np.float32)


@pytest.mark.parametrize("fs,nch", [(44100, 2), (22050, 1), (48000, 2), (8000, 1), (11025, 3), (16000, 6)])
def test_frontend_matches_resample_poly(fs, nch):
    rng = np.random.default_rng(fs + nch)
    n = int(fs * 1.7) + 13
    raw = (rng.standard_normal((n, nch)) * 6000).clip(-32768, 32767).astype(np.int16)
    t = np.arange(n) / fs
    raw[:, 0] += (9000 * np.sin(2 * np.pi * 997.0 * t)).astype(np.int16)
    got = an_mod.pcm_frontend(raw, nch, fs, 11025)
    want = _host_statement(raw, nch, fs, 11025)
    assert got.dtype == np.float32 and got.shape == want.shape
    assert np.max(np.abs(got - want)) < 2e-6          # float32 rounding of a float64 dot product
    dev = an_mod.pcm_frontend(raw, nch, fs, 11025, to_host=False)
    assert dev.is_cuda and np.array_equal(dev.cpu().numpy(), got)
    assert len(an_mod.pcm_frontend(raw[:0], nch, fs, 11025)) == 0


def _file_level_api(tmp_path, fs, nch):
    """A WAV of a known track at fs with nch channels: read (device down-mix + resample) and
    fingerprint.  The samples are the correctly rounded front-end statement of tests/exact_resample.py
    (its tie zone is empty on this file), so the hashes equal the oracle's on those samples bit for bit."""
    mono11 = synth_track(4242, 8.0)
    up_fs, down_fs = up_down(TARGET, fs)
    x = resample_poly(mono11.astype(np.float64), up_fs, down_fs)
    pcm = np.stack([x * g for g in (0.8, 0.7)[:nch]], axis=1).clip(-32768, 32767).astype(np.int16)
    fn = str(tmp_path / "s.wav")
    with wave.open(fn, "wb") as w:
        w.setnchannels(nch); w.setsampwidth(2); w.setframerate(fs)
        w.writeframes(pcm.tobytes())
    d, sr = an_mod._wav_reader(fn, sr=TARGET, channels=1)
    up, down = up_down(fs, TARGET)
    ref, S, m = reference(downmix(pcm, nch), up, down)
    assert sr == TARGET and d.dtype == np.float32 and len(d) == len(ref)
    assert check_rounded(d, ref, S, m, "%d Hz x %d WAV" % (fs, nch)) == 0
    want = ref.astype(np.float32)
    assert np.array_equal(d, want)
    d2, sr2 = an_mod._wav_reader(fn)                      # no target rate: native rate, still mono
    assert sr2 == fs and np.array_equal(d2, downmix(pcm, nch))
    an = Analyzer()
    h = an.wavfile2hashes(fn)
    assert np.array_equal(h, orc.fingerprint(want)) and abs(an.soundfiledur - 8.0) < 0.01


def test_wav_reader_and_file_level_api(tmp_path):
    _file_level_api(tmp_path, 44100, 2)


@pytest.mark.parametrize("nch", [1, 2])
def test_wav_reader_and_file_level_api_48k(tmp_path, nch):
    _file_level_api(tmp_path, 48000, nch)
