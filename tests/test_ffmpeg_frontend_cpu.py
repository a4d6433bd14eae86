"""The statement of ffmpeg's down-mix and resampler (tests/swr_reference.py) against FFmpeg's own
output (tests/golden/ffmpeg_frontend.npz), and the library's host design against the statement."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import ffmpeg_frontend_cases as FC
from tests import swr_reference as R

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "ffmpeg_frontend.npz"))
LIB = os.path.join(os.path.dirname(os.path.dirname(__file__)), "audfprint_b200", "libafp.so")


@pytest.mark.parametrize("rate", FC.RATES)
def test_statement_equals_ffmpeg(rate):
    n = 0
    for name, r, ch, pcm in FC.cases():
        if r == rate:
            assert np.array_equal(R.frontend(pcm, ch, r), GOLD["out_" + name]), name
            n += 1
    assert n == 2 * len(FC.lengths(rate))


def test_song_heads_equal_ffmpeg():
    for rate, seed in FC.SONGS:
        got = R.frontend(FC.song(rate, seed)[:2 * rate], 2, rate)[:4000]
        assert np.array_equal(got, GOLD["song_%d_head" % rate][:4000])


def _design(lib, rate):
    P, L = C.c_int32(), C.c_int32()
    assert lib.afp_swr_design(rate, R.OUT_RATE, None, 0, C.byref(P), C.byref(L)) == 0
    bank = np.empty(P.value * L.value, np.float32)
    assert lib.afp_swr_design(rate, R.OUT_RATE, bank.ctypes.data_as(C.c_void_p), bank.size, None, None) == 0
    return bank.reshape(P.value, L.value)


@pytest.mark.skipif(not os.path.exists(LIB), reason="libafp.so not built")
def test_host_design_equals_statement():
    lib = C.CDLL(LIB)
    lib.afp_swr_design.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    for rate in FC.RATES + (12000, 7350):
        if rate != R.OUT_RATE:
            assert np.array_equal(_design(lib, rate), R.design(rate)), rate
    assert lib.afp_swr_design(44099, R.OUT_RATE, None, 0, None, None) == -3      # AFP_ERR_UNSUPPORTED
    assert lib.afp_swr_design(192000, R.OUT_RATE, None, 0, None, None) == -3
    assert lib.afp_swr_design(0, R.OUT_RATE, None, 0, None, None) == -2          # AFP_ERR_INVALID
    assert lib.afp_swr_design(44100, R.OUT_RATE, np.zeros(4, np.float32).ctypes.data_as(C.c_void_p), 4,
                              None, None) == -2


def test_statement_refusals():
    with pytest.raises(R.Unsupported):
        R.geometry(44099)
    with pytest.raises(R.Unsupported):
        R.geometry(192000)
    with pytest.raises(R.Unsupported):
        R.frontend(np.zeros(30, np.int16), 3, 44100)


def test_fma_rounds_once():
    # a b + c = 1 + 2^-23 + 2^-24 - 2^-54: just below the float32 midpoint of 1 + 2^-23 and 1 + 2^-22,
    # which float64 rounding of the sum would reach (and then round to even, the wrong way)
    a = np.array([2**-12 * (1 + 2**-15)], np.float32)
    b = np.array([2**-12 * (1 - 2**-15)], np.float32)
    c = np.array([1 + 2**-23], np.float32)
    assert (a.astype(np.float64) * b + c).astype(np.float32)[0] == np.float32(1 + 2**-22)
    assert R._fma(a, b, c)[0] == np.float32(1 + 2**-23)
    rng = np.random.default_rng(5)
    x, y, z = (rng.standard_normal(4096).astype(np.float32) for _ in range(3))
    from fractions import Fraction as F
    want = [np.float32(float(F(float(p)) * F(float(q)) + F(float(r)))) for p, q, r in zip(x[:256], y[:256], z[:256])]
    assert np.array_equal(R._fma(x[:256], y[:256], z[:256]), np.array(want, np.float32))


@pytest.mark.skipif(not os.path.exists(LIB), reason="libafp.so not built")
def test_host_length_equals_statement():
    lib = C.CDLL(LIB)
    lib.afp_swr_length.argtypes = [C.c_int64, C.c_int32, C.c_int32, C.POINTER(C.c_int64)]
    n = C.c_int64()
    for rate in FC.RATES:
        for frames in FC.lengths(rate) + (30 * rate, 30 * rate + 1, 12345):
            assert lib.afp_swr_length(frames, rate, R.OUT_RATE, C.byref(n)) == 0
            assert n.value == R.out_length(frames, rate), (rate, frames)
    assert lib.afp_swr_length(100, 192000, R.OUT_RATE, C.byref(n)) == -3
    assert lib.afp_swr_length(100, 44099, R.OUT_RATE, C.byref(n)) == -3
    assert lib.afp_swr_length(-1, 44100, R.OUT_RATE, C.byref(n)) == -2


def test_wav_channel_mask(tmp_path):
    from audfprint_b200 import analyzer as A
    pcm = np.zeros(40, np.int16)
    p = tmp_path / "a.wav"
    p.write_bytes(FC.wav_bytes(pcm, 44100, 2))
    assert A._wav_channel_mask(str(p)) is None
    for mask in (0x3, 0x30, 0):
        p.write_bytes(FC.wav_extensible_bytes(pcm, 44100, 2, mask))
        assert A._wav_channel_mask(str(p)) == mask
    A._swr_check(str(p), pcm, 2, 44100, R.OUT_RATE)                  # mask 0: no layout named
    p.write_bytes(FC.wav_extensible_bytes(pcm, 44100, 2, 0x30))      # BL | BR
    with pytest.raises(ValueError):
        A._swr_check(str(p), pcm, 2, 44100, R.OUT_RATE)
    with pytest.raises(ValueError):
        A._swr_check(str(p), pcm, 3, 44100, R.OUT_RATE)
