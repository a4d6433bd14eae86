"""CPU: the extended-precision K1 reference (tests/exact_stft.py) and the bars built on it.

* The helper's longdouble rfft agrees with a longdouble DFT whose angles are reduced exactly.
* The reference's own float64 arithmetic (the oracle: pocketfft, np.abs, np.log, lfilter; bit-equal
  to the reference by the golden tests) meets the FP64 bars on every input of the GPU test, and the
  float32 statement of FP32 mode meets the FP32 bars.  So the bars K1 is held to in
  tests/test_gpu_k1_exact.py are bars the reference itself meets."""
import numpy as np
import pytest

from tests import exact_stft as ex


def exact_angle_rdft(frames):
    """X[k] = sum_n x[n] exp(-2 pi i n k / 512), n k reduced mod 512 in integers and pi in
    longdouble: the angles are exact to the last bit of longdouble."""
    pi = 4 * np.arctan(ex.LD(1))
    nk = (np.arange(ex.N_FFT)[:, None] * np.arange(ex.NBINS)[None, :]) % ex.N_FFT
    ang = 2 * pi * nk.astype(ex.LD) / ex.N_FFT
    return frames @ np.cos(ang) - 1j * (frames @ np.sin(ang))


@pytest.mark.parametrize("name", ["noise_s1", "fs_square", "f32_random", "len_513"])
def test_extended_rfft_matches_exact_angle_dft(name):
    frames = ex.windowed_frames(ex.case_pcm(name))
    frames = frames[np.linspace(0, len(frames) - 1, min(60, len(frames))).astype(int)]
    got = np.fft.rfft(frames, axis=1)
    assert got.dtype == np.clongdouble
    want = exact_angle_rdft(frames)
    norms = np.sqrt(np.sum(frames * frames, axis=1))
    assert np.all(norms > 0)
    rel = np.max(np.abs(got - want), axis=1) / norms
    assert np.max(rel) <= 1e-16, float(np.max(rel))


def test_dynamic_range_cases_reach_the_floor():
    """The floor (max / 1e6) bites where the cases say it does, so K1's floored-sum path runs."""
    for name in ("dr_tone_lsb", "dr_clicks", "fs_cos_64"):
        _, mag, _ = ex.extended_sgram(ex.case_pcm(name))
        assert np.min(mag) < np.max(mag) / 1e6, name
    _, mag, _ = ex.extended_sgram(ex.case_pcm("dr_zeros"))
    assert np.max(mag) == 0


@pytest.mark.parametrize("name", list(ex.CASES))
def test_reference_arithmetic_meets_the_bars(name):
    pcm = ex.case_pcm(name)
    precisions = ("fp64", "fp32") if ex.CASES[name] else ("fp64",)
    b = ex.K1Bars(pcm, precisions)
    T = 1 + len(pcm) // ex.N_HOP
    assert b.mag.shape == (257, T) and b.sg.shape == (256, T) and b.norms.shape == (T,)
    # pocketfft in float64: |X| from the oracle's complex STFT and from its conditioned_sgram
    assert np.array_equal(np.abs(b.ref_complex), b.ref_mag["fp64"])
    for p in precisions:
        ratio = b.ref_mag_ratio[p]
        # the reference FFT stays under the fixed constant on its own: on these inputs the bar
        # is C_MAG_MIN unless K1's own reference needs more
        assert ratio <= ex.C_MAG_MIN, (p, ratio)
        assert ratio <= b.c_mag(p)
        assert b.sg_use(b.ref_sg[p], p) <= 1.0, (p, b.sg_use(b.ref_sg[p], p))
    if "fp32" in precisions:
        m64 = b.ref_mag["fp64"]
        assert np.max(np.abs(b.ref_mag["fp32"] - m64)) <= ex.FP32_MAG_RTOL * np.max(m64)
