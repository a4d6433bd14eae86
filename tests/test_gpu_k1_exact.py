"""GPU: K1 against the extended-precision reference of tests/exact_stft.py at every frame and every
bin, in FP64 and in FP32 mode.

Each input goes through Analyzer.stft_magnitude (afp_stft_mag: the WRITE_MAG instantiations of
afp_stft_kernel) and Analyzer.conditioned_sgram (afp_sgram: the product instantiations, the stats
and floored-sum kernels, the high-pass); int16 and float32 PCM in both precisions cover all eight
<R, PcmT, WRITE_MAG> instantiations.  The bars are those of tests/exact_stft.py: every magnitude
within C_MAG u ||x_w(t)|| of the extended one (C_MAG at least 64, and 4 x what the reference's own
arithmetic needs on the input), every sgram element within what such magnitudes allow.  A K1 that
changes the last bits of the spectrogram passes if it stays inside them."""
import functools

import numpy as np
import pytest

from audfprint_b200 import Analyzer, _lib
from tests import exact_stft as ex

pytestmark = pytest.mark.gpu

PARAMS = [(name, p) for name, fp32 in ex.CASES.items() for p in (("fp64", "fp32") if fp32 else ("fp64",))]


@functools.lru_cache(maxsize=4)
def bars(name):
    return ex.K1Bars(ex.case_pcm(name), ("fp64", "fp32") if ex.CASES[name] else ("fp64",))


def analyzer(precision):
    an = Analyzer()
    an.precision = precision
    return an


def check(b, mag, sg, precision, record_property):
    ratio, ref_ratio = b.mag_ratio(mag, precision), b.ref_mag_ratio[precision]
    use, ref_use = b.sg_use(sg, precision), b.sg_use(b.ref_sg[precision], precision)
    med, ref_med = b.sg_median_err(sg, precision), b.sg_median_err(b.ref_sg[precision], precision)
    for key, v in (("mag_ratio", ratio), ("mag_ratio_ref", ref_ratio), ("sg_use", use), ("sg_use_ref", ref_use),
                   ("sg_err", b.sg_err(sg)), ("sg_err_ref", b.ref_sg_err[precision]),
                   ("sg_med", med), ("sg_med_ref", ref_med)):
        record_property(key, "%.3g" % v)
    assert np.all(np.isfinite(mag)) and np.all(np.isfinite(sg))
    assert ratio <= b.c_mag(precision), ("magnitude", precision, ratio, ref_ratio)
    assert use <= 1.0, ("sgram", precision, use, ref_use)
    # above the floor, K1's typical sgram error against the reference arithmetic's
    assert med <= ex.C_MED * (ref_med + b.med_quantum()), ("sgram median", precision, med, ref_med)
    if precision == "fp32":   # the north-star bound, at every frame
        m64 = b.ref_mag["fp64"]
        assert np.max(np.abs(mag - m64)) <= ex.FP32_MAG_RTOL * np.max(m64)


@pytest.mark.parametrize("name,precision", PARAMS)
def test_k1_matches_extended_reference(name, precision, record_property):
    pcm = ex.case_pcm(name)
    b = bars(name)
    an = analyzer(precision)
    mag = an.stft_magnitude(pcm)
    sg = an.conditioned_sgram(pcm)
    T = 1 + len(pcm) // ex.N_HOP
    assert mag.shape == (257, T) and sg.shape == (256, T)
    check(b, mag, sg, precision, record_property)


# A CUDA tensor that starts 1, 3 or 5 int16 (1, 2 or 3 float32) samples past a 16-byte boundary:
# no run of the file is 16-byte aligned, so K1 stages every tile by scalar loads.  Offset 0 is the
# aligned device pointer (bulk copies).  The staging must not change a bit.
ALIGN_CASES = [("noise_s1", 0), ("noise_s1", 1), ("noise_s1", 3), ("noise_s1", 5),
               ("f32_random", 0), ("f32_random", 1), ("f32_random", 2), ("f32_random", 3)]


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
@pytest.mark.parametrize("name,offset", ALIGN_CASES)
def test_k1_device_pcm_at_any_alignment(name, offset, precision, record_property):
    import torch
    pcm = ex.case_pcm(name)
    n, T = len(pcm), 1 + len(pcm) // ex.N_HOP
    dtype = _lib.PCM_I16 if pcm.dtype == np.int16 else _lib.PCM_F32
    an = analyzer(precision)
    ctx = an._configure(1)
    buf = torch.zeros(n + 16, dtype=torch.int16 if dtype == _lib.PCM_I16 else torch.float32,
                      device=torch.device("cuda", ctx.device))
    assert buf.data_ptr() % 16 == 0
    buf[offset:offset + n] = torch.from_numpy(pcm).to(buf.device)
    torch.cuda.synchronize(buf.device)
    ptr = buf.data_ptr() + offset * buf.element_size()
    mag = np.empty((T, 257), np.float64)
    sg = np.empty((T, 256), np.float64)
    ctx.check(ctx.lib.afp_stft_mag(ctx.h, ptr, dtype, 0, n, mag.ctypes.data, 1))
    ctx.check(ctx.lib.afp_sgram(ctx.h, ptr, dtype, 0, n, sg.ctypes.data, 1))
    mag, sg = mag.T, sg.T
    check(bars(name), mag, sg, precision, record_property)
    # the host-PCM path stages through an aligned buffer
    assert np.array_equal(mag, an.stft_magnitude(pcm))
    assert np.array_equal(sg, an.conditioned_sgram(pcm))
