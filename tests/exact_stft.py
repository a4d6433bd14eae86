"""Extended-precision reference of K1 (STFT, |X|, log, floor, mean, high-pass) and the accuracy
bars K1 is held to.  TEST INFRASTRUCTURE, like tests/cases.py.

The reference spectrogram is float64 all the way (pocketfft `rfft`, `np.abs`, `np.log`,
`lfilter`).  Here the same steps run in `np.longdouble` (64-bit mantissa on x86-64), 11 bits more
than float64, so that the error of a float64 (or float32) implementation can be measured element by
element: the extended result stands in for the exact one.

The bars (DESIGN.md §2), with u = 2^-53 in FP64 mode and 2^-24 in FP32 mode and x_w(t) the
windowed frame t:
  magnitudes, per bin:     |M - M_ext| <= C_MAG * u * ||x_w(t)||_2,
                           C_MAG = max(C_MAG_MIN, C_MAG_OVER_REF * the reference arithmetic's own ratio);
  sgram, per element:      |S - S_ext| <= what magnitudes within that bar allow after log, floor,
                           mean and high-pass, plus the log routine's error (K1Bars.sg_bound).
In FP64 mode the reference arithmetic is the oracle (pocketfft in float64, bit-equal to the
reference by the golden tests); in FP32 mode it is `float32_sgram` below, the same steps with a
float32 FFT and log.  tests/test_k1_exact_reference_cpu.py checks that both meet the bars.
"""
from __future__ import annotations

import numpy as np

from audfprint_b200.synth import SR, pcm_to_float, synth_track
from oracle import afp_oracle as orc

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "np.longdouble must have a 64-bit mantissa (x86-64 extended precision)"

N_FFT, N_HOP, NBINS = 512, 256, 257
HPF_POLE = 0.98

U = {"fp64": 2.0 ** -53, "fp32": 2.0 ** -24}
C_MAG_MIN = 64.0
C_MAG_OVER_REF = 4.0
C_SG_U = 32.0
# K1's median sgram error above the floor may be this many times the reference arithmetic's
C_MED = 4.0
# __logf (CUDA C Programming Guide, intrinsic functions): 2^-21.41 absolute for x in [0.5, 2],
# 3 ulp elsewhere
LOGF_ABS = 2.0 ** -21.41
LOGF_ULPS = 3.0
# FP32 mode's north-star bound on magnitudes, relative to the file's largest
FP32_MAG_RTOL = 1e-5


def pcm_as_float(pcm: np.ndarray) -> np.ndarray:
    """PCM as the reference's reader hands it on: int16 / 32768 as float32, float32 as given."""
    a = np.asarray(pcm)
    if a.dtype == np.int16:
        return pcm_to_float(a)
    assert a.dtype == np.float32, a.dtype
    return a


def _frame_index(n: int) -> np.ndarray:
    nfr = 1 + n // N_HOP                                # = 1 + (n + 512 - 512) // 256
    return (np.arange(nfr) * N_HOP)[:, None] + np.arange(N_FFT)[None, :]


def windowed_frames(pcm: np.ndarray) -> np.ndarray:
    """(T, 512) longdouble: reflect-pad by 256, hop-256 frames, times the reference's window."""
    d = pcm_as_float(pcm).astype(LD)
    padded = np.pad(d, N_FFT // 2, mode="reflect")
    return padded[_frame_index(len(d))] * orc.analysis_window().astype(LD)


def hpf_rows(x: np.ndarray, pole) -> np.ndarray:
    """lfilter([1, -1], [1, -pole]) along axis 1 as the explicit recurrence y = z + x,
    z = -x + pole * y, in the dtype of x."""
    y = np.empty_like(x)
    z = np.zeros(x.shape[0], x.dtype)
    for t in range(x.shape[1]):
        xt = x[:, t]
        yt = z + xt
        z = -xt + pole * yt
        y[:, t] = yt
    return y


def extended_sgram(pcm: np.ndarray):
    """(sgram (256, T), mag (257, T), frame_norms (T,)), all longdouble."""
    frames = windowed_frames(pcm)
    norms = np.sqrt(np.sum(frames * frames, axis=1))
    mag = np.abs(np.fft.rfft(frames, axis=1)).T          # complex256 -> longdouble
    smax = np.max(mag)
    if smax > 0:
        s = np.log(np.maximum(mag, smax / LD(1e6)))
        s = s - np.mean(s)                               # over all 257 x T values
    else:
        s = mag.copy()                                   # all-zero input: no log, no mean
    return hpf_rows(s, LD(HPF_POLE))[:-1, :], mag, norms


def float32_sgram(pcm: np.ndarray):
    """FP32 mode's arithmetic in NumPy: float32 frames x float32 window, float32 rfft, |X| and log;
    float64 floor, mean and high-pass.  Returns (sgram (256, T), mag (257, T)) as float64."""
    d = pcm_as_float(pcm)
    padded = np.pad(d, N_FFT // 2, mode="reflect")
    frames = padded[_frame_index(len(d))] * orc.analysis_window().astype(np.float32)
    mag32 = np.abs(np.fft.rfft(frames, axis=1)).T
    assert mag32.dtype == np.float32
    smax = float(np.max(mag32))
    if smax > 0:
        with np.errstate(divide="ignore"):
            lg = np.log(mag32).astype(np.float64)
        s = np.maximum(lg, np.log(smax / 1e6))
        s = s - np.mean(s)
    else:
        s = mag32.astype(np.float64)
    return hpf_rows(s, HPF_POLE)[:-1, :], mag32.astype(np.float64)


def mag_ratio(mag: np.ndarray, ext_mag: np.ndarray, norms: np.ndarray, u: float) -> float:
    """max over frames and bins of |mag - ext_mag| / (u ||x_w(t)||); a silent frame must be exact."""
    err = np.abs(np.asarray(mag, np.float64).astype(LD) - ext_mag)
    scale = LD(u) * norms[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(scale > 0, err / scale, np.where(err > 0, np.inf, 0.0))
    return float(np.max(r))


def sgram_err(sg: np.ndarray, ext_sg: np.ndarray) -> float:
    return float(np.max(np.abs(np.asarray(sg, np.float64).astype(LD) - ext_sg)))


def abs_hpf_rows(x: np.ndarray, pole: float = HPF_POLE) -> np.ndarray:
    """The high-pass filter with every tap of its impulse response (1, -(1-p), -(1-p)p, ...) made
    positive, along axis 1: g_t = x_t + (1-p) * sum_{j>=1} p^(j-1) x_{t-j}.  For e >= |x|,
    abs_hpf_rows(e) bounds |hpf(x)| element by element."""
    g = np.empty_like(x)
    acc = np.zeros(x.shape[0], x.dtype)
    for t in range(x.shape[1]):
        g[:, t] = x[:, t] + (1.0 - pole) * acc
        acc = pole * acc + x[:, t]
    return g


class K1Bars:
    """The extended reference of one input, the reference arithmetic's own error on it and the
    resulting bars, in the precisions given."""

    def __init__(self, pcm: np.ndarray, precisions=("fp64", "fp32")):
        self.sg, self.mag, self.norms = extended_sgram(pcm)
        self.sg_max = float(np.max(np.abs(self.sg)))
        self.mag_max = float(np.max(self.mag))
        # largest |log| of a floored magnitude
        self.log_max = max(abs(np.log(self.mag_max)), abs(np.log(self.mag_max / 1e6))) if self.mag_max > 0 else 0.0
        self.ref_sg, self.ref_mag = {}, {}
        if "fp64" in precisions:
            d = pcm_as_float(pcm)
            self.ref_sg["fp64"], self.ref_mag["fp64"] = orc.conditioned_sgram(d)
            self.ref_complex = orc.stft_complex(d)
        if "fp32" in precisions:
            self.ref_sg["fp32"], self.ref_mag["fp32"] = float32_sgram(pcm)
        self.ref_mag_ratio = {p: mag_ratio(m, self.mag, self.norms, U[p]) for p, m in self.ref_mag.items()}
        self.ref_sg_err = {p: sgram_err(s, self.sg) for p, s in self.ref_sg.items()}

    def mag_ratio(self, mag: np.ndarray, precision: str) -> float:
        return mag_ratio(mag, self.mag, self.norms, U[precision])

    def c_mag(self, precision: str) -> float:
        return max(C_MAG_MIN, C_MAG_OVER_REF * self.ref_mag_ratio[precision])

    def sg_err(self, sg: np.ndarray) -> float:
        return sgram_err(sg, self.sg)

    def log_err(self, precision: str) -> float:
        """Error of K1's log of one magnitude: the FP64 table log is within 1e-16 + 1 ulp of the
        result (a factor 4 to spare); FP32 mode's 0.5 * __logf(|X|^2) within half of __logf's."""
        if precision == "fp64":
            return 4.0 * U["fp64"] * (1.0 + self.log_max)
        return 0.5 * max(LOGF_ABS, LOGF_ULPS * 2.0 ** -23 * 2.0 * self.log_max)

    def _floor_terms(self, precision: str):
        """(D, dfloor, floor): the magnitude bar per element, how far K1's floor (max / 1e6 of its
        own magnitudes) can be from the extended one, and the extended floor."""
        dmag = (self.c_mag(precision) * U[precision] * self.norms.astype(np.float64))[None, :] * np.ones((NBINS, 1))
        return dmag, float(np.max(dmag)) * 1e-6, self.mag_max / 1e6

    def above_floor(self, precision: str) -> np.ndarray:
        """(256, T) mask of the elements that no magnitude within the bar can floor."""
        dmag, dfloor, floor = self._floor_terms(precision)
        return (self.mag.astype(np.float64) - dmag > floor + dfloor)[:-1, :]

    def sg_bound(self, precision: str) -> np.ndarray:
        """(256, T) bound on |S - S_ext| for an S whose magnitudes meet the magnitude bar.

        Log of a magnitude.  K1's floor is max(M) / 1e6 of its own magnitudes, so it is within
        dfloor = max(D) / 1e6 of the extended floor F, D = C_MAG u ||x_w(t)|| being the bar.
          * Certainly floored (M_ext + D below F - dfloor, with the log's error to spare): both sides
            take the floor, and the logs differ by at most dfloor / (F - dfloor) plus the FP64 log
            of the floor (the floor is applied in FP64 in both modes).
          * Otherwise the floored magnitudes differ by at most max(D, dfloor) and neither is below
            m_lo = max(M_ext - D, F - dfloor): the logs differ by at most max(D, dfloor) / m_lo
            plus the error of K1's log routine (log_err).
        Call that per-element bound lam.  The mean of the 257 x T logs then moves by at most
        mean(lam).  The high-pass filter h (taps 1, -(1-p), -(1-p)p, ...) maps the log errors to at
        most abs_hpf_rows(lam), and a constant shift c of its input to c * p^t at frame t (its step
        response).  C_SG_U u64 (max|S_ext| + the largest |log|) covers the rounding of the mean and
        of the filter, which run in FP64 in both modes."""
        T = self.mag.shape[1]
        if not self.mag_max > 0:
            return np.zeros((256, T))
        dmag, dfloor, floor = self._floor_terms(precision)
        mag = self.mag.astype(np.float64)
        lerr = self.log_err(precision)
        floored = (mag + dmag) * (1.0 + 2.0 * lerr) <= floor - dfloor
        m_lo = np.maximum(mag - dmag, floor - dfloor)
        lam = np.where(floored, dfloor / (floor - dfloor) + self.log_err("fp64"),
                       np.maximum(dmag, dfloor) / m_lo + lerr)
        step = HPF_POLE ** np.arange(T, dtype=np.float64)
        b = abs_hpf_rows(lam)[:-1, :] + float(np.mean(lam)) * step[None, :]
        return b + C_SG_U * U["fp64"] * (self.sg_max + self.log_max)

    def med_quantum(self) -> float:
        """What rounding the extended sgram to float64 for the comparison can add to a median."""
        return U["fp64"] * (1.0 + self.log_max)

    def sg_median_err(self, sg: np.ndarray, precision: str) -> float:
        """Median of |S - S_ext| over the elements above the floor (0 if there are none).  A
        median over many elements is not decided by the luck of one rounding at a quiet bin, so
        K1's can be compared with the reference arithmetic's."""
        m = self.above_floor(precision)
        if not np.any(m):
            return 0.0
        return float(np.median(np.abs(np.asarray(sg, np.float64)[m] - self.sg.astype(np.float64)[m])))

    def sg_use(self, sg: np.ndarray, precision: str) -> float:
        """max over elements of |S - S_ext| / sg_bound: at most 1 passes."""
        err = np.abs(np.asarray(sg, np.float64) - self.sg.astype(np.float64))
        b = self.sg_bound(precision)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(b > 0, err / b, np.where(err > 0, np.inf, 0.0))
        return float(np.max(r)) if r.size else 0.0


# ---- the inputs ---------------------------------------------------------------------------------
# Lengths around the reflection (N <= 512), and lengths giving T = 15, 16, 17, 31, 32, 33 frames
# (a tile is 16 frames) with N % 256 in {0, 1, 255}: the first tile's reflected head and the last
# tile's tail are staged by scalar loads, the rest by bulk copies.
LENGTHS = [1, 2, 3, 100, 255, 256, 257, 511, 512, 513] + \
          [(t - 1) * N_HOP + r for t in (15, 16, 17, 31, 32, 33) for r in (0, 1, 255)]
COSINE_BINS = [1, 64, 127, 128, 129, 255]
LONG_SECONDS = 400.0     # 17,227 frames, 1,077 tiles: every K1 CTA runs >= 2 persistent iterations

# name -> FP32 mode claimed for it (False: outside the range FP32 mode is stated for)
CASES = {}
CASES.update({"noise_s%d" % s: True for s in (0, 1, 2)})
CASES.update({"len_%d" % n: True for n in LENGTHS})
CASES.update({"fs_square": True, "fs_nyquist": True, "fs_dc": True})
CASES.update({"fs_cos_%d" % k: True for k in COSINE_BINS})
CASES.update({"dr_tone_lsb": True, "dr_lsb": True, "dr_clicks": True, "dr_zeros": True})
CASES.update({"f32_random": True, "f32_tiny": False, "f32_huge": False})
CASES["long_400s"] = True


def _lsb_noise(seed: int, n: int) -> np.ndarray:
    return np.random.default_rng(seed).integers(-1, 2, n).astype(np.int16)


def case_pcm(name: str) -> np.ndarray:
    """int16 or float32 PCM of a case of CASES, from its name alone."""
    n2 = 2 * SR
    if name.startswith("noise_s"):                       # the golden signals, 10 s
        return synth_track(int(name[7:]), 10.0)
    if name.startswith("len_"):
        n = int(name[4:])
        return synth_track(11, 1.0)[:n].copy()
    if name == "fs_square":                              # full-scale square wave: -32768 / +32767
        t = np.arange(n2)
        return np.where(np.sin(2 * np.pi * 441.0 * t / SR) >= 0, 32767, -32768).astype(np.int16)
    if name == "fs_nyquist":                             # +32767, -32768, ...: all energy at bin 256
        return np.where(np.arange(n2) % 2 == 0, 32767, -32768).astype(np.int16)
    if name == "fs_dc":                                  # bin 0, which K1 pairs with bin 256
        return np.full(n2, -32768, np.int16)
    if name.startswith("fs_cos_"):                       # a cosine centred on bin k, amplitude 30000
        k = int(name[7:])
        return np.round(30000.0 * np.cos(2 * np.pi * k * np.arange(n2) / N_FFT)).astype(np.int16)
    if name == "dr_tone_lsb":                            # > 120 dB of spectrum: the floor bites
        t = np.arange(3 * SR)
        x = np.round(30000.0 * np.sin(2 * np.pi * 1000.0 * t / SR)) + _lsb_noise(21, len(t))
        return x.astype(np.int16)
    if name == "dr_lsb":
        return _lsb_noise(22, 3 * SR)
    if name == "dr_clicks":                              # clicks over exact digital silence
        x = np.zeros(4 * SR, np.int16)
        x[100::2999] = 25000
        x[1600::2999] = -32768
        return x
    if name == "dr_zeros":
        return np.zeros(2 * SR, np.int16)
    if name.startswith("f32_"):                          # float PCM, not multiples of 1/32768
        x = np.random.default_rng(23).uniform(-0.9, 0.9, 3 * SR).astype(np.float32)
        scale = {"f32_random": 1.0, "f32_tiny": 2.0 ** -100, "f32_huge": 2.0 ** 100}[name]
        return (x * np.float32(scale)).astype(np.float32)
    if name == "long_400s":
        return synth_track(31, LONG_SECONDS)
    raise KeyError(name)
