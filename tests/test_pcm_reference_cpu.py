"""The extended-precision statement of the PCM front-end (tests/exact_resample.py) against
scipy.signal.resample_poly, and the teeth of its bar: a float64 emulation of the kernel's loop meets
`check_rounded`, a float32 accumulator and a round-toward-zero conversion do not.  CPU only."""
import numpy as np
import pytest
from scipy.signal import resample_poly

from tests.exact_resample import (LD, RATE_PAIRS, U53, check_rounded, downmix, noise_tone, reference, taps_for,
                                  terms, up_down)


def _kernel_emulation(mono, up, down, acc_dtype=np.float64, round_to_zero=False):
    """The kernel's loop in NumPy: j ascending (tap index descending), one accumulator per output."""
    ref_len = -(-len(mono) * up // down)
    t, x = terms(mono, up, down, taps_for(up, down), np.arange(ref_len), np.float64)
    t, x = t.astype(acc_dtype), x.astype(acc_dtype)
    acc = np.zeros(ref_len, acc_dtype)
    for i in reversed(range(t.shape[1])):
        acc += t[:, i] * x[:, i]
    out = acc.astype(np.float32)
    if round_to_zero:
        out = np.where(np.abs(out.astype(np.float64)) > np.abs(acc.astype(np.float64)),
                       np.nextafter(out, np.float32(0)), out)
    return out


def _mono(src, seconds=0.3, ch=2):
    return downmix(noise_tone(int(src * seconds) + 7, ch, src, src), ch)


@pytest.mark.parametrize("src,dst", RATE_PAIRS)
def test_statement_equals_resample_poly(src, dst):
    """Same taps, same centre n*down + half, same length as scipy's polyphase resampler.  scipy
    sums the m terms of an output serially in float64, so the bar is its worst case, 1.01 m u S."""
    up, down = up_down(src, dst)
    mono = _mono(src)
    ref, S, m = reference(mono, up, down)
    rp = resample_poly(mono.astype(np.float64), up, down)
    assert rp.shape == ref.shape
    err = np.abs(rp.astype(LD) - ref)
    assert np.all(err <= 1.01 * m * U53 * S), float(np.max(err / (U53 * S)))
    # the statement's outputs at a subset equal those of the whole signal
    n = np.array([0, 1, len(ref) // 2, len(ref) - 1])
    sub, S_sub, _ = reference(mono, up, down, n)
    assert np.array_equal(sub, ref[n]) and np.array_equal(S_sub, S[n])


def test_downmix_is_the_rounded_mean():
    rng = np.random.default_rng(5)
    for ch in (1, 2, 3, 6, 8, 16):
        raw = rng.integers(-32768, 32768, (4001, ch)).astype(np.int16)
        raw[0] = -32768
        want = [np.float32(float(int(r.astype(np.int64).sum())) / (32768.0 * ch)) for r in raw[:200]]
        assert np.array_equal(downmix(raw, ch)[:200], np.array(want, np.float32)), ch
        assert downmix(raw, ch)[0] == -1.0


@pytest.mark.parametrize("src,dst", [(44100, 11025), (48000, 11025), (8000, 11025), (44056, 11025)])
def test_bar_accepts_float64_and_rejects_float32_and_truncation(src, dst):
    up, down = up_down(src, dst)
    mono = _mono(src)
    ref, S, m = reference(mono, up, down)
    assert check_rounded(_kernel_emulation(mono, up, down), ref, S, m) <= 2
    with pytest.raises(AssertionError, match="not correctly rounded"):
        check_rounded(_kernel_emulation(mono, up, down, acc_dtype=np.float32), ref, S, m)
    with pytest.raises(AssertionError, match="not correctly rounded"):
        check_rounded(_kernel_emulation(mono, up, down, round_to_zero=True), ref, S, m)


def test_check_rounded_tie_zone():
    """A sum exactly on a float32 boundary is a tie-zone sample; either neighbour passes."""
    ref = np.array([LD(1) + LD(2.0 ** -24), LD(0.75)], LD)
    S = np.array([1.0, 1.0])
    for got0 in (np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(2))):
        assert check_rounded(np.array([got0, 0.75], np.float32), ref, S, 2) == 1
    with pytest.raises(AssertionError, match="not correctly rounded"):
        check_rounded(np.array([1.0, np.nextafter(np.float32(0.75), np.float32(1))], np.float32), ref, S, 2)
