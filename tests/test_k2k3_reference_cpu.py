"""CPU: the K2/K3 reference of tests/k2k3_reference.py, applied to the oracle's own logs, gives
exactly orc.find_peaks and orc.fingerprint.  With tests/test_oracle_golden.py (oracle == live
reference) this closes the chain CUDA == helper == oracle == reference that
tests/test_gpu_k2_k3_constructed.py relies on."""
import numpy as np
import pytest

from audfprint_b200.synth import synth_track, pcm_to_float
from oracle import afp_oracle as orc
from tests import cases
from tests import k2k3_reference as ref


def oracle_item(d):
    """(logs [T][256], logfloor, mean, allzero) as K1 hands them to K2, from the oracle's STFT:
    log|X| without the Nyquist row, log(max/1e6), and the mean of the floored 257-row logs."""
    mag = np.abs(orc.stft_complex(d))
    smax = np.max(mag)
    if smax == 0.0:
        return np.zeros((mag.shape[1], 256)), 0.0, 0.0, True
    floor = smax / 1e6
    with np.errstate(divide="ignore"):
        logs = np.log(mag)[:-1].T.copy()
    return logs, float(np.log(floor)), float(np.mean(np.log(np.maximum(mag, floor)))), False


def check(d, shifts, p):
    if len(d) == 0:
        return
    offs = orc.shift_offsets(shifts) if shifts > 1 else [0]
    lists = []
    for off in offs:
        # a shift past the end of the signal is an item without frames
        pk = ref.item_peaks(oracle_item(d[off:]) if len(d) > off else (np.zeros((0, 256)), 0.0, 0.0, False), p)
        assert pk == orc.find_peaks(d[off:], p.density, p.f_sd, p.maxpks), (shifts, off)
        lists.append(pk)
    assert np.array_equal(ref.file_hashes(lists, p),
                          orc.fingerprint(d, p.density, p.fanout, shifts, p.f_sd, p.maxpks)), shifts


@pytest.mark.parametrize("name,seed,secs", cases.NOISE_CASES)
def test_helper_equals_oracle_on_noise_cases(name, seed, secs):
    d = pcm_to_float(synth_track(seed, secs))
    check(d, 1, ref.Params())
    if secs <= 10:
        check(d, 4, ref.Params(shifts=4))


@pytest.mark.parametrize("name", cases.ADVERSARIAL)
def test_helper_equals_oracle_on_adversarial_cases(name):
    d = pcm_to_float(cases.adversarial_pcm(name))
    check(d, 1, ref.Params())
    check(d, 4, ref.Params(shifts=4))


@pytest.mark.parametrize("name,seed,secs,dens,fan", cases.DENSITY_CASES)
def test_helper_equals_oracle_at_other_densities(name, seed, secs, dens, fan):
    d = pcm_to_float(synth_track(seed, secs))
    check(d, 1, ref.Params(density=dens, fanout=fan))


def test_forward_thresholds_replay_the_forward_pass():
    """The edge checks of the GPU tests count candidates with thresholds replayed from the accepted
    lists; on a real track that replay accepts exactly what forward_prune accepted."""
    p = ref.Params(density=100.0, f_sd=4.0, maxpks=3)
    d = pcm_to_float(synth_track(3, 5.0))
    pk, s, acc = ref.item_peaks(oracle_item(d), p, detail=True)
    thr = ref.forward_thresholds(s, acc, p)
    for t in range(s.shape[1]):
        cand = np.nonzero(orc.local_max_mask(s[:, t]) & (s[:, t] > thr[:, t]))[0]
        assert sorted(((s[b, t], int(b)) for b in cand), reverse=True)[:p.maxpks] == acc[t]
    assert np.count_nonzero(ref.candidate_counts(s, acc, p) > p.maxpks) > 10
