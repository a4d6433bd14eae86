"""Reference for the K2 -> K3 -> merge chain on a given log-magnitude spectrogram.

It composes the oracle's own functions (oracle/afp_oracle.py) and nothing else, so that
`tests/test_k2k3_reference_cpu.py` can show it equal to `orc.find_peaks` / `orc.fingerprint` on the
oracle's own logs, and `tests/test_gpu_k2_k3_constructed.py` can hold the CUDA chain to it on
constructed spectrograms that PCM never produces.

An item is (logs, logfloor, mean, allzero) with `logs` float [T][256] in the device layout
(frame-major), the same numbers afp_fingerprint_from_logs takes.  float32 logs (the FP32
spectrogram mode) are widened to float64, as K2 does.
"""
from __future__ import annotations

import numpy as np

from oracle import afp_oracle as orc

NBINS = 256


class Params:
    """The analyzer settings the chain depends on (audfprint_analyze.py:125-151)."""

    def __init__(self, density=20.0, f_sd=30.0, maxpks=5, fanout=3, mindt=2, targetdt=63, targetdf=31,
                 shifts=1):
        self.density, self.f_sd, self.maxpks, self.fanout = float(density), float(f_sd), int(maxpks), int(fanout)
        self.mindt, self.targetdt, self.targetdf, self.shifts = int(mindt), int(targetdt), int(targetdf), int(shifts)

    def __repr__(self):
        return "Params(%s)" % ", ".join("%s=%r" % kv for kv in sorted(vars(self).items()))


def item_sgram(logs, lf, mean):
    """Floor, mean removal, high-pass (audfprint_analyze.py:286-295): (256, T) float64."""
    x = np.maximum(np.asarray(logs, np.float64).T, lf) - mean
    return orc.hpf_rows(x)


def item_peaks(item, p: Params, detail=False):
    """Analyzer.find_peaks from the logs on: list of (col, bin), column-major, bins ascending.
    With detail=True also (sgram, forward accepted lists) for the callers' edge checks."""
    logs, lf, mean, allzero = item
    T = len(logs)
    if T == 0 or allzero:      # the reference skips log and mean; a zero sgram has no peaks (:287-290)
        return ([], None, []) if detail else []
    s = item_sgram(logs, lf, mean)
    etab = orc.gaussian_table(NBINS, p.f_sd)
    a_dec = orc.decay_constant(p.density)
    acc = orc.forward_prune(s, a_dec, etab, p.maxpks)
    keep = orc.backward_prune(s, acc, a_dec, etab)
    cols, bins = np.nonzero(keep.T)
    pk = list(zip(cols.tolist(), bins.tolist()))
    return (pk, s, acc) if detail else pk


def file_hashes(peak_lists, p: Params):
    """peaks2landmarks + landmarks2hashes of every shift's list, then the union over shifts
    (audfprint_analyze.py:310-343, 81-96, 401-422)."""
    rows = np.concatenate([orc.landmarks_to_hashes(orc.peaks_to_landmarks(pl, p.fanout, p.mindt, p.targetdt,
                                                                          p.targetdf))
                           for pl in peak_lists])
    return orc.unique_rows(rows)


def forward_thresholds(s, acc, p: Params):
    """The threshold each column of the forward pass is compared with, replayed from the accepted
    lists with the oracle's arithmetic (audfprint_analyze.py:204-230): (256, T)."""
    nb, T = s.shape
    etab = orc.gaussian_table(nb, p.f_sd)
    a_dec = orc.decay_constant(p.density)
    thr = orc.spread_local_maxes(np.max(s[:, :min(10, T)], axis=1), etab)
    out = np.empty_like(s)
    for t in range(T):
        out[:, t] = thr
        for val, b in acc[t]:
            thr = np.maximum(thr, val * etab[nb - b: 2 * nb - b])
        thr = thr * a_dec
    return out


def candidate_counts(s, acc, p: Params):
    """Forward candidates per column (local maxima above the threshold), before the maxpks cap."""
    thr = forward_thresholds(s, acc, p)
    return np.array([int(np.count_nonzero(orc.local_max_mask(s[:, t]) & (s[:, t] > thr[:, t])))
                     for t in range(s.shape[1])], np.int64)
