"""GPU: K2 (peak picking), K3 (pairing) and the cross-shift merge on constructed spectrograms and
peak lists, bit for bit against the oracle-composed reference of tests/k2k3_reference.py.

From PCM, K2 and K3 only ever see continuous noise: exact ties, values that share their high word,
plateaus across the lanes' 8-bin boundaries, saturated columns, comparisons at equality and
subnormal thresholds practically never occur.  afp_fingerprint_from_logs feeds the product's K2 ->
K3 -> merge launchers a given log spectrogram instead, so each family below builds the case it
targets, asserts on the reference side that the case is really reached, and then asks for the
peaks of every shift and the hashes of every file to be identical, in FP64 and in FP32 mode (float
logs, widened to double by K2 and by the reference alike).

K3 is also checked through afp_landmarks_from_peaks (Analyzer.peaks2landmarks) on dense peak lists
across its pairing parameters, on lists whose columns cross 2^20, and on one PCM file longer than
2^20 frames."""
import ctypes as C

import numpy as np
import pytest
import scipy.ndimage

from audfprint_b200 import Analyzer
from oracle import afp_oracle as orc
from tests import k2k3_reference as ref

pytestmark = pytest.mark.gpu

PRECISIONS = ("fp64", "fp32")
NB = 256


# ---- device side ----------------------------------------------------------------------------------
def analyzer(p, precision="fp64"):
    an = Analyzer(density=p.density)
    an.f_sd, an.maxpksperframe, an.maxpairsperpeak = p.f_sd, p.maxpks, p.fanout
    an.mindt, an.targetdt, an.targetdf, an.shifts = p.mindt, p.targetdt, p.targetdf, p.shifts
    an.precision = precision
    return an


def fetch_peaks(ctx, shift, nfiles):
    poff = np.empty(nfiles + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, shift, None, 1, poff.ctypes.data_as(C.POINTER(C.c_int64))))
    rows = np.empty((int(poff[-1]), 2), np.int32)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, shift, rows.ctypes.data, 1, None))
    return [rows[poff[f]:poff[f + 1]] for f in range(nfiles)]


def device_run(p, files, precision):
    """files: [file][shift] items (logs [T][256], logfloor, mean, allzero) ->
    (peaks [shift][file] int32 (n,2), hashes [file] int32 (n,2)) from afp_fingerprint_from_logs."""
    ctx = analyzer(p, precision)._configure(p.shifts)
    items = [it for f in files for it in f]
    frames = np.array([len(it[0]) for it in items], np.int32)
    stats = np.array([[it[1], it[2], 1.0 if it[3] else 0.0] for it in items], np.float64).reshape(-1, 3)
    dt = np.float32 if precision == "fp32" else np.float64
    logs = np.ascontiguousarray(np.concatenate([np.asarray(it[0], dt).reshape(-1, NB) for it in items]))
    total = C.c_int64(-1)
    ctx.check(ctx.lib.afp_fingerprint_from_logs(ctx.h, logs.ctypes.data, 1, len(files), frames.ctypes.data,
                                                stats.ctypes.data, C.byref(total)))
    rows = np.empty((int(total.value), 2), np.int32)
    roff = np.empty(len(files) + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, rows.ctypes.data, 1, roff.ctypes.data_as(C.POINTER(C.c_int64))))
    peaks = [fetch_peaks(ctx, s, len(files)) for s in range(p.shifts)]
    return peaks, [rows[roff[f]:roff[f + 1]] for f in range(len(files))]


def check(p, files, precision):
    """Reference vs device for every item and file; returns the reference's (peaks, sgram, accepted)
    per item, file-major, for the family's edge checks."""
    dt = np.float32 if precision == "fp32" else np.float64
    files = [[(np.asarray(logs, dt).reshape(-1, NB), float(lf), float(mean), bool(az)) for logs, lf, mean, az in f]
             for f in files]
    assert all(len(f) == p.shifts for f in files)
    detail = [[ref.item_peaks(it, p, detail=True) for it in f] for f in files]
    want_h = [ref.file_hashes([d[0] for d in fd], p) for fd in detail]
    got_pk, got_h = device_run(p, files, precision)
    for fi, fd in enumerate(detail):
        for s, d in enumerate(fd):
            want = np.asarray(d[0], np.int32).reshape(-1, 2)
            assert np.array_equal(got_pk[s][fi], want), (p, precision, "peaks", fi, s)
        assert np.array_equal(got_h[fi], want_h[fi]), (p, precision, "hashes", fi)
    return [d for fd in detail for d in fd]


def one_shift(items):
    return [[it] for it in items]


def smooth_logs(rng, T, tsd=2.0, fsd=3.0, scale=4.0, offset=-2.0):
    """A smooth random log spectrogram [T][256]: white noise blurred in time and frequency."""
    if T == 0:
        return np.zeros((0, NB))
    x = scipy.ndimage.gaussian_filter(rng.standard_normal((T, NB)), (tsd, fsd), mode="wrap")
    return offset + scale * x / max(np.std(x), 1e-12)


def floored_item(logs, q=0.05):
    """(logs, logfloor, mean, False) with the floor at the q-quantile and the mean of the floored logs."""
    lf = float(np.quantile(logs, q)) if logs.size else 0.0
    return logs, lf, float(np.mean(np.maximum(logs, lf))) if logs.size else 0.0, False


def accepted(details):
    return sum(len(lst) for _, _, acc in details for lst in acc)


def final(details):
    return sum(len(pk) for pk, _, _ in details)


# ---- K2 families ------------------------------------------------------------------------------------
SMOOTH = [  # (density, f_sd, maxpks)
    (20.0, 30.0, 5), (10.0, 2.0, 1), (100.0, 60.0, 3), (100.0, 2.0, 16), (10.0, 60.0, 16), (20.0, 2.0, 3),
    (100.0, 30.0, 1), (10.0, 30.0, 5)]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("density,f_sd,maxpks", SMOOTH)
def test_smooth_random_fields(precision, density, f_sd, maxpks):
    rng = np.random.default_rng(int(density) * 1000 + int(f_sd) * 17 + maxpks)
    p = ref.Params(density=density, f_sd=f_sd, maxpks=maxpks, shifts=2)
    files = []
    for T in (40, 150, 333):
        a = floored_item(smooth_logs(rng, T, tsd=rng.uniform(0.5, 3), fsd=rng.uniform(0.7, 3)))
        b = floored_item(smooth_logs(rng, T - 1, tsd=1.0, fsd=1.0))
        files.append([a, b])
    det = check(p, files, precision)
    assert final(det) > 50 and accepted(det) > 150
    assert sum(1 for _, _, acc in det for lst in acc if len(lst) >= min(maxpks, 2)) > 10


def tie_items(rng, ngroups, T, nitems):
    """Quantised logs in which groups of bins share identical rows: their high-passed values tie exactly."""
    out = []
    for _ in range(nitems):
        grp = rng.integers(0, ngroups, NB)
        base = rng.integers(0, 6, (ngroups, T)).astype(np.float64)
        out.append((base[grp].T.copy(), -1.0, 2.5, False))
    return out


def tie_pairs(details):
    """Consecutive accepted entries of one column with equal values, as (bin, bin) pairs."""
    return [(b1, b2) for _, _, acc in details for lst in acc
            for (v1, b1), (v2, b2) in zip(lst, lst[1:]) if v1 == v2]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("density,f_sd,maxpks", [(100.0, 4.0, 16), (20.0, 30.0, 5), (100.0, 2.0, 3)])
def test_exact_ties_are_ranked_by_bin(precision, density, f_sd, maxpks):
    rng = np.random.default_rng(7 + maxpks)
    p = ref.Params(density=density, f_sd=f_sd, maxpks=maxpks)
    det = check(p, one_shift(tie_items(rng, 40, 400, 3)), precision)
    pairs = tie_pairs(det)
    assert len(pairs) >= (1000 if maxpks == 16 else 50)
    assert any(b1 // 8 == b2 // 8 for b1, b2 in pairs)                  # within a lane
    assert any(b1 // 8 != b2 // 8 for b1, b2 in pairs)                  # across lanes
    if maxpks == 16:
        assert any(min(b1, b2) < 8 for b1, b2 in pairs)                 # lane 0
        assert any(max(b1, b2) >= 248 for b1, b2 in pairs)              # lane 31


def low_word_items(rng, nitems):
    """Column 0 holds 128 local maxima (odd bins) whose values share their high 32 bits and differ in
    the low word; column 1 is loud on the even bins, so that the initial threshold (a spread of the
    per-bin max of the first 10 columns) stays below column 0's odd bins.  With mean 0 and no floor,
    column 0 of the sgram is the logs themselves (y = 0 + x)."""
    out = []
    hi = np.float64(10.0).view(np.uint64) & np.uint64(0xFFFFFFFF00000000)
    for k in range(nitems):
        T = 2 + k % 11
        logs = rng.uniform(0.0, 3.0, (T, NB))
        lo = rng.integers(0, 1 << 32, NB // 2, dtype=np.uint64)
        logs[0, 1::2] = (hi | lo).view(np.float64)
        logs[0, 0::2] = 0.0
        if T > 1:
            logs[1, 0::2], logs[1, 1::2] = 11.0, 0.0
        out.append((logs, -np.inf, 0.0, False))
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("maxpks", [16, 5])
def test_values_that_differ_in_the_low_word(precision, maxpks):
    rng = np.random.default_rng(99 + maxpks)
    p = ref.Params(density=20.0, f_sd=2.0, maxpks=maxpks)
    det = check(p, one_shift(low_word_items(rng, 48)), precision)
    if precision == "fp64":
        # ranking column 0's candidates by (high word, bin) alone would accept other peaks
        differ = 0
        for _, s, acc in det:
            thr = ref.forward_thresholds(s, acc, p)[:, 0]
            cand = np.nonzero(orc.local_max_mask(s[:, 0]) & (s[:, 0] > thr))[0]
            assert len(cand) > maxpks
            hi_only = sorted(((int(s[b, 0].view(np.uint64) >> np.uint64(32)), int(b)) for b in cand),
                             reverse=True)[:maxpks]
            differ += [b for _, b in hi_only] != [b for _, b in acc[0]]
        assert differ == len(det)


def plateau_items(rng, T, nitems):
    """Rows grouped in contiguous runs of equal logs (hence equal sgram rows): plateaus that end on
    the lane boundaries 7|8, 15|16, 247|248, at bin 0 and at bin 255, plus wholly flat items."""
    forced = [(8, 16, 248), (9, 17, 249), (7, 15, 247), (1, 8, 255), (2, 16, 254)]
    out = []
    for k in range(nitems):
        if k % 6 == 5:
            cuts = [0, NB]                                              # every column flat
        else:
            cuts = sorted(set([0, NB] + list(forced[k % 5]) + rng.integers(1, NB, 30).tolist()))
        runs = np.zeros(NB, np.int64)
        for r, (a, b) in enumerate(zip(cuts, cuts[1:])):
            runs[a:b] = r
        heights = rng.integers(0, 8, (len(cuts) - 1, T)).astype(np.float64)
        out.append((heights[runs].T.copy(), -1.0, 3.0, False))
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("maxpks", [5, 16])
def test_plateaus_across_lane_boundaries(precision, maxpks):
    rng = np.random.default_rng(31 + maxpks)
    p = ref.Params(density=100.0, f_sd=4.0, maxpks=maxpks)
    det = check(p, one_shift(plateau_items(rng, 200, 12)), precision)
    right_ends = [(b, t) for _, s, acc in det for t, lst in enumerate(acc) for _, b in lst
                  if b > 0 and s[b - 1, t] == s[b, t]]
    assert any(b in (8, 16, 248) for b, _ in right_ends)                # plateau across a lane boundary
    assert any(b % 8 != 0 for b, _ in right_ends)                       # plateau inside a lane
    assert any(b in (7, 15, 247) for b, _ in right_ends)
    flat = [det[k] for k in range(len(det)) if k % 6 == 5]
    assert all(b == 255 for _, _, acc in flat for lst in acc for _, b in lst)
    assert accepted(flat) > 0


def saturation_items(rng, T, nitems):
    """Every odd bin a local maximum with a random level: far more candidates per column than maxpks."""
    out = []
    for _ in range(nitems):
        logs = np.zeros((T, NB))
        logs[:, 1::2] = rng.uniform(2.0, 8.0, (T, NB // 2))
        out.append((logs, -1.0, 1.0, False))
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("maxpks", list(range(1, 17)))
def test_saturated_columns(precision, maxpks):
    rng = np.random.default_rng(500 + maxpks)
    p = ref.Params(density=100.0, f_sd=2.0, maxpks=maxpks)
    det = check(p, one_shift(saturation_items(rng, 120, 2)), precision)
    over = sum(int(np.count_nonzero(ref.candidate_counts(s, acc, p) > maxpks)) for _, s, acc in det)
    assert over >= 100
    assert max(len(lst) for _, _, acc in det for lst in acc) == maxpks


def equality_items(rng, nitems):
    """Column 0 is the loudest of the first 10 columns: its local maxima meet a threshold equal to
    their own value (s > thr fails by equality).  The last column is a loud onset of isolated spikes:
    the backward pass starts from their spread, equal to their own values at the spikes (val >= thr
    passes by equality)."""
    out = []
    for k in range(nitems):
        T = 12 + 7 * k
        logs = rng.uniform(0.0, 1.0, (T, NB))
        logs[0] += 6.0 + 2.0 * np.sin(np.arange(NB) / (3.0 + k))
        spikes = rng.choice(NB, 6, replace=False)
        logs[-1, spikes] += rng.uniform(20.0, 30.0, 6)
        out.append((logs, -1.0, 0.5, False))
    return out


@pytest.mark.parametrize("precision", PRECISIONS)
def test_comparisons_at_equality(precision):
    rng = np.random.default_rng(4242)
    p = ref.Params(density=20.0, f_sd=2.0, maxpks=5)
    det = check(p, one_shift(equality_items(rng, 10)), precision)
    etab = orc.gaussian_table(NB, p.f_sd)
    fwd_eq = bwd_eq = 0
    for pk, s, acc in det:
        thr0 = ref.forward_thresholds(s, acc, p)[:, 0]
        fwd_eq += int(np.count_nonzero(orc.local_max_mask(s[:, 0]) & (s[:, 0] == thr0)))
        spread = orc.spread_local_maxes(s[:, -1], etab)
        T = s.shape[1]
        kept = [v for v, b in acc[-1] if v == spread[b] and (T - 1, b) in pk]
        bwd_eq += len(kept)
    assert fwd_eq >= 10 and bwd_eq >= 10


def test_floor_and_empty_items():
    rng = np.random.default_rng(77)
    T = 90
    partly = floored_item(smooth_logs(rng, T), q=0.5)
    with_inf = smooth_logs(rng, T)
    with_inf[rng.random((T, NB)) < 0.2] = -np.inf
    lf = float(np.quantile(with_inf[np.isfinite(with_inf)], 0.1))
    at_floor = np.full((T, NB), -3.0)
    below = at_floor - rng.uniform(0.0, 5.0, (T, NB))
    decreasing = -1.0 - 0.5 * np.arange(T)[:, None] - rng.uniform(0.0, 0.3, NB)[None, :]
    items = [partly,
             (with_inf, lf, float(np.mean(np.maximum(with_inf, lf))), False),
             (at_floor, -3.0, -3.5, False),                             # the whole item at the floor
             (below, -3.0, -3.0, False),                                # every log below the floor
             (smooth_logs(rng, T), 0.0, 0.0, True),                     # all-zero input: no peaks whatever the logs
             (np.zeros((0, NB)), 0.0, 0.0, False),
             (decreasing, -np.inf, 0.0, False)]                         # all-negative sgram
    for precision in PRECISIONS:
        for p in (ref.Params(), ref.Params(density=100.0, f_sd=4.0, maxpks=16)):
            det = check(p, one_shift(items), precision)
            assert len(det[0][0]) > 0 and len(det[1][0]) > 0
            assert all(len(d[0]) == 0 for d in det[3:])
            assert np.max(det[6][1]) < 0.0


@pytest.mark.parametrize("precision", PRECISIONS)
def test_subnormal_thresholds_and_peaks(precision):
    """A loud start, then 37,000 columns of one constant level, at density 100: the high-passed values
    decay as 0.98^t and the thresholds faster, into subnormal numbers, where peaks are still accepted."""
    rng = np.random.default_rng(2)
    T = 37003
    logs = np.full((T, NB), -12.0)
    logs[:3] = -12.0 + rng.normal(0.0, 3.0, (3, NB))
    p = ref.Params(density=100.0)
    det = check(p, [[(logs, -30.0, -12.0, False)]], precision)
    pk, s, acc = det[0]
    tiny = np.finfo(np.float64).tiny
    assert sum(1 for t, b in pk if 0.0 < s[b, t] < tiny) >= 10
    assert sum(1 for lst in acc for v, _ in lst if v < tiny) >= 10


@pytest.mark.parametrize("precision", PRECISIONS)
def test_item_lengths_and_shift_items(precision):
    """T = 0..17 (the initial 10-column window, the 4-column chunks of the 2-stage ring), 31-33, 1000
    and 7752; per file the 4 shift items are: T frames, one frame fewer, a copy of shift 0 (every hash
    a duplicate), one frame fewer again."""
    rng = np.random.default_rng(1234)
    p = ref.Params(density=100.0, maxpks=5, shifts=4)
    files = []
    for T in list(range(18)) + [31, 32, 33, 1000, 7752]:
        a = floored_item(smooth_logs(rng, T, tsd=0.7, fsd=2.0))
        b = floored_item(smooth_logs(rng, max(T - 1, 0), tsd=0.7, fsd=2.0))
        d = floored_item(smooth_logs(rng, max(T - 1, 0), tsd=0.7, fsd=2.0))
        files.append([a, b, a, d])
    det = check(p, files, precision)
    short = [det[4 * T][0] for T in range(1, 18)]
    assert sum(1 for pk in short if pk) >= 12
    assert all(len(det[4 * f][0]) == len(det[4 * f + 2][0]) for f in range(len(files)))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_batch_beyond_one_wave(precision):
    """1,400 items: more than the 1,320 K2 CTAs (10 per SM) resident at once on a 132-SM H100."""
    rng = np.random.default_rng(8)
    p = ref.Params()
    items = [floored_item(smooth_logs(rng, int(rng.integers(16, 40)), tsd=0.8)) for _ in range(1400)]
    det = check(p, one_shift(items), precision)
    assert sum(1 for pk, _, _ in det[1320:] if pk) >= 60


# ---- K3 --------------------------------------------------------------------------------------------
def dense_peaks(rng, cols, maxpks, full=0.8):
    """(col, bin) rows, column-major with bins ascending: maxpks peaks in most columns."""
    rows = []
    for c in cols:
        n = maxpks if rng.random() < full else int(rng.integers(0, maxpks + 1))
        for b in np.sort(rng.choice(NB, n, replace=False)):
            rows.append((int(c), int(b)))
    return rows


PAIRING = [  # (mindt, targetdt, targetdf, fanout)
    (0, 3, 1, 1), (0, 63, 31, 16), (0, 64, 32, 7), (1, 3, 32, 16), (1, 63, 1, 4), (1, 64, 31, 12),
    (2, 3, 31, 2), (2, 63, 32, 16), (2, 64, 1, 9), (2, 63, 31, 3), (0, 17, 8, 5), (1, 40, 20, 6),
    (2, 5, 2, 8), (0, 33, 16, 10), (1, 9, 31, 11), (2, 50, 12, 13), (0, 64, 31, 14), (1, 63, 32, 15)]


def landmarks(an, pk):
    return np.asarray(an.peaks2landmarks(pk), np.int32).reshape(-1, 4)


def oracle_landmarks(pk, p):
    return np.asarray(orc.peaks_to_landmarks(pk, p.fanout, p.mindt, p.targetdt, p.targetdf), np.int32).reshape(-1, 4)


@pytest.mark.parametrize("mindt,targetdt,targetdf,fanout", PAIRING)
def test_peaks2landmarks_pairing_parameters(mindt, targetdt, targetdf, fanout):
    """Dense lists (16 peaks in most columns) over 1,400 columns: past two landmark windows
    (about 640 source columns each at maxpks 16)."""
    rng = np.random.default_rng(mindt * 10000 + targetdt * 100 + targetdf + fanout)
    p = ref.Params(maxpks=16, fanout=fanout, mindt=mindt, targetdt=targetdt, targetdf=targetdf)
    pk = dense_peaks(rng, range(1400), 16)
    want = oracle_landmarks(pk, p)
    assert len(want) > 1000
    assert np.array_equal(landmarks(analyzer(p), pk), want)


@pytest.mark.parametrize("maxpks", [1, 16])
def test_peaks2landmarks_across_column_2_20(maxpks):
    """Peak columns just below and above 2^20: K3 packs a column into 20 bits of shared memory."""
    rng = np.random.default_rng(20 + maxpks)
    p = ref.Params(maxpks=maxpks, fanout=3)
    cols = list(range((1 << 20) - 1500, (1 << 20) + 1500))
    pk = dense_peaks(rng, cols, maxpks, full=0.5)
    want = oracle_landmarks(pk, p)
    assert np.any(want[:, 0] >= 1 << 20) and np.any(want[:, 0] + want[:, 3] >= 1 << 20)
    assert np.any(want[:, 0] < 1 << 20)
    assert np.array_equal(landmarks(analyzer(p), pk), want)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("shifts,fanout,mindt,targetdt,targetdf", [
    (1, 16, 2, 63, 31), (2, 8, 0, 64, 32), (4, 4, 1, 3, 1), (4, 4, 0, 63, 31)])
def test_hook_full_merge_buffer(precision, shifts, fanout, mindt, targetdt, targetdf):
    """maxpks 16 with shifts*maxpks*fanout = 256: the merge buffer of one (file, column) can fill."""
    rng = np.random.default_rng(shifts * 100 + fanout + mindt)
    p = ref.Params(density=100.0, f_sd=2.0, maxpks=16, fanout=fanout, mindt=mindt, targetdt=targetdt,
                   targetdf=targetdf, shifts=shifts)
    T = 1400
    files = [[saturation_items(rng, T - (s > 0), 1)[0] for s in range(shifts)] for _ in range(2)]
    check(p, files, precision)
    want = ref.file_hashes([ref.item_peaks(files[0][s], p) for s in range(shifts)], p)
    assert np.max(np.bincount(want[:, 0])) >= (4 if targetdf == 1 else 128)


def test_fingerprint_of_a_file_longer_than_2_20_frames():
    """One PCM file of 2^20 + 3,000 frames (6.8 h at 11025 Hz): digital silence with a noise burst
    around frame 2^20.  Its hashes must be the oracle's pairing, hashing and union applied to the
    peaks the GPU itself found (the oracle's K2 over a million columns would take too long)."""
    rng = np.random.default_rng(5)
    n = ((1 << 20) + 3000) * 256
    pcm = np.zeros(n, np.int16)
    lo, hi = ((1 << 20) - 2500) * 256, ((1 << 20) + 2500) * 256
    pcm[lo:hi] = np.clip(rng.normal(0.0, 3000.0, hi - lo), -32768, 32767).astype(np.int16)
    for shifts in (1, 2):
        p = ref.Params(shifts=shifts)
        an = analyzer(p)
        got = an.fingerprint_batch([pcm])[0]
        ctx = an._configure(shifts)
        peaks = [[tuple(r) for r in fetch_peaks(ctx, s, 1)[0].tolist()] for s in range(shifts)]
        assert min(c for c, _ in peaks[0]) < (1 << 20) - 1000 and max(c for c, _ in peaks[0]) > (1 << 20) + 1000
        assert np.array_equal(got, ref.file_hashes(peaks, p)), shifts
