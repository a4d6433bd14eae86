"""K3 (one CTA per file, peaks paired into shared-memory hash slots, sorted unique rows per column) and
the item statistics (floored tile sums whose last CTA re-reduces the item) of the fingerprint batch.

- K3: the hashes of every file equal the reference's pairing, hashing and union over shifts applied to
  the peaks the device itself found (tests/k2k3_reference.py), at shifts 1 to 4, maxpks up to 16 and
  shifts * maxpks * fanout up to 256.  The batch holds an empty file, a file shorter than one frame,
  one shorter than a K3 window and files of many windows with pairs across window boundaries.
- Statistics: a batch mixing digital silence, an all-negative item (logs below 0 everywhere), items
  whose floor bites and normal items gives each file the hashes it has alone, and the hashes and
  conditioned spectrograms recorded in tests/golden/k3_stats.npz from the three-launch statistics
  path and the landmark / merge K3 that these kernels replace (tools/make_golden_k3_stats.py).
- The chunked host-PCM path (K3 per chunk on its own stream, one scan and gather after the join)
  gives the device-resident path's rows and offsets."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

from audfprint_b200 import Analyzer
from audfprint_b200.synth import synth_track, SR
from tests import cases
from tests import k2k3_reference as ref

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "k3_stats.npz")
K3_SLOTS, K3_THREADS = 4096, 256   # afp_hash.cu


def k3_window(shifts, maxpks, fanout):
    w = K3_SLOTS // (shifts * maxpks * fanout)
    return w // K3_THREADS * K3_THREADS if w >= K3_THREADS else w


def analyzer(p):
    an = Analyzer(density=p.density)
    an.maxpksperframe, an.maxpairsperpeak = p.maxpks, p.fanout
    an.mindt, an.targetdt, an.targetdf, an.shifts = p.mindt, p.targetdt, p.targetdf, p.shifts
    return an


def fetch_peaks(ctx, shift, nfiles):
    poff = np.empty(nfiles + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, shift, None, 1, poff.ctypes.data_as(C.POINTER(C.c_int64))))
    rows = np.empty((int(poff[-1]), 2), np.int32)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, shift, rows.ctypes.data, 1, None))
    return [rows[poff[f]:poff[f + 1]] for f in range(nfiles)]


def reference_hashes(peak_lists, p):
    lists = [[tuple(r) for r in pk.tolist()] for pk in peak_lists]
    if not any(lists):
        return np.zeros((0, 2), np.int32)
    return np.asarray(ref.file_hashes([pl for pl in lists if pl], p), np.int32).reshape(-1, 2)


def k3_files():
    return [np.zeros(0, np.int16),                         # empty
            synth_track(31, 1.0)[:100].copy(),             # one frame
            synth_track(32, 1.0)[:2000].copy(),            # 8 frames: inside one window at any setting
            synth_track(33, 2.0),                          # 87 frames
            synth_track(34, 25.0)[:275001].copy(),         # 1,075 frames: many windows, ragged end
            cases.adversarial_pcm("silence_gap")]


@pytest.mark.parametrize("shifts,maxpks,fanout,density", [
    (1, 5, 3, 20.0), (1, 16, 16, 100.0), (2, 16, 8, 100.0), (3, 7, 12, 70.0), (4, 16, 4, 100.0),
    (4, 1, 1, 20.0), (4, 5, 3, 20.0), (2, 3, 2, 50.0)])
def test_k3_hashes_against_reference(shifts, maxpks, fanout, density):
    p = ref.Params(density=density, maxpks=maxpks, fanout=fanout, shifts=shifts)
    an = analyzer(p)
    files = k3_files()
    got = an.fingerprint_batch(files)
    ctx = an._configure(shifts)
    peaks = [fetch_peaks(ctx, s, len(files)) for s in range(shifts)]
    W = k3_window(shifts, maxpks, fanout)
    across = 0
    for f in range(len(files)):
        want = reference_hashes([peaks[s][f] for s in range(shifts)], p)
        assert np.array_equal(got[f], want), (p, f)
        if len(want):
            across += int(np.count_nonzero(want[:, 0] // W != (want[:, 0] + (want[:, 1] & 63)) // W))
    assert len(got[0]) == 0 and len(got[1]) == 0
    assert across > 0, (p, W)                 # pairs whose target lies in the next window


# ---- statistics -------------------------------------------------------------------------------------
def stats_files():
    """(name, pcm): normal items, digital silence, an all-negative item and items whose floor bites."""
    rng = np.random.default_rng(77)
    quiet = rng.integers(-1, 2, 4 * SR).astype(np.int16)   # |S| << 1 everywhere: every log is negative
    return [("normal", synth_track(9100, 6.0)),
            ("zeros", cases.adversarial_pcm("zeros")),
            ("all_negative", quiet),
            ("silence_gap", cases.adversarial_pcm("silence_gap")),
            ("normal_ragged", synth_track(9101, 9.3)[:102533].copy()),
            ("impulses", cases.adversarial_pcm("impulses")),
            ("short300", cases.adversarial_pcm("short300"))]


def stats_outputs(precision, shifts):
    """What the statistics feed, for the golden file: the batch's hashes and each file's conditioned
    spectrogram (sha256 of its bytes)."""
    an = Analyzer()
    an.precision, an.shifts = precision, shifts
    names, sigs = zip(*stats_files())
    hashes = an.fingerprint_batch(list(sigs))
    sg = [hashlib.sha256(np.ascontiguousarray(an.conditioned_sgram(x)).tobytes()).hexdigest() for x in sigs]
    return names, hashes, sg


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
@pytest.mark.parametrize("shifts", [1, 4])
def test_stats_mixed_batch(precision, shifts):
    names, hashes, sg = stats_outputs(precision, shifts)
    g = np.load(GOLDEN)
    key = "%s_s%d" % (precision, shifts)
    an = Analyzer()
    an.precision, an.shifts = precision, shifts
    for f, (name, x) in enumerate(stats_files()):
        assert np.array_equal(hashes[f], an.fingerprint_batch([x])[0]), (key, name, "batch vs alone")
        assert np.array_equal(hashes[f], g["%s_%s_hashes" % (key, name)]), (key, name, "hashes vs golden")
        assert sg[f] == str(g["%s_%s_sgram" % (precision, name)]), (key, name, "sgram vs golden")
    lens = [len(h) for h in hashes]
    assert lens[1] == 0 and lens[0] > 0 and lens[2] > 0 and lens[3] > 0


# ---- chunked host-PCM path -------------------------------------------------------------------------
@pytest.mark.parametrize("shifts", [1, 4])
def test_chunked_host_pcm_matches_resident(shifts):
    """26 files of 1.3 M samples (68 MB of int16): the host-PCM call copies and processes it in chunks."""
    import torch
    n = 1_300_000
    base = [synth_track(500 + i, 20.0) for i in range(4)] + [cases.adversarial_pcm("silence_gap")]
    sigs = [np.resize(base[i % len(base)], n) for i in range(26)]
    sigs[7] = np.zeros(n, np.int16)
    sigs[11] = sigs[11][:n - 12345]
    stride = (n + 7) // 8 * 8
    hp = np.zeros(len(sigs) * stride + 8, np.int16)
    for i, s in enumerate(sigs):
        hp[i * stride:i * stride + len(s)] = s
    offs = np.arange(len(sigs) + 1, dtype=np.int64) * stride
    lens = np.array([len(s) for s in sigs], np.int64)
    assert hp.nbytes >= 64 << 20
    an = Analyzer()
    an.shifts = shifts
    rows_h, off_h = an.fingerprint_packed(hp, offs, sample_lengths=lens)
    rows_d, off_d = an.fingerprint_packed(torch.from_numpy(hp).cuda(), offs, sample_lengths=lens)
    assert np.array_equal(off_h, off_d)
    assert np.array_equal(rows_h, rows_d)
    assert off_h[8] == off_h[7] and off_h[-1] > 0


# ---- item-table reuse --------------------------------------------------------------------------------
def test_same_layout_batches_and_other_entry_points():
    """A batch with the layout of the previous one reuses the item and tile tables on the device.  Other
    PCM, another layout in between, and the entry points that write the item table themselves
    (peaks2landmarks, hashing explicit peak lists, the conditioned spectrogram) must not leave a stale
    table behind."""
    n = 5 * SR
    a = [synth_track(700 + i, 5.0) for i in range(6)]
    b = [synth_track(800 + i, 5.0) for i in range(6)]
    c = [synth_track(900 + i, 3.0 + 0.7 * i) for i in range(6)]
    assert all(len(x) == n for x in a + b)
    an = Analyzer()
    alone = {id(x): an.fingerprint_batch([x])[0] for x in a + b + c}

    def check(sigs):
        for x, h in zip(sigs, an.fingerprint_batch(sigs)):
            assert np.array_equal(h, alone[id(x)])

    check(a)
    check(b)                                   # same layout, other samples
    check(a)
    check(c)                                   # another layout
    check(a)
    an.peaks2landmarks([(3, 10), (5, 12), (9, 14)])
    check(a)
    ctx = an._configure(an.shifts)
    rows = np.array([[3, 10], [5, 12], [9, 14]], np.int32)
    off = np.array([0, 3], np.int64)
    total = C.c_int64(-1)
    ctx.check(ctx.lib.afp_fingerprint_from_peaks(ctx.h, rows.ctypes.data, 1, 1,
                                                 off.ctypes.data_as(C.POINTER(C.c_int64)), None, C.byref(total)))
    assert total.value > 0
    check(a)
    an.conditioned_sgram(b[1])
    check(a)
