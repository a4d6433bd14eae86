"""afp_fingerprint_from_peaks: the hashes of a ragged batch of peak lists in one pass.  Every file's
rows must equal wavfile2hashes of that .afpk file as the reference states it (peaks2landmarks,
landmarks2hashes, sorted unique rows: tests/k2k3_reference.py::file_hashes); the workspace must be
left as afp_fingerprint_batch leaves it (afp_fetch_peaks returns the input, store_batch(None) stores
what the fetched rows store); a malformed file must fail with the per-file call's code, flag only
that file and leave no batch behind."""
import ctypes as C

import numpy as np
import pytest
import torch

from audfprint_b200 import Analyzer, HashTable, _lib
from tests.k2k3_reference import Params, file_hashes

pytestmark = pytest.mark.gpu
I64P = C.POINTER(C.c_int64)


def _params(an):
    return Params(maxpks=an.maxpksperframe, fanout=an.maxpairsperpeak, mindt=an.mindt, targetdt=an.targetdt,
                  targetdf=an.targetdf)


def _want(peaks, an):
    if len(peaks) == 0:
        return np.zeros((0, 2), np.int32)
    return np.asarray(file_hashes([[tuple(r) for r in np.asarray(peaks).tolist()]], _params(an)),
                      np.int32).reshape(-1, 2)


def _call(an, arrays, shifts=1, on_host=True):
    """One afp_fingerprint_from_peaks -> (rc, status, per-file rows or None)."""
    ctx = an._configure(shifts)
    n = len(arrays)
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum([len(a) for a in arrays])
    rows = np.ascontiguousarray(np.concatenate([np.asarray(a, np.int32).reshape(-1, 2) for a in arrays])) \
        if off[-1] else np.zeros((1, 2), np.int32)
    keep = rows
    if on_host:
        ptr = rows.ctypes.data
    else:
        keep = torch.from_numpy(rows).cuda(ctx.device)
        torch.cuda.synchronize()
        ptr = keep.data_ptr()
    status = np.full(max(n, 1), -99, np.int32)
    total = C.c_int64(-1)
    rc = ctx.lib.afp_fingerprint_from_peaks(ctx.h, ptr, 1 if on_host else 0, n, off.ctypes.data_as(I64P),
                                            status.ctypes.data, C.byref(total))
    if rc:
        return rc, status[:n], None
    roff = np.empty(n + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, roff.ctypes.data_as(I64P)))
    assert roff[-1] == total.value
    out = np.empty((int(roff[-1]), 2), np.int32)
    ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, out.ctypes.data, 1, None))
    del keep
    return 0, status[:n], [out[roff[i]:roff[i + 1]] for i in range(n)]


def _fetch_peaks(an, n):
    ctx = _lib.context(an.device)
    poff = np.empty(n + 1, np.int64)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, 0, None, 1, poff.ctypes.data_as(I64P)))
    rows = np.empty((int(poff[-1]), 2), np.int32)
    ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, 0, rows.ctypes.data, 1, None))
    return [rows[poff[i]:poff[i + 1]] for i in range(n)]


def _random_peaks(rng, ncols, span, maxpks, base=0, full=False):
    """Column-major peaks with bins ascending: ncols distinct columns in [base, base + span), 1..maxpks
    distinct bins each (exactly maxpks with full)."""
    if ncols == 0:
        return np.zeros((0, 2), np.int32)
    cols = np.sort(rng.choice(span, size=min(ncols, span), replace=False)) + base
    out = []
    for c in cols:
        k = maxpks if full else int(rng.integers(1, maxpks + 1))
        for b in np.sort(rng.choice(256, size=k, replace=False)):
            out.append((int(c), int(b)))
    return np.array(out, np.int32).reshape(-1, 2)


def _ragged(rng, maxpks):
    lists = [np.zeros((0, 2), np.int32), np.array([[0, 17]], np.int32), np.array([[5, 255]], np.int32)]
    lists += [_random_peaks(rng, int(rng.integers(1, 300)), 2000, maxpks) for _ in range(20)]
    lists.append(_random_peaks(rng, 50, 200, maxpks, base=0))               # dense, from column 0
    lists.append(_random_peaks(rng, 200, 1 << 12, maxpks, base=(1 << 20) - 2048))   # crosses 2^20
    lists.append(_random_peaks(rng, 100, 1 << 10, maxpks, base=(1 << 21) + 3))
    lists.insert(7, np.zeros((0, 2), np.int32))
    return lists


@pytest.mark.parametrize("shifts", [1, 4])
@pytest.mark.parametrize("on_host", [True, False])
def test_ragged_batch_equals_reference(shifts, on_host):
    rng = np.random.default_rng(11 + shifts + 2 * on_host)
    an = Analyzer(density=20.0)
    lists = _ragged(rng, an.maxpksperframe)
    rc, status, got = _call(an, lists, shifts, on_host)
    assert rc == 0 and not status.any()
    for pk, g in zip(lists, got):
        np.testing.assert_array_equal(g, _want(pk, an))
    for pk, f in zip(lists, _fetch_peaks(an, len(lists))):      # the scatter's round trip
        np.testing.assert_array_equal(f, pk)


@pytest.mark.parametrize("maxpks", list(range(1, 17)))
def test_saturated_columns(maxpks):
    rng = np.random.default_rng(100 + maxpks)
    an = Analyzer(density=20.0)
    an.maxpksperframe = maxpks
    an.maxpairsperpeak = min(3, 256 // maxpks)
    lists = [_random_peaks(rng, 40, 120, maxpks, full=True), _random_peaks(rng, 30, 60, maxpks, base=7, full=True)]
    rc, status, got = _call(an, lists)
    assert rc == 0
    for pk, g in zip(lists, got):
        np.testing.assert_array_equal(g, _want(pk, an))


def test_4096_files_one_call():
    rng = np.random.default_rng(4096)
    an = Analyzer(density=20.0)
    lists = [_random_peaks(rng, int(rng.integers(0, 40)), 400, an.maxpksperframe) for _ in range(4096)]
    ctx = an._configure(1)
    before = ctx.launch_count()
    rc, status, got = _call(an, lists)
    launches = ctx.launch_count() - before
    assert rc == 0 and launches <= 8, launches          # scatter, K3 landmarks, count, scans, write
    for pk, g in zip(lists, got):
        np.testing.assert_array_equal(g, _want(pk, an))


@pytest.mark.parametrize("shifts", [1, 4])
def test_store_in_place_equals_fetched_rows(shifts):
    import random
    rng = np.random.default_rng(5 + shifts)
    an = Analyzer(density=20.0)
    lists = _ragged(rng, an.maxpksperframe)
    names = ["f%d" % i for i in range(len(lists))]
    rc, _, got = _call(an, lists, shifts)
    assert rc == 0
    a = HashTable(hashbits=10, depth=6, maxtime=1 << 22)
    random.seed(3)
    a.store_batch(names, None)
    ra = random.random()
    b = HashTable(hashbits=10, depth=6, maxtime=1 << 22)
    random.seed(3)
    b.store_batch(names, got)
    assert ra == random.random()
    np.testing.assert_array_equal(a.table, b.table)
    np.testing.assert_array_equal(a.counts, b.counts)
    np.testing.assert_array_equal(a.hashesperid, b.hashesperid)


def _per_file_code(an, pk):
    ctx = an._configure(1)
    pk = np.ascontiguousarray(pk, np.int32)
    n = C.c_int64(0)
    return ctx.lib.afp_landmarks_from_peaks(ctx.h, pk.ctypes.data, len(pk), 1, C.byref(n))


def _bad_lists(rng, an):
    P = an.maxpksperframe
    too_many = np.array([[3, b] for b in range(P + 1)] + [[9, 1]], np.int32)
    unsorted = np.array([[4, 10], [2, 11], [6, 1]], np.int32)
    dup_bin = np.array([[4, 10], [4, 10], [6, 1]], np.int32)
    bad_bin = np.array([[1, 256], [2, 3]], np.int32)
    neg_col = np.array([[-1, 3], [2, 3]], np.int32)
    return [("too_many", too_many, _lib_code("UNSUPPORTED")), ("unsorted", unsorted, _lib_code("INVALID")),
            ("dup_bin", dup_bin, _lib_code("INVALID")), ("bad_bin", bad_bin, _lib_code("INVALID")),
            ("neg_col", neg_col, _lib_code("INVALID"))]


def _lib_code(name):
    return {"INVALID": -2, "UNSUPPORTED": -3}[name]


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_malformed_file_fails_alone(where):
    rng = np.random.default_rng(77)
    an = Analyzer(density=20.0)
    good = [_random_peaks(rng, 30, 300, an.maxpksperframe) for _ in range(9)]
    for name, bad, code in _bad_lists(rng, an):
        assert _per_file_code(an, bad) == code, name
        k = {"first": 0, "middle": 4, "last": len(good)}[where]
        lists = good[:k] + [bad] + good[k:]
        rc, status, _ = _call(an, lists)
        assert rc == code, name
        want = np.zeros(len(lists), np.int32)
        want[k] = code
        np.testing.assert_array_equal(status, want)
        ctx = _lib.context(an.device)
        with pytest.raises(_lib.AfpError):          # AFP_ERR_STATE: no batch to fetch
            ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, None))
    # the lowest failing file decides the code
    lists = good[:2] + [_bad_lists(rng, an)[1][1], good[2], _bad_lists(rng, an)[0][1]]
    rc, status, _ = _call(an, lists)
    assert rc == -2 and status.tolist() == [0, 0, -2, 0, -3]


def test_column_bound():
    """A last column of 2^28 is the bound: with maxpks = fanout = 1 the workspace takes about
    10 bytes per column, 2.7 GB for the 2^28 + 1 columns.  One column more is AFP_ERR_INVALID, as in
    the per-file call."""
    an = Analyzer(density=20.0)
    an.maxpksperframe, an.maxpairsperpeak = 1, 1
    top = 1 << 28
    pk = np.array([[0, 5], [3, 9], [top - 40, 100], [top - 10, 110], [top, 120]], np.int32)
    small = np.array([[1, 2], [4, 3]], np.int32)
    rc, status, got = _call(an, [small, pk])
    assert rc == 0
    np.testing.assert_array_equal(got[0], _want(small, an))
    np.testing.assert_array_equal(got[1], _want(pk, an))
    over = np.array([[2, 3], [top + 1, 7]], np.int32)
    assert _per_file_code(an, over) == -2
    rc, status, _ = _call(an, [small, over])
    assert rc == -2 and status.tolist() == [0, -2]


def test_wavfile2hashes_afpk_and_list_form(tmp_path):
    """The .afpk branch of wavfile2hashes and its list form give the reference's rows."""
    from audfprint_b200 import analyzer as an_mod
    rng = np.random.default_rng(9)
    an = Analyzer(density=20.0)
    an.shifts = 4
    names = []
    for i in range(6):
        pk = _random_peaks(rng, 80 + 10 * i, 900, an.maxpksperframe, base=i)
        fn = str(tmp_path / ("p%d.afpk" % i))
        an_mod.peaks_save(fn, pk)
        names.append((fn, pk))
    for fn, pk in names:
        np.testing.assert_array_equal(an.wavfile2hashes(fn), _want(pk, an))
    an.max_frames_per_call = 1500                # several chunks
    got = an.wavfiles2hashes([fn for fn, _ in names])
    for g, (_, pk) in zip(got, names):
        np.testing.assert_array_equal(g, _want(pk, an))


@pytest.mark.parametrize("on_host", [True, False])
def test_offsets_need_not_start_at_zero(on_host):
    """File f is rows [off[f], off[f+1]) of the buffer: rows before off[0] are not read."""
    rng = np.random.default_rng(21)
    an = Analyzer(density=20.0)
    lists = [_random_peaks(rng, 60, 500, an.maxpksperframe) for _ in range(3)]
    junk = np.array([[9, 300], [-4, 1], [7, 7]], np.int32)           # would fail every check
    rows = np.ascontiguousarray(np.concatenate([junk] + lists))
    off = np.cumsum([len(junk)] + [len(a) for a in lists]).astype(np.int64)
    ctx = an._configure(1)
    buf = rows if on_host else torch.from_numpy(rows).cuda(ctx.device)
    torch.cuda.synchronize()
    ptr = rows.ctypes.data if on_host else buf.data_ptr()
    ctx.check(ctx.lib.afp_fingerprint_from_peaks(ctx.h, ptr, 1 if on_host else 0, 3, off.ctypes.data_as(I64P),
                                                 None, None))
    roff = np.empty(4, np.int64)
    ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, roff.ctypes.data_as(I64P)))
    out = np.empty((int(roff[-1]), 2), np.int32)
    ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, out.ctypes.data, 1, None))
    for k, pk in enumerate(lists):
        np.testing.assert_array_equal(out[roff[k]:roff[k + 1]], _want(pk, an))


def test_reference_afpk_hashes():
    """The hashes the reference's wavfile2hashes forms from the .afpk files it wrote
    (tests/golden/precompute.npz), from one call over all of them."""
    import os
    from tests.conftest import GOLDEN
    g = np.load(os.path.join(GOLDEN, "precompute.npz"))
    an = Analyzer(density=100.0)
    outs = [str(o) for o in g["peaks_s1/outputs"]]
    lists = [np.frombuffer(g["peaks_s1/" + o].tobytes()[16:], "<i4").reshape(-1, 2) for o in outs]
    for shifts in (1, 4):
        rc, status, got = _call(an, lists, shifts)
        assert rc == 0
        for o, h in zip(outs, got):
            np.testing.assert_array_equal(h, g["afpk_hashes/" + o])
