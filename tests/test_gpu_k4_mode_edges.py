"""K4's offset-histogram mode search - the quick filter, the dense dtime histogram, its local
maxima, the repeated first arg-max above threshcount, the +-window count and clear and the
max_alignments_per_id cap - against k4_reference (tests/k4_reference.py, pinned to the reference
by tests/test_k4_modes_cpu.py) on the constructed families of tests/k4_mode_cases.py.

Each family runs on every path that can take it: the fast kernel, the general kernel
(force_general_kernel) and the long path (the queries padded with rows that probe an empty bucket,
tests/test_gpu_k4_ranking_edges.py's `padded`), or, for the mixed family, short and long queries
in one call.  Per query it checks, bit for bit:
  * the plain rows in rank order, rank column included, and Matcher.last_status column 0 (the
    intended path ran);
  * the publish-mode rows and candidate list;
  * the rows of find_time_range alone (finished on the device): columns 0-4 against the reference
    rows, columns 5-6 against orc.time_range at time_quantile 0.02 and 0.5.
It also checks that a negative threshcount and a query time whose histogram would not fit int
indexing are refused by every entry point with nothing written, and that threshcount 0 still
matches on the general kernel and the long path."""
import ctypes as C

import numpy as np
import pytest

from audfprint_b200 import Matcher
from oracle import afp_oracle as orc
from tests import k4_mode_cases as mc
from tests.test_gpu_k4_ranking_edges import LONG, Ref, matcher, padded

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in mc.all_cases()}
STATUS = {"fast": 0, "general": -1, "long": LONG}


def path_queries(case, path):
    """The case's queries as `path` runs them, and the status column 0 each must report."""
    if path == "mixed":
        pad = case.long_only
    else:
        pad = range(len(case.queries)) if path == "long" else ()
    qs = [padded(case.sc, q) if i in pad else q for i, q in enumerate(case.queries)]
    st = [LONG if i in pad else (0 if path == "mixed" else STATUS[path]) for i in range(len(qs))]
    return qs, st


def groups(case, n):
    """Query indices of each call."""
    return [list(range(n))] if case.calls == 1 else [[i] for i in range(n)]


def scrub():
    """Fill the first 200 row slots of query 0 with rows of id 4000 (a table of its own), so that a
    row a path counts but never writes cannot pass for a right one an earlier call left there."""
    sc = mc.scene()
    mc.plant(sc, [{3 * i: 2 for i in range(200)}], how="mult", first=4000)
    rows = matcher(0, 1, 10, force=True, maxalign=300).match_batch(sc.ht(), [sc.query()], sort=False)[0]
    assert len(rows) == 200 and np.all(rows[:, 0] == 4000)


def time_range_rows(ref, window, quant):
    rows = ref.rows.copy()
    for r in rows:
        r[5], r[6] = orc.time_range(ref.h, int(r[0]), int(r[2]), window, quant)
    return rows


@pytest.mark.parametrize("name", list(CASES))
def test_mode_edges(name):
    import torch
    case = CASES[name]
    r = mc.reached(case)
    if name == "many_queries":
        assert len(case.queries) > 2 * torch.cuda.get_device_properties(0).multi_processor_count
    refs = [Ref(case.sc, q, case.thresh, case.sdepth, case.window, case.maxalign) for q in case.queries]
    for ref, rows in zip(refs, r.rows):
        assert np.array_equal(ref.rows, rows)
    ht = case.sc.ht()
    for path in case.paths:
        qs, want_st = path_queries(case, path)
        m = matcher(case.window, case.thresh, case.sdepth, force=(path == "general"), maxalign=case.maxalign)
        gs = groups(case, len(qs))
        scrub()
        for g in gs:                                       # plain rows; consecutive calls back to back
            got = m.match_batch(ht, [qs[i] for i in g], sort=False)
            st = Matcher.last_status(ht, len(g))[:, 0]
            for k, i in enumerate(g):
                assert st[k] == want_st[i], (path, "plain status", i, st.tolist())
                assert np.array_equal(got[k], refs[i].rows), (path, "plain rows", i)
        for g in gs:                                       # publish mode
            packed = np.ascontiguousarray(np.concatenate([qs[i] for i in g]))
            qoff = np.concatenate([[0], np.cumsum([len(qs[i]) for i in g])]).astype(np.int64)
            rows, roff, cand, cnts = m._publish_call(ht, packed, qoff)
            st = Matcher.last_status(ht, len(g))[:, 0]
            for k, i in enumerate(g):
                ref = refs[i]
                assert st[k] == want_st[i], (path, "publish status", i, st.tolist())
                assert tuple(cnts[k]) == ref.pcnt, (path, i, cnts[k].tolist(), ref.pcnt)
                n = ref.pcnt[0]
                assert np.array_equal(cand[k, :n, 0].astype(np.int64), ref.pid), (path, "publish ids", i)
                assert np.array_equal(cand[k, :n, 1].astype(np.int64), ref.praw), (path, "publish raw", i)
                assert np.array_equal(rows[roff[k]:roff[k + 1]], ref.prows), (path, "publish rows", i)
        m.find_time_range = True                           # the device finish of find_time_range alone
        for quant in (0.02, 0.5):
            m.time_quantile = quant
            for g in gs:
                got = m.match_batch(ht, [qs[i] for i in g], sort=False)
                for k, i in enumerate(g):
                    want = time_range_rows(refs[i], case.window, quant)
                    assert np.array_equal(got[k][:, :5], want[:, :5]), (path, "time range rows", quant, i)
                    assert np.array_equal(got[k][:, 5:], want[:, 5:]), (path, "time range", quant, i)


# ---- refusals ------------------------------------------------------------------------------------
def small_scene():
    sc = mc.scene()
    mc.plant(sc, [{10: 3, 12: 2}])
    return sc


def params(window=1, thresh=1, sdepth=10, maxalign=100):
    from audfprint_b200 import _lib
    return _lib.MatcherParams(window, thresh, sdepth, maxalign, 0, 0, 0)


def abi_calls(ctx, q, p):
    """(name, call) of every entry point that takes matcher parameters; each call returns
    (status, total_rows, qmax) with total_rows and qmax preset to sentinels."""
    import torch
    from audfprint_b200.matcher import timebits_breaks
    qoff = np.array([0, len(q)], np.int64)
    qp = qoff.ctypes.data_as(C.POINTER(C.c_int64))
    br = timebits_breaks()
    brp = br.ctypes.data_as(C.POINTER(C.c_int64))

    def batch():
        t = C.c_int64(-77)
        return ctx.lib.afp_match_batch(ctx.h, q.ctypes.data, 1, 1, qp, C.byref(p), C.byref(t)), t.value, None

    def options():
        t = C.c_int64(-77)
        return ctx.lib.afp_match_options_batch(ctx.h, q.ctypes.data, 1, 1, qp, C.byref(p), 0, 1, 0.02, brp,
                                               C.byref(t)), t.value, None

    def shard_rank():
        t = C.c_int64(-77)
        qmax = torch.full((1,), -77, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        rc = ctx.lib.afp_match_options_shard_rank(ctx.h, q.ctypes.data, 1, 1, qp, C.byref(p), 1, 0, 0.02, brp,
                                                  C.c_void_p(qmax.data_ptr()), C.byref(t))
        return rc, t.value, int(qmax.item())
    return [("afp_match_batch", batch), ("afp_match_options_batch", options),
            ("afp_match_options_shard_rank", shard_rank)]


def test_negative_threshcount_is_refused_everywhere():
    """threshcount -1: AFP_ERR_INVALID from every entry point, total_rows and qmax untouched, and
    no earlier result is replaced; Matcher and the sharded match raise ValueError."""
    from audfprint_b200 import dist
    sc = small_scene()
    ht = sc.ht()
    q = sc.query()
    ctx = ht._sync_device()
    ok = matcher(1, 1, 10).match_batch(ht, [q], sort=False)[0]
    assert len(ok) == 2
    for name, call in abi_calls(ctx, q, params(thresh=-1)):
        rc, total, qmax = call()
        assert rc == -2 and total == -77 and qmax in (None, -77), (name, rc, total, qmax)
        assert b"bad matcher parameters" in ctx.lib.afp_last_error(ctx.h), name
    m = matcher(1, -1, 10)
    for call in (lambda: m.match_batch(ht, [q]), lambda: m.match_hashes(ht, q), lambda: m.match_hashes(ht, q, 0),
                 lambda: dist.match_sharded_batch(m, ht, (q, np.array([0, len(q)])))):
        with pytest.raises(ValueError, match="threshcount"):
            call()
    assert np.array_equal(matcher(1, 1, 10).match_batch(ht, [q], sort=False)[0], ok)


def test_window_above_4096_is_refused():
    sc = small_scene()
    ht = sc.ht()
    ctx = ht._sync_device()
    for name, call in abi_calls(ctx, sc.query(), params(window=4097)):
        rc, total, qmax = call()
        assert rc == -2 and total == -77 and qmax in (None, -77), (name, rc, total)


@pytest.mark.parametrize("path", ["short", "long"])
def test_query_time_near_int32_max_is_refused(path):
    """A query time within 2^mtb + 2 * window + 6 of INT32_MAX: the histogram would not fit int
    indexing, AFP_ERR_UNSUPPORTED on the short and the long path (a long query with short ones of
    small query times in the same call), nothing written."""
    sc = small_scene()
    ht = sc.ht()
    ctx = ht._sync_device()
    big = np.array([[2 ** 31 - 1 - (1 << sc.mtb), 1]], np.int32)
    q = np.concatenate([sc.query(), big])
    if path == "long":
        q = np.concatenate([padded(sc, q), sc.query()])
        qoff = np.array([0, len(q) - len(sc.query()), len(q)], np.int64)
    else:
        qoff = np.array([0, len(q)], np.int64)
    t = C.c_int64(-77)
    rc = ctx.lib.afp_match_batch(ctx.h, q.ctypes.data, 1, len(qoff) - 1, qoff.ctypes.data_as(C.POINTER(C.c_int64)),
                                 C.byref(params()), C.byref(t))
    assert rc == -3 and t.value == -77
    assert b"query time too large" in ctx.lib.afp_last_error(ctx.h)
    with pytest.raises(Exception, match="query time too large"):
        matcher(1, 1, 10).match_batch(ht, (q, qoff))
    # the context still matches after the refusal
    ok =matcher(1, 1, 10).match_batch(ht, [sc.query()], sort=False)[0]
    assert len(ok) == 2


def test_threshcount_zero_still_matches():
    """threshcount 0 is accepted: the general kernel and the long path give the reference's rows."""
    case = CASES["thresh_0"]
    ht = case.sc.ht()
    want = case.rows(0)
    assert len(want) == 4
    for path in ("general", "long"):
        qs, _ = path_queries(case, path)
        got = matcher(case.window, 0, case.sdepth, force=(path == "general")).match_batch(ht, qs, sort=False)[0]
        assert np.array_equal(got, want), path
