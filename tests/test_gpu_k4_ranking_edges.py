"""K4's ranked candidate lists against the reference (tests/k4_reference.py), bit for bit, at the
edges where a ranking goes subtly wrong: every handover boundary of the fast kernel, exact weight
ties, weights that share a float32 image or sit in the clamped end bins of its histogram, the
pruning bound equal to the K-th weight, the general kernel's split bucket multiplicities, id
segments and unsorted probe, the long path's tie at rank K, and the sharded merge.

Every table is constructed so that each slot a query probes holds an id the test chose; most probed
ids appear once (filler ids of low weight, as in a real table), and the ids that matter are
planted.  Each case compares, on every path that can take the query (fast kernel, general kernel,
long path through padding rows that probe an empty bucket):
  * the publish list (id, raw, weight) in order, with (entries, n_above);
  * the plain rows in candidate-rank order, rank column included;
and asserts which branch of the fast kernel ran (Matcher.last_status column 0).  Each family first
asserts on the reference side that its edge is really reached."""
import ctypes as C

import numpy as np
import pytest

from audfprint_b200 import HashTable, Matcher
from tests import k4_reference as k4

pytestmark = pytest.mark.gpu

LONG_HITS = 1 << 24
LONG = 6                                    # afp_fetch_match_status: the long-query path
MMAX, SCAP, XCAP, KCAP = 12288, 4096, 2048, 1024     # csrc/afp_match_fast.cu, afp_match_common.cuh
MSLOTS, PROBE_MAX = 16384, 256


class Scene:
    """A table built bucket by bucket.  group(ids, m) takes a fresh bucket, puts `ids` in its
    first slots (entry time qt + dt) and adds m query rows that probe it, all at time qt (hashes
    that differ above the bucket bits), so every hit of an id in one group has the same dtime."""

    def __init__(self, hashbits=12, depth=64, mtb=14, nids=1 << 16, hpi=1 << 20):
        self.hashbits, self.depth, self.mtb, self.nids = hashbits, depth, mtb, nids
        self.table = np.zeros((1 << hashbits, depth), np.uint32)
        self.counts = np.zeros(1 << hashbits, np.int32)
        self.hpi = np.full(nids, hpi, np.uint32)
        self.rows = []
        self.next_b = 1                      # bucket 0 stays empty: the padding rows probe it
        self.next_fill = nids                # filler ids are handed out downwards from the top

    def fill(self, n, hpi=None):
        ids = np.arange(self.next_fill - n, self.next_fill)
        self.next_fill -= n
        if hpi is not None:
            self.hpi[ids] = hpi
        return ids

    def group(self, ids, m=1, qt=0, dt=100):
        b = self.next_b
        self.next_b += 1
        ids = np.asarray(ids, np.int64)
        assert b < (1 << self.hashbits) and len(ids) <= self.depth and qt + dt < (1 << self.mtb)
        assert ids.max(initial=0) < self.nids and (self.nids << self.mtb) < (1 << 32)
        self.table[b, :len(ids)] = ((ids + 1) << self.mtb) + qt + dt
        self.counts[b] = len(ids)
        self.rows += [(qt, b + (k << self.hashbits)) for k in range(m)]
        return b

    def probe(self, b, qt):
        self.rows.append((qt, b))

    def query(self):
        return np.array(self.rows, np.int32).reshape(-1, 2)

    def ht(self):
        ht = HashTable(hashbits=self.hashbits, depth=self.depth, maxtime=1 << self.mtb)
        ht.table, ht.counts, ht.hashesperid = self.table, self.counts, self.hpi
        return ht


def members(ids, sc, raw, hpi, qt=0, dt=100, width=None):
    """Give every id `raw` records, one per group of single-probed buckets (so raw = number of
    records), aligned at one dtime: each id yields a row once raw > threshcount."""
    ids = np.asarray(ids, np.int64)
    sc.hpi[ids] = hpi
    width = width or sc.depth
    for _ in range(raw):
        for s in range(0, len(ids), width):
            sc.group(ids[s:s + width], 1, qt, dt)


def singles(ids, sc, hpi=None, width=None, qt=0):
    """One record each (raw 1 in a bucket probed once), at scattered dtimes."""
    ids = np.asarray(ids, np.int64)
    if hpi is not None:
        sc.hpi[ids] = hpi
    width = width or sc.depth
    for s in range(0, len(ids), width):
        sc.group(ids[s:s + width], 1, qt, 100 + s // width)


def matcher(window, thresh, sdepth, force=False, maxalign=100):
    m = Matcher()
    m.window, m.threshcount, m.search_depth = window, thresh, sdepth
    m.max_alignments_per_id = maxalign
    m.force_general_kernel = force
    return m


class Ref:
    def __init__(self, sc, q, thresh, sdepth, window, maxalign=100):
        h = k4.hits(sc.table, sc.counts, sc.hashbits, sc.depth, sc.mtb, q)
        self.h = h
        self.ids, self.raw, self.w = k4.candidates(h, sc.hpi, thresh, sdepth)
        self.rows = k4.rows_in_rank_order(h, self.ids, self.raw, window, thresh, maxalign)
        self.pid, self.praw, self.pw, self.pcnt = k4.candidates(h, sc.hpi, thresh, sdepth, publish=True)
        self.prows = k4.rows_in_rank_order(h, self.pid, self.praw, window, thresh, maxalign)
        uid, cnt = np.unique(h[:, 0], return_counts=True)
        self.uid, self.ucnt = uid, cnt


def padded(sc, q):
    """q plus rows that probe the empty bucket 0 until rows * depth reaches the long-path limit:
    same hits, same results, the long-query path takes it."""
    n = max(0, -(-LONG_HITS // sc.depth) - len(q))
    pad = np.stack([np.zeros(n, np.int64), np.arange(n, dtype=np.int64) << sc.hashbits], 1)
    assert np.all(sc.counts[(pad[:, 1] & ((1 << sc.hashbits) - 1))] == 0)
    return np.concatenate([q, pad.astype(np.int32)])


def run(sc, thresh, sdepth, status, window=1, paths=("fast", "general", "long"), q=None, ref=None, maxalign=100):
    """Compare every path with the reference.  status = (plain, publish) expected in column 0 of
    the fast kernel's status.  Returns the reference."""
    ht = sc.ht()
    q = sc.query() if q is None else q
    ref = ref or Ref(sc, q, thresh, sdepth, window, maxalign)
    for path in paths:
        qq = padded(sc, q) if path == "long" else q
        m = matcher(window, thresh, sdepth, force=(path == "general"), maxalign=maxalign)
        qoff = np.array([0, len(qq)], np.int64)
        got = m.match_batch(ht, [qq], sort=False)[0]
        st = Matcher.last_status(ht, 1)[0]
        want_st = {"fast": status[0], "general": -1, "long": LONG}[path]
        assert st[0] == want_st, (path, "plain", st.tolist())
        assert np.array_equal(got, ref.rows), (path, "plain rows")
        rows, roff, cand, cnts = m._publish_call(ht, np.ascontiguousarray(qq), qoff)
        st = Matcher.last_status(ht, 1)[0]
        want_st = {"fast": status[1], "general": -1, "long": LONG}[path]
        assert st[0] == want_st, (path, "publish", st.tolist())
        assert tuple(cnts[0]) == ref.pcnt, (path, cnts[0].tolist(), ref.pcnt)
        k = ref.pcnt[0]
        assert np.array_equal(cand[0, :k, 0].astype(np.int64), ref.pid), (path, "publish ids")
        assert np.array_equal(cand[0, :k, 1].astype(np.int64), ref.praw), (path, "publish raw")
        assert np.array_equal(cand[0, :k, 2].view(np.uint64), ref.pw.view(np.uint64)), (path, "publish weights")
        assert np.array_equal(rows, ref.prows), (path, "publish rows")
    return ref


def kth(ref, k):
    """(weight, id) at rank k of the plain list."""
    return ref.w[k], ref.ids[k]


# ---- handover boundaries: the fast kernel finishes at the limit, hands over one past it ---------
def set_clusters(ids):
    """Longest run of occupied slots of the fast kernel's member set (linear probing, 16384 slots,
    hash (id * 0x9E3779B1) >> 18) after inserting `ids`: independent of insertion order, and an
    insertion never probes more slots than the run it lands in."""
    h = ((np.asarray(ids, np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)) >> np.uint64(18)
    occ = np.zeros(MSLOTS, bool)
    for x in h.astype(np.int64):
        while occ[x]:
            x = (x + 1) & (MSLOTS - 1)
        occ[x] = True
    if occ.all():
        return MSLOTS
    start = int(np.argmin(occ))                         # an empty slot: unroll the ring from there
    r = np.roll(occ, -start).astype(np.int8)
    edges = np.diff(np.r_[0, r, 0])
    return int((np.nonzero(edges == -1)[0] - np.nonzero(edges == 1)[0]).max())


@pytest.mark.parametrize("nmem,status", [(MMAX, 0), (MMAX + 1, 1)])
def test_set_full_boundary(nmem, status):
    """12288 members: the set holds them without a probe sequence of PROBE_MAX (shown below on
    the host for these ids), status 0.  12289: status 1 (FS_SET_FULL)."""
    sc = Scene(hashbits=9, depth=512, nids=1 << 15, hpi=1 << 20)
    ids = np.arange(1, nmem + 1)
    members(ids, sc, raw=2, hpi=1000 + 7 * ids, width=256)
    assert set_clusters(ids) < PROBE_MAX
    ref = run(sc, 1, 100, (status, status))
    assert np.count_nonzero(ref.ucnt >= 2) == nmem and len(ref.ids) == 100


def warp_cap(nq, depth):
    """Member hits one warp of the fast kernel may append (afp_match.cu: mh_cap / 32)."""
    return min(max(-(-nq * depth // 32) * 32, 32768), 131072) // 32


@pytest.mark.parametrize("m,n,status", [(16, 64, 0), (25, 41, 2)])
def test_hits_full_boundary(m, n, status):
    """One bucket probed m times (m > threshcount: every id in it is a member) holding n ids:
    m * n member hits in warp 0's segment - exactly its capacity (status 0), one more (status 2,
    FS_HITS_FULL)."""
    sc = Scene(hashbits=8, depth=64)
    ids = np.arange(10, 10 + n)
    sc.hpi[ids] = 3                                      # one weight: id order decides
    sc.group(ids, m)
    assert m * n - warp_cap(m, sc.depth) == (1 if status else 0)
    run(sc, 5, 100, (status, status))


@pytest.mark.parametrize("nx,status", [(XCAP, 0), (XCAP + 1, 3)])
def test_extras_full_boundary(nx, status):
    """5 strong and 5 weak members (K = 10); nx single-record ids of hashesperid 1 outrank the
    K-th member: pass 3 admits 2048 (status 0), 2049 is one too many (status 3, FS_EXTRAS_FULL)."""
    sc = Scene()
    members(np.arange(1, 6), sc, raw=4, hpi=1)
    members(np.arange(6, 11), sc, raw=2, hpi=1000)
    singles(np.arange(100, 100 + nx), sc, hpi=1)
    ref = run(sc, 1, 10, (status, status))
    assert np.count_nonzero(ref.ucnt == 1) == nx and ref.w[9] > 2 / 1000
    assert list(ref.ids[:5]) == [5, 4, 3, 2, 1] and np.all(ref.w[5:] == 1.0)


def bm_hash(ids):
    return ((np.asarray(ids, np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(12)


@pytest.mark.parametrize("nmem,status", [(20, 0), (19, 4)])
def test_ndist_unknown_boundary(nmem, status):
    """More than 2^20 ids (hashed bitmap), publish mode, search_depth 20: 20 members fix the depth
    (status 0); with 19 the number of distinct ids is unknown (status 4, FS_NDIST_UNKNOWN).  The
    ids are chosen so that no two share a bitmap bit (no false members)."""
    sc = Scene(mtb=11, nids=(1 << 20) + 4096)
    rng = np.random.default_rng(5)
    pool = rng.permutation(np.arange(1 << 19, sc.nids - 4096))[:400]
    _, first = np.unique(bm_hash(pool), return_index=True)
    pool = pool[np.sort(first)]
    mem, sng = pool[:nmem], pool[nmem:nmem + 200]
    members(mem, sc, raw=2, hpi=rng.integers(50, 60, nmem))
    singles(sng, sc, hpi=rng.integers(20, 200, 200))
    assert len(np.unique(bm_hash(np.r_[mem, sng]))) == nmem + 200
    ref = run(sc, 1, 20, (0, status), paths=("fast", "general"))
    assert ref.pcnt[0] == 20 and np.count_nonzero(ref.ucnt >= 2) == nmem


@pytest.mark.parametrize("nmem,status", [(KCAP, 0), (KCAP + 1, 5)])
def test_depth_boundary_with_ties_at_rank_k(nmem, status):
    """nmem members (raw 2 / hashesperid 50) and single-record ids (1 / 25) of the SAME weight
    0.04, ids interleaved, search_depth 1100: K = nmem = 1024 stays on the fast kernel, 1025 is
    handed over (status 5, FS_DEPTH).  The K-th entry ties with the next one, so id order alone
    decides who is in.  The pruning bound min(m_max, threshcount) / min(hashesperid) = 1/25 equals
    the K-th weight exactly, and so does every bucket group's m / hmin: pass 3 must run, read the
    groups and admit the tied single-record ids with larger ids, and only those."""
    sc = Scene(depth=128, hpi=1 << 20)
    mem = 2 * np.arange(1, nmem + 1)
    sng = 2 * np.arange(0, nmem + 8) + 1
    members(mem, sc, raw=2, hpi=50)
    singles(sng, sc, hpi=25)
    ref = run(sc, 1, 1100, (status, 5))
    assert len(ref.ids) == nmem and np.all(ref.w == 0.04) and 1 / 25 == 0.04
    assert ref.ids[-1] > 1 and np.any(np.isin(ref.ids, sng)) and np.any(np.isin(ref.ids, mem))
    wk, idk = kth(ref, nmem - 1)
    tied_out = np.setdiff1d(np.r_[mem, sng], ref.ids)
    assert len(tied_out) and np.all(tied_out < idk)


def test_publish_depth_beyond_the_members():
    """Publish mode, search_depth 50 over a query with 10 members and 500 single-record ids: the
    depth exceeds the members, so the weight bin is cut for all 10 and pass 3 fills the rest.  Each
    CTA first ranks a query whose 50th of 60 members sits in a much higher bin (the CTAs are
    persistent: nothing of that query's selection may leak into the next)."""
    import torch
    sc = Scene()
    members(np.arange(1, 61), sc, raw=4, hpi=np.arange(1, 61))
    singles(sc.fill(100), sc)
    q_high = sc.query()
    sc.rows = []
    members(np.arange(100, 110), sc, raw=2, hpi=1000)
    singles(sc.fill(500), sc)
    q_low = sc.query()
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    qs = [q_high] * nsm + [q_low] * nsm
    refs = [Ref(sc, q, 1, 50, 1) for q in (q_high, q_low)]
    assert refs[0].pcnt[0] == 50 and refs[0].pw[49] == 4 / 50
    assert refs[1].pcnt[0] == 50 and list(refs[1].pid[:10]) == list(range(109, 99, -1))
    ht = sc.ht()
    qoff = np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.int64)
    for force in (False, True):
        m = matcher(1, 1, 50, force=force)
        rows, roff, cand, cnts = m._publish_call(ht, np.ascontiguousarray(np.concatenate(qs)), qoff)
        st = Matcher.last_status(ht, len(qs))[:, 0]
        assert np.all(st == (-1 if force else 0)), st.tolist()
        for i in range(len(qs)):
            r = refs[i // nsm]
            assert tuple(cnts[i]) == r.pcnt and np.array_equal(cand[i, :50, 0].astype(np.int64), r.pid), (force, i)
            assert np.array_equal(cand[i, :50, 2].view(np.uint64), r.pw.view(np.uint64)), (force, i)
            assert np.array_equal(rows[roff[i]:roff[i + 1]], r.prows), (force, i)


@pytest.mark.parametrize("nmem,status", [(SCAP - XCAP, 0), (SCAP - XCAP + 1, 7)])
def test_ties_boundary(nmem, status):
    """nmem members of one weight 0.02 - raw 2 / 100 and raw 3 / 150 - all in one weight bin:
    2048 are gathered and sorted (status 0), 2049 hand the query over (status 7, FS_TIES).
    Single-record ids of the same weight (1 / 50) with larger ids enter through pass 3."""
    sc = Scene(depth=256)
    ids = np.arange(1, nmem + 1)
    members(ids[ids % 3 != 0], sc, raw=2, hpi=100, width=256)
    members(ids[ids % 3 == 0], sc, raw=3, hpi=150, width=256)
    singles(np.arange(nmem + 1, nmem + 6), sc, hpi=50)
    ref = run(sc, 1, 10, (status, status))
    assert np.all(ref.w == 0.02) and ref.ids[0] == nmem + 5 and ref.ids[5] == nmem


# ---- weights and ties at rank K-1 / K ----------------------------------------------------------
@pytest.mark.parametrize("single_side", ["above", "below"])
def test_equal_weights_from_different_pairs(single_side):
    """Weight 0.02 three ways - member 2/100, member 3/150, single-record 1/50 - straddling rank
    K = 5; the single-record id is the largest of the three (it is in) or the smallest (out)."""
    sc = Scene()
    members([1000, 1001, 1002], sc, raw=4, hpi=1)
    a, b, c = (200, 300, 400) if single_side == "above" else (300, 400, 200)
    members([a], sc, raw=2, hpi=100)
    members([b], sc, raw=3, hpi=150)
    members([10, 11, 12], sc, raw=2, hpi=1000)
    singles([c], sc, hpi=50)
    singles(sc.fill(500), sc, hpi=1 << 20)
    ref = run(sc, 1, 5, (0, 0))
    assert ref.w[3] == ref.w[4] == 0.02
    assert (c in ref.ids) == (single_side == "above")
    assert list(ref.ids[3:]) == sorted([a, b, c], reverse=True)[:2]


def same_float_pair():
    """Two hashesperid values h1 < h2 near 2^25 whose weights 8/h differ as doubles but have the
    same float32 image."""
    for h in range(1 << 25, (1 << 25) + 4096):
        w1, w2 = 8 / h, 8 / (h + 1)
        if w1 != w2 and np.float32(w1) == np.float32(w2):
            return h, h + 1
    raise AssertionError("no pair")


def test_weights_sharing_a_float_image():
    """Members of weights 8/h1 > 8/h2 that share one float32 image (one histogram bin): the larger
    weight has the SMALLER id, K falls between them, so only the exact double comparison gets it."""
    h1, h2 = same_float_pair()
    sc = Scene(hpi=1 << 30)
    members([50, 51], sc, raw=2, hpi=1000)
    members([7], sc, raw=8, hpi=h1)
    members([9], sc, raw=8, hpi=h2)
    members([3, 4], sc, raw=2, hpi=(1 << 26))
    singles(sc.fill(300), sc)
    ref = run(sc, 1, 3, (0, 0))
    assert list(ref.ids) == [51, 50, 7] and np.float32(8 / h1) == np.float32(8 / h2) and 8 / h1 > 8 / h2


def test_zero_hashesperid_members_and_singles():
    """hashesperid 0: weight inf, min(hashesperid) unknown (no pruning).  Three inf members and
    three inf single-record ids with interleaved ids, K = 4 falls among them."""
    sc = Scene()
    members([20, 40, 60], sc, raw=2, hpi=0)
    members([1, 2, 3, 4, 5], sc, raw=2, hpi=10)
    singles([30, 50, 70], sc, hpi=0)
    singles(sc.fill(500), sc)
    with np.errstate(divide="ignore"):
        ref = run(sc, 1, 4, (0, 0))
    assert list(ref.ids) == [70, 60, 50, 40] and np.all(np.isinf(ref.w))


@pytest.mark.parametrize("end", ["top", "bottom"])
def test_clamped_end_bins(end):
    """Weights at or above 2^8 (members with >= 256 hits and hashesperid 1) and at or below 2^-24
    (hashesperid >= 2^25) all fall in the histogram's clamped end bin; K falls inside it."""
    if end == "top":
        sc = Scene(hashbits=10, depth=16)
        for i, m in ((5, 300), (6, 256), (7, 260), (8, 256)):
            sc.hpi[i] = 1
            sc.group([i], m)
        members([1, 2], sc, raw=2, hpi=1)
        ref = run(sc, 1, 3, (0, 0))
        assert list(ref.ids) == [5, 7, 8] and ref.w[2] == 256.0
    else:
        sc = Scene(hpi=(1 << 31))
        members([100, 101], sc, raw=2, hpi=1)
        members([5, 6, 7], sc, raw=2, hpi=1 << 25)
        members([8], sc, raw=3, hpi=(1 << 26) + 1)
        members([9], sc, raw=2, hpi=(1 << 25) + 8)
        singles(sc.fill(300), sc)
        ref = run(sc, 1, 4, (0, 0))
        assert list(ref.ids) == [101, 100, 7, 6] and ref.w[2] == 2.0 ** -24


def test_bucket_probed_from_two_chunks():
    """A query of ~4,900 rows (three chunks of 2048 in the fast kernel): 39 buckets are probed once
    in the first chunk and again in the last, which makes their 78 ids members (weights 2/40 ..
    2/44).  Five single-record ids of weight 1/21 == 2/42 tie with members at rank K = 35, the
    pruning bound 1/21 equals the K-th member's weight: pass 3 reads every chunk."""
    sc = Scene(hashbits=14, depth=8, hpi=1 << 20)
    rng = np.random.default_rng(3)
    shared = []
    for i in range(1, 40):
        sc.hpi[[i, 3000 + i]] = 40 + i % 5
        shared.append(sc.group([i, 3000 + i], 1, qt=10, dt=100))
    for _ in range(4800):
        sc.group(sc.fill(8), 1, qt=int(rng.integers(0, 2000)))
    sng = sc.fill(5, hpi=21)
    sc.group(sng, 1, qt=5)
    for b in shared:
        sc.probe(b, 10)                                 # the same time: both hits align
    q = sc.query()
    assert len(q) > 2 * 2048 and np.all(np.isin(sc.counts[q[:39, 1]], 2))
    ref = run(sc, 1, 35, (0, 0), q=q)
    assert np.all(np.isin(sng, ref.ids)) and ref.w[34] == 2 / 42 == 1 / 21
    assert np.count_nonzero(np.isin(ref.ids, np.r_[np.arange(1, 40), np.arange(3001, 3040)])) == 30


# ---- general kernel edges ----------------------------------------------------------------------
@pytest.mark.parametrize("m", [255, 256, 510, 511])
def test_split_bucket_multiplicity(m):
    """A bucket probed m times from one hash at m query times (the general kernel splits records
    above 255 into several): raw counts m and m + 1 exactly, equal weights at rank K."""
    sc = Scene(hashbits=8, depth=1024, mtb=14)
    ids = np.arange(1, 9)
    sc.hpi[ids] = 7
    sc.hpi[[5, 7]] = 14
    b = sc.group(ids, 0, dt=600)
    for t in range(m):
        sc.probe(b, t)
    members(ids[:3], sc, raw=1, hpi=7)                 # raw m + 1 for ids 1-3
    ref = run(sc, 5, 5, (0, 0))
    assert list(ref.ids) == [3, 2, 1, 8, 6] and list(ref.raw) == [m + 1] * 3 + [m] * 2


def test_id_segment_edges():
    """Ids 32767/32768 and 65535/65536 (the general kernel counts ids in 32768-id segments) with
    equal weights around rank K."""
    sc = Scene(nids=1 << 17)
    members([32767, 32768, 65535, 65536], sc, raw=2, hpi=40)
    members([32766, 65537], sc, raw=3, hpi=60)
    members([10, 11], sc, raw=2, hpi=1)
    singles([32769, 65534], sc, hpi=20)
    singles(sc.fill(300), sc)
    ref = run(sc, 1, 6, (0, 0))
    assert list(ref.ids) == [11, 10, 65537, 65536, 65535, 65534]


@pytest.mark.parametrize("nq", [16384, 16385])
def test_sorted_and_unsorted_probe(nq):
    """16384 query rows are sorted in the general kernel's shared memory, 16385 take the unsorted
    probe; buckets probed by several rows at different times."""
    sc = Scene(hashbits=12, depth=8, hpi=1 << 20)
    rng = np.random.default_rng(nq)
    bs = []
    for i in range(1, 301):
        ids = np.r_[i, sc.fill(1)]
        sc.hpi[i] = 5 + i % 3
        bs.append(sc.group(ids, 1, qt=0, dt=300))
    while len(sc.rows) < nq:
        k = int(rng.integers(0, len(bs)))
        sc.probe(bs[k], int(rng.integers(0, 3)))
    q = sc.query()[:nq]
    q = q[rng.permutation(len(q))]
    ref = run(sc, 2, 200, (0, 0), q=q, paths=("fast", "general"))
    assert len(q) == nq and len(ref.rows) > 0


def test_radix_select_decided_by_id_digits():
    """3000 members of one weight (more than GCAP = 1024 undecided keys) with ids spread over three
    bytes, search_depth 1000: the general kernel's radix select runs out of weight digits and picks
    by id; the fast kernel hands the query over (status 7)."""
    sc = Scene(hashbits=8, depth=256, mtb=10, nids=1 << 21)
    rng = np.random.default_rng(9)
    ids = np.sort(rng.choice(np.arange(1, 1 << 21), 3000, replace=False))
    members(ids, sc, raw=2, hpi=77, width=250)
    ref = run(sc, 1, 1000, (7, 7))
    assert np.all(ref.w == 2 / 77) and np.array_equal(ref.ids, ids[::-1][:1000])


# ---- sharded merge -----------------------------------------------------------------------------
@pytest.mark.parametrize("nshards", [2, 3])
def test_sharded_merge_with_ties_across_shards(nshards):
    """Equal weights on both sides of rank D, spread over the shards: afp_shard_pack /
    afp_shard_merge with the shards visited one after another give the single table's rows."""
    import torch
    sc = Scene(nids=4000)
    tied = np.array([150, 1100, 1200, 2100, 2200, 2900, 900, 1900])
    members(tied, sc, raw=2, hpi=100)
    members([10, 1010, 2010], sc, raw=3, hpi=1)
    singles([1500, 2500, 500], sc, hpi=50)
    singles(sc.fill(200), sc)
    q = sc.query()
    sdepth, rcap = 7, 16
    ref = Ref(sc, q, 1, sdepth, 1)
    assert ref.w[sdepth - 1] == 0.02 and np.count_nonzero(ref.pw[:ref.pcnt[0]] == 0.02) > 0
    assert np.count_nonzero(np.isin(tied, ref.ids)) not in (0, len(tied))
    ht = sc.ht()
    ctx = ht._sync_device()
    m = matcher(1, 1, sdepth)
    qoff = np.array([0, len(q)], np.int64)
    rb = int(ctx.lib.afp_shard_record_bytes(sdepth, rcap))
    bufs = []
    for s in range(nshards):
        lo, hi = (sc.nids * s) // nshards, (sc.nids * (s + 1)) // nshards
        ht.restrict_device_ids(lo, hi)
        m._publish_call(ht, q, qoff)
        buf = torch.empty((1, rb), dtype=torch.uint8, device="cuda")
        ctx.check(ctx.lib.afp_shard_pack(ctx.h, rcap, buf.data_ptr()))
        bufs.append(buf)
    ht._touch()
    gathered = torch.cat(bufs, dim=0)
    total = C.c_int64(0)
    ctx.check(ctx.lib.afp_shard_merge(ctx.h, gathered.data_ptr(), nshards, 1, sdepth, rcap, C.byref(total)))
    rows = np.empty((int(total.value), 7), np.int32)
    roff = np.zeros(2, np.int64)
    ctx.check(ctx.lib.afp_fetch_match_rows(ctx.h, rows.ctypes.data if len(rows) else None, 1,
                                           roff.ctypes.data_as(C.POINTER(C.c_int64))))
    assert np.array_equal(rows, ref.rows)
