"""The fast matching kernel (csrc/afp_match_fast.cu) against the oracle and against the general
kernel, on random tables big enough that most probed track ids are hit exactly once - the regime it
is built for - with pruning of single-record ids, pass 3 (single-record ids that DO outrank
members), no pruning (hashesperid == 0 referenced), hashed bitmap (> 2^20 ids), chunked long
queries, a member-set overflow handed to the general kernel, and table-shard (publish) mode.
Rows are compared with the oracle as sets, so a wrong id deep in the candidate list that yields no
row goes unseen here: tests/test_gpu_k4_ranking_edges.py compares the ranked lists themselves, in
order, and reaches each handover reason on both sides of its limit."""
import numpy as np
import pytest

from audfprint_b200 import HashTable, Matcher
from oracle import afp_oracle as orc

pytestmark = pytest.mark.gpu


def make_table(seed, hashbits, depth, nids, mtb=12, fill=1.0):
    rng = np.random.default_rng(seed)
    nb = 1 << hashbits
    table = ((rng.integers(1, nids, size=(nb, depth), dtype=np.int64) << mtb)
             + rng.integers(0, 1 << mtb, size=(nb, depth), dtype=np.int64)).astype(np.uint32)
    counts = np.full(nb, depth, np.int32)
    if fill < 1.0:
        counts = rng.integers(0, int(depth * 1.2) + 1, size=nb).astype(np.int32)     # ragged, some over-full
    return table, counts


def make_query(seed, nrows, hashbits, tmax=430, dup=0.35):
    """Rows (time, hash) sorted by (time, hash); a fraction of the hashes repeats at neighbouring
    times, as the 4 sub-frame shifts of a real query do (bucket multiplicity m up to 4)."""
    rng = np.random.default_rng(seed)
    base = np.stack([rng.integers(0, tmax, nrows), rng.integers(0, 1 << 20, nrows)], axis=1)
    extra = []
    for t, h in base[rng.random(nrows) < dup]:
        for k in range(1, int(rng.integers(2, 5))):
            extra.append((t + k, h))
    q = np.unique(np.concatenate([base, np.array(extra, np.int64).reshape(-1, 2)]), axis=0)
    return q.astype(np.int32)


def plant(table, counts, q, hashbits, depth, mtb, tid, delta, nrows, rng):
    """Put `nrows` entries of track `tid` where query rows will find them at offset `delta`."""
    pick = rng.choice(len(q), size=nrows, replace=False)
    for t, h in q[pick]:
        b = int(h) & ((1 << hashbits) - 1)
        n = min(depth, int(counts[b]))
        if n == 0:
            continue
        table[b, int(rng.integers(0, n))] = ((tid + 1) << mtb) + ((int(t) + delta) & ((1 << mtb) - 1))


def hpi_of(table, counts, depth, mtb, nids):
    valid = np.arange(depth)[None, :] < np.minimum(counts, depth)[:, None]
    return np.maximum(np.bincount((table[valid] >> mtb).astype(np.int64) - 1, minlength=nids), 1).astype(np.uint32)


def as_ht(table, counts, hashbits, depth, mtb, hpi):
    ht = HashTable(hashbits=hashbits, depth=depth, maxtime=1 << mtb)
    ht.table, ht.counts, ht.hashesperid = table, counts, hpi
    return ht


def check(ht, qs, window=2, thresh=5, sdepth=100, expect_general=None, maxal=100):
    table, counts, hpi = ht.table, ht.counts, ht.hashesperid
    m = Matcher()
    m.window, m.threshcount, m.search_depth, m.max_alignments_per_id = window, thresh, sdepth, maxal
    fast = m.match_batch(ht, qs, sort=False)
    ngen = Matcher.last_general_count(ht)
    status = Matcher.last_status(ht, len(qs))
    g = Matcher()
    g.window, g.threshcount, g.search_depth, g.max_alignments_per_id = window, thresh, sdepth, maxal
    g.force_general_kernel = True
    gen = g.match_batch(ht, qs, sort=False)
    assert Matcher.last_general_count(ht) == len(qs)
    for i, q in enumerate(qs):
        assert np.array_equal(fast[i], gen[i]), ("fast vs general", i)
        want = orc.match_hashes(table, counts, ht.hashbits, ht.depth, ht.maxtimebits, hpi, q, window=window,
                                threshcount=thresh, search_depth=sdepth, max_alignments_per_id=maxal)
        assert fast[i].shape == want.shape and sorted(map(tuple, fast[i])) == sorted(map(tuple, want)), i
    if expect_general is not None:
        assert ngen == expect_general, (ngen, status[:12].tolist())
    return fast, ngen


def publish_equal(ht, qs, sdepth=100, thresh=5):
    out = []
    for force in (False, True):
        m = Matcher()
        m.window, m.threshcount, m.search_depth = 2, thresh, sdepth
        m.force_general_kernel = force
        arrs = [np.asarray(q, np.int32) for q in qs]
        qoff = np.zeros(len(arrs) + 1, np.int64)
        qoff[1:] = np.cumsum([len(a) for a in arrs])
        rows, roff, cand, cnts = m._publish_call(ht, np.ascontiguousarray(np.concatenate(arrs)), qoff)
        out.append((rows, roff, cand, cnts, Matcher.last_general_count(ht)))
    (r0, o0, c0, n0, g0), (r1, o1, c1, n1, g1) = out
    assert np.array_equal(o0, o1) and np.array_equal(r0, r1) and np.array_equal(n0, n1)
    for i in range(len(qs)):
        k = n0[i, 0]
        assert np.array_equal(c0[i, :k], c1[i, :k]), i
    return g0


HB, DEPTH, MTB, NIDS = 19, 100, 12, 1 << 20        # 52 M entries over 1 M ids: hashesperid ~ 50


@pytest.fixture(scope="module")
def big():
    """A table in the regime of BASELINE configs[2] (scaled 2x down): a 1000-row query touches
    ~80k entries of ~77k different ids.  Eight queries, each with a planted true track."""
    table, counts = make_table(1, HB, DEPTH, NIDS, MTB)
    rng = np.random.default_rng(2)
    qs = [make_query(100 + i, 650 + 30 * i, HB) for i in range(8)]
    for i, q in enumerate(qs):
        plant(table, counts, q, HB, DEPTH, MTB, 5000 + i, 300 + 7 * i, 120, rng)
    plant(table, counts, qs[0], HB, DEPTH, MTB, 5000, 1500, 60, rng)          # a second alignment
    hpi = hpi_of(table, counts, DEPTH, MTB, NIDS)
    return table, counts, hpi, qs


def test_big_table_regime_all_queries_on_the_fast_kernel(big):
    table, counts, hpi, qs = big
    ht = as_ht(table, counts, HB, DEPTH, MTB, hpi)
    batch = qs[:6] + [np.zeros((0, 2), np.int32), qs[1][:1], qs[2][:7]]
    fast, ngen = check(ht, batch, expect_general=0)
    for i in range(6):
        assert len(fast[i]) >= 1 and fast[i][0, 0] == 5000 + i and fast[i][0, 2] == 300 + 7 * i
    assert len(fast[0]) >= 2
    check(ht, batch, window=0, thresh=4, sdepth=20, expect_general=0)
    check(ht, batch, window=0, thresh=3, sdepth=20)       # m = 4 > threshcount: most buckets' ids become members
    check(ht, batch, window=1, thresh=5, sdepth=1, expect_general=0)
    check(ht, batch, window=2, thresh=5, sdepth=100, maxal=0, expect_general=0)
    assert publish_equal(ht, batch) == 0


def test_single_record_ids_that_outrank_members_pass3(big):
    """Tracks with a tiny hashesperid reach the candidate list with ONE hit (weight 1/2 beats
    130/400): the reference ranks by raw/hashesperid (audfprint_match.py:136-146)."""
    table, counts, hpi, qs = big
    hpi = hpi.copy()
    rng = np.random.default_rng(4)
    hpi[5000:5008] = 400                                          # the true tracks are long ones
    light = rng.choice(NIDS, size=300, replace=False)
    hpi[light] = rng.integers(1, 3, size=300)                     # 300 very short tracks
    ht = as_ht(table, counts, HB, DEPTH, MTB, hpi)
    fast, ngen = check(ht, qs[4:8], thresh=4, sdepth=100, expect_general=0)
    # light ids really took the first candidate slots: the true track is found, not at rank 0
    assert all(len(r) and r[0, 0] == 5004 + i and r[0, 4] > 0 for i, r in enumerate(fast))
    check(ht, qs[4:8], thresh=5, sdepth=100, expect_general=0)
    check(ht, qs[4:8], thresh=2, sdepth=100)
    assert publish_equal(ht, qs[4:8]) == 0


def test_zero_hashesperid_referenced_no_pruning(big):
    table, counts, hpi, qs = big
    hpi = hpi.copy()
    rng = np.random.default_rng(6)
    hpi[rng.choice(NIDS, size=200, replace=False)] = 0           # weight = raw / 0 = inf for those
    ht = as_ht(table, counts, HB, DEPTH, MTB, hpi)
    check(ht, qs[:3], expect_general=0)


def test_long_query_is_chunked_and_dense_query_is_handed_over(big):
    table, counts, hpi, qs = big
    rng = np.random.default_rng(10)
    table = table.copy()
    counts = np.full(len(counts), 8, np.int32)                     # only 8 live slots per bucket
    long_q = make_query(500, 6000, HB, tmax=3000)                  # > 2048 rows: sorted in chunks
    plant(table, counts, long_q, HB, DEPTH, MTB, 31337, 444, 300, rng)
    ht = as_ht(table, counts, HB, DEPTH, MTB, hpi)
    assert len(long_q) > 3 * 2048
    fast, ngen = check(ht, [long_q, long_q[:100]], expect_general=0)
    assert fast[0][0, 0] == 31337 and fast[0][0, 2] == 444
    # a table of few ids: nearly every id is hit many times -> the member set overflows -> the
    # general kernel takes the query, same rows
    table2, counts2 = make_table(11, 14, 64, 20000, MTB)
    hpi2 = hpi_of(table2, counts2, 64, MTB, 20000)
    ht2 = as_ht(table2, counts2, 14, 64, MTB, hpi2)
    dense = make_query(501, 1500, 14)
    small = make_query(502, 20, 14, dup=0.0)
    fast2, ngen2 = check(ht2, [dense, small, dense[:900]])
    assert 1 <= ngen2 <= 2


def test_more_than_2_20_ids_hashed_bitmap():
    nids = 1500000
    table, counts = make_table(7, HB, DEPTH, nids, 11, fill=0.8)
    rng = np.random.default_rng(8)
    qs = [make_query(400 + i, 750, HB) for i in range(4)]
    for i, q in enumerate(qs):
        plant(table, counts, q, HB, DEPTH, 11, 1400000 + i, 20 * i, 100, rng)
    hpi = hpi_of(table, counts, DEPTH, 11, nids)
    ht = as_ht(table, counts, HB, DEPTH, 11, hpi)
    fast, ngen = check(ht, qs, expect_general=0)
    assert all(r[0, 0] == 1400000 + i for i, r in enumerate(fast))
    publish_equal(ht, qs)
