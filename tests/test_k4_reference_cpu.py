"""CPU: the K4 reference of tests/k4_reference.py equals the oracle's own functions - match rows,
ranked candidates, the list a table shard publishes - on both match.npz databases and their
golden queries, and on small random tables with ties, hashesperid 0 and high bucket multiplicity.
With tests/test_oracle_golden.py (oracle == reference) this closes the chain that
tests/test_gpu_k4_ranking_edges.py relies on: CUDA == helper == oracle == reference."""
import numpy as np
import pytest

from audfprint_b200 import dist as afd
from oracle import afp_oracle as orc
from tests import cases
from tests import k4_reference as k4
from tests.conftest import expand_table

SETTINGS = [(2, 5, 100), (1, 2, 3), (1, 1, 1000), (0, 0, 7)]      # (window, threshcount, search_depth)


def check(table, counts, hashbits, depth, mtb, hpi, q, window, thresh, sdepth):
    h = k4.hits(table, counts, hashbits, depth, mtb, q)
    assert np.array_equal(h, orc.get_hits(table, counts, hashbits, depth, mtb, q))
    with np.errstate(divide="ignore"):
        want = orc.match_hashes(table, counts, hashbits, depth, mtb, hpi, q, window=window, threshcount=thresh,
                                search_depth=sdepth)
    got = k4.np_rows(table, counts, hashbits, depth, mtb, hpi, q, window, thresh, sdepth)
    assert np.array_equal(k4.by_count(got), want)
    if len(h) == 0:
        return
    ids, raw, w = k4.candidates(h, hpi, thresh, sdepth)
    with np.errstate(divide="ignore"):
        oid, oraw = orc.rank_candidates(h, hpi, thresh, sdepth)
    assert np.array_equal(ids, oid) and np.array_equal(raw, oraw)
    assert np.array_equal(got, orc.offset_histogram_rows(h, ids, raw, window, thresh))
    # the order is (weight desc, id desc), strictly
    assert np.all((w[:-1] > w[1:]) | ((w[:-1] == w[1:]) & (ids[:-1] > ids[1:])))
    # publish mode: depth over the distinct ids; merge_sharded_results of ONE shard gives the rows
    pid, praw, pw, (entries, n_above) = k4.candidates(h, hpi, thresh, sdepth, publish=True)
    uid, ucnt = np.unique(h[:, 0], return_counts=True)
    assert entries == min(len(uid), sdepth) == len(pid) and n_above == np.count_nonzero(ucnt > thresh)
    assert np.array_equal(pid[:len(ids)], ids) and np.array_equal(pw[:len(ids)], w)
    prows = k4.rows_in_rank_order(h, pid, praw, window, thresh)
    cand = np.stack([pid, praw, pw], axis=1)
    merged = afd.merge_sharded_results([{"n_above": n_above, "cand": cand, "rows": prows}], sdepth)
    assert np.array_equal(merged, got)


@pytest.mark.parametrize("db", ["db", "db2"])
def test_reference_equals_oracle_on_the_golden_databases(golden_match, db):
    table, counts, hashbits, depth, mtb, hpi = expand_table(golden_match, db)
    for j in range(cases.DB_QUERIES):
        for tag in ("clean", "noisy"):
            q = golden_match["q%d_%s/q" % (j, tag)]
            for window, thresh, sdepth in SETTINGS:
                check(table, counts, hashbits, depth, mtb, hpi, q, window, thresh, sdepth)
            # the golden hits are the reference's own get_hits
            h = k4.hits(table, counts, hashbits, depth, mtb, q)
            assert np.array_equal(h, golden_match["%s/q%d_%s/hits" % (db, j, tag)])


def test_reference_equals_oracle_on_ties_zero_hashesperid_and_multiplicity():
    """Weights tied through different (raw, hashesperid) pairs, hashesperid 0 (weight inf) and
    buckets probed up to 40 times at once."""
    rng = np.random.default_rng(17)
    hashbits, depth, mtb, nids = 8, 12, 10, 60
    nb = 1 << hashbits
    table = ((rng.integers(1, nids + 1, (nb, depth), dtype=np.int64) << mtb)
             + rng.integers(0, 300, (nb, depth))).astype(np.uint32)
    counts = rng.integers(0, depth + 3, nb).astype(np.int32)
    hpi = rng.choice(np.array([0, 25, 50, 100, 150, 300], np.uint32), nids)
    for seed, nq in ((0, 200), (1, 60), (2, 1), (3, 0)):
        r = np.random.default_rng(seed)
        q = np.stack([r.integers(0, 200, nq), r.integers(0, 40, nq)], 1).astype(np.int32)
        for window, thresh, sdepth in SETTINGS:
            check(table, counts, hashbits, depth, mtb, hpi, q, window, thresh, sdepth)
