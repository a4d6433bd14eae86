"""CPU: on every family of tests/k4_mode_cases.py, k4_reference.rows_in_rank_order and the oracle's
offset_histogram_rows / time_range equal the reference's own _approx_match_counts, stored in
tests/golden/k4_modes.npz by oracle/make_golden_k4_modes.py.  With tests/test_gpu_k4_mode_edges.py
this closes the chain device == k4_reference == reference at the mode search's edges.  Also: a
negative threshcount is refused by the Python entry points before any device work."""
import os

import numpy as np
import pytest

from audfprint_b200 import HashTable, Matcher
from audfprint_b200 import dist
from oracle import afp_oracle as orc
from tests import k4_mode_cases as mc

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "k4_modes.npz")
CASES = {c.name: c for c in mc.all_cases()}


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as g:
        return {k: g[k] for k in g.files}


def test_golden_has_every_family(golden):
    assert sorted({k.split("/")[0] for k in golden}) == sorted(CASES)


@pytest.mark.parametrize("name", list(CASES))
def test_reference_rows_equal_golden(golden, name):
    case = CASES[name]
    mc.reached(case)
    roff = golden[name + "/roff"]
    assert len(roff) == len(case.queries) + 1
    for i in range(len(case.queries)):
        want = golden[name + "/rows"][roff[i]:roff[i + 1]]
        h = case.hits(i)
        ids, raw = case.candidates(i)
        assert np.array_equal(case.rows(i), want), (name, i)
        assert np.array_equal(orc.offset_histogram_rows(h, ids, raw, case.window, case.thresh, case.maxalign), want)
        for key, quant in (("t02", 0.02), ("t50", 0.5)):
            tr = golden[name + "/" + key][roff[i]:roff[i + 1]]
            assert np.array_equal(tr[:, :5], want[:, :5])
            got = [orc.time_range(h, int(r[0]), int(r[2]), case.window, quant) for r in want]
            assert np.array_equal(np.array(got, np.int64).reshape(-1, 2), tr[:, 5:]), (name, i, key)


def test_negative_threshcount_raises_before_any_device_work():
    """Matcher._params refuses threshcount < 0, so match_batch, match_hashes (with and without
    hashesfor), tables without a device copy (the options path) and the sharded match all raise."""
    class HostOnly:
        """A table with only get_hits (no device copy)."""
        def get_hits(self, q):
            raise AssertionError("reached the table")

    q = np.array([[0, 1], [3, 2]], np.int32)
    m = Matcher()
    m.threshcount = -1
    ht = HashTable(hashbits=10, depth=8, maxtime=1 << 12)
    calls = [lambda: m.match_batch(ht, [q]), lambda: m.match_hashes(ht, q), lambda: m.match_hashes(ht, q, 0),
             lambda: dist.match_sharded_batch(m, ht, (q, np.array([0, 2])))]
    for call in calls:
        with pytest.raises(ValueError, match="threshcount"):
            call()
    m.find_time_range = True
    for qs in ([q], [q, q]):
        with pytest.raises(ValueError, match="threshcount"):
            m.match_batch(HostOnly(), qs)
