"""CPU: the oracle against outputs of the reference on seeds and parameter settings that the other
golden files do not cover, stored in tests/golden/live_reference.npz by oracle/make_golden_live.py
(which also holds the reference-side code that produced them)."""
import os

import numpy as np
import pytest

from audfprint_b200.synth import synth_track, synth_query, pcm_to_float
from oracle import afp_oracle as orc
from oracle.make_golden_live import ANALYZER_PARAMS, MATCHER_PARAMS, SEEDS, SPREAD_CASES
from tests.conftest import GOLDEN


@pytest.fixture(scope="module")
def live():
    return np.load(os.path.join(GOLDEN, "live_reference.npz"))


def test_oracle_equals_live_reference_on_fresh_seeds(live):
    ref = {k[len("seeds/"):]: live[k] for k in live.files if k.startswith("seeds/")}
    tracks = []
    for seed in SEEDS:
        d = pcm_to_float(synth_track(seed, 14.0 + seed % 5))
        for shifts in (1, 4):
            got = orc.fingerprint(d, shifts=shifts)
            assert np.array_equal(got, ref["h_%d_%d" % (seed, shifts)].reshape(-1, 2)), (seed, shifts)
        tracks.append(orc.fingerprint(d, shifts=1))
    import random
    rng = random.Random(4)
    t = orc.Table(hashbits=14, depth=6, maxtimebits=12)
    for i, h in enumerate(tracks):
        t.store("s%d" % i, h, rng)
    assert np.array_equal(t.table, ref["table"]) and np.array_equal(t.counts, ref["counts"])
    hpi = ref["hpi"]
    for j, seed in enumerate(SEEDS):
        q, _ = synth_query(synth_track(seed, 14.0 + seed % 5), 77 + j, seconds=6.0, noise_sigma=0.01)
        qh = orc.fingerprint(pcm_to_float(q), shifts=4)
        assert np.array_equal(qh, ref["q_%d" % seed].reshape(-1, 2))
        hits = orc.get_hits(t.table, t.counts, 14, 6, 12, qh)
        assert np.array_equal(hits, ref["hits_%d" % seed].reshape(-1, 4))
        rows = orc.match_hashes(t.table, t.counts, 14, 6, 12, hpi, qh, window=2, threshcount=3, search_depth=4)
        want = ref["rows_%d" % seed].reshape(-1, 7)
        assert rows.shape == want.shape and np.array_equal(rows[:1], want[:1]), seed   # best match identical
        assert sorted(map(tuple, rows[:, :4])) == sorted(map(tuple, want[:, :4]))        # same alignments


def test_oracle_equals_live_reference_on_non_default_parameters(live):
    """The parameter settings the GPU tests check against the ORACLE only
    (test_non_default_analyzer_parameters_vs_oracle, test_matcher_edge_parameters_vs_oracle) -
    density / fanout / shifts / f_sd / maxpksperframe and window / threshcount / search_depth /
    max_alignments_per_id - checked here oracle vs reference, which closes the chain."""
    ref = {k[len("params/"):]: live[k] for k in live.files if k.startswith("params/")}
    for k, (density, fanout, shifts, f_sd, maxpks) in enumerate(ANALYZER_PARAMS):
        for i in range(2):
            d = pcm_to_float(synth_track(6000 + 10 * k + i, 9.0 + i))
            got = orc.fingerprint(d, density=density, fanout=fanout, shifts=shifts, f_sd=f_sd, maxpks=maxpks)
            assert np.array_equal(got, ref["h_%d_%d" % (k, i)].reshape(-1, 2)), (k, i)
            if shifts == 1:
                pk = orc.find_peaks(d, density=density, f_sd=f_sd, maxpks=maxpks)
                assert np.array_equal(np.array(pk, np.int32).reshape(-1, 2), ref["p_%d_%d" % (k, i)].reshape(-1, 2)), (k, i)
    table, counts, hpi = ref["table"], ref["counts"], ref["hpi"]
    nexact = 0
    for k, (window, thresh, sdepth, maxal) in enumerate(MATCHER_PARAMS):
        for j in range(4):
            qh = ref["q_%d" % j].reshape(-1, 2)
            want = ref["rows_%d_%d" % (k, j)].reshape(-1, 7)
            rows = orc.match_hashes(table, counts, 12, 8, 14, hpi, qh, window=window, threshcount=thresh,
                                    search_depth=sdepth, max_alignments_per_id=maxal)
            assert rows.shape == want.shape and np.array_equal(rows[:, 1], want[:, 1]), (k, j)
            # rank order among equal weights / equal counts is implementation-defined in the reference
            assert sorted(map(tuple, rows[:, :4])) == sorted(map(tuple, want[:, :4])), (k, j)
            nexact += int(np.array_equal(rows, want))
    assert nexact >= 12


def test_spread_local_maxes_equals_reference_spreadpeaksinvector(live):
    """The stand-alone method north_star names (audfprint_analyze.py:153-160): the oracle function
    the GPU test compares afp_spread_peaks with, against the reference's own method."""
    for i, (n, width) in enumerate(SPREAD_CASES):
        v, want = live["spread/%d/in" % i], live["spread/%d/out" % i]
        assert len(v) == n
        got = orc.spread_local_maxes(v, orc.gaussian_table(n, width))
        assert np.array_equal(got, want), (n, width)
