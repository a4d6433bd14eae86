"""The sequential FLAC decoder of tests/flac_reference.py against FFmpeg 8.0's stored decodes
(tests/golden/flac.npz, tests/golden/flac_edges.npz), the coverage of the edge corpus, and the corpus
recipe against its stored bytes (tools/make_golden_flac_edges.py)."""
import os
import sys

import numpy as np
import pytest

from audfprint_b200 import flac
from tests import flac_reference as ref
from tests.conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden_flac_edges as recipe  # noqa: E402


@pytest.fixture(scope="module")
def ge():
    return np.load(os.path.join(GOLDEN, "flac_edges.npz"))


@pytest.fixture(scope="module")
def decoded(ge):
    rec, out = ref.Record(), {}
    for n in [str(n) for n in ge["names"]]:
        out[n] = ref.decode(flac.parse(ge[n + "/flac"].tobytes()), rec)
    return rec, out


def test_reference_equals_ffmpeg_on_flac_npz():
    g = np.load(os.path.join(GOLDEN, "flac.npz"))
    gb = np.load(os.path.join(GOLDEN, "bundled.npz"))
    for n in [str(n) for n in g["names"]]:
        pcm, status = ref.decode(flac.parse(g[n + "/flac"].tobytes()))
        assert status == int(g[n + "/meta"][3]), n
        if status:
            continue
        key = str(g[n + "/pcm_of"]) if n + "/pcm_of" in g.files else n
        want = gb["query/pcm"] if n == "bundled_query" else g[key + "/pcm"]
        assert np.array_equal(pcm, want), n


def test_reference_equals_ffmpeg_on_the_edge_corpus(ge, decoded):
    """Status 0 exactly where FFmpeg returned every written sample, and then FFmpeg's samples."""
    _, out = decoded
    for n, (pcm, status) in out.items():
        rate, nch, bps, want_status, nff, written = (int(v) for v in ge[n + "/meta"])
        assert status == want_status, n
        if status == 0:
            assert nff in (written, -2) or written == 0, n
            assert np.array_equal(pcm, ge[n + "/pcm"]), n
        else:
            # FFmpeg dropped a frame or gave up; none of these streams has CRC-16 damage, the one
            # documented case where FFmpeg reads a stream refused here
            assert nff < written, n


def test_the_corpus_reaches_every_edge(decoded):
    rec, _ = decoded
    s = rec.seen
    assert set(range(4, 25)) <= s["depth"]
    assert set(range(11)) <= s["chmode"]
    assert {(c, b) for c, b in ((1, 8), (2, 12), (4, 16), (5, 20), (6, 24))} | {(0, b) for b in range(4, 25)} <= \
        s["ss_code"]
    assert set(range(5, 26)) <= s["side_depth"]
    assert {(17, w) for w in range(1, 17)} | {(16, w) for w in range(1, 16)} <= s["wasted"]
    assert {("fixed", o) for o in range(5)} | {("lpc", o) for o in range(1, 33)} | \
        {("constant", 0), ("verbatim", 0)} <= s["subframe"]
    assert {2, 3, 4} <= s["fixed_bs_eq_order"] and s["first_partition_empty"]
    assert set(range(1, 16)) <= s["prec"] and set(range(16)) <= s["shift"] and set(range(1, 16)) <= s["coef_min"]
    assert s["lpc_sum_wide"] == {True}
    assert set(range(15)) <= s["rice0"] and set(range(31)) <= s["rice1"]
    assert set(range(32)) <= s["escape0"] and set(range(32)) <= s["escape1"]
    assert set(range(16)) <= s["po"]
    assert 65 in s["unary_long"]
    assert s["residual_extreme"] == {-(1 << 31) + 1, (1 << 31) - 1}
    assert 14 in s["quotient_limit"]
    assert set(range(1, 16)) <= s["bs_code"] and set(range(15)) <= s["sr_code"]
    assert {1, 2, 256} <= s["bs6"] and {1, 256, 65535} <= s["bs7"]
    assert {("fixed", k) for k in range(1, 7)} | {("variable", k) for k in range(1, 7)} <= s["numlen"]
    assert {ref.CHAIN, ref.RESERVED, ref.CORRUPT} <= s["refused"]


def test_the_recipe_makes_the_stored_bytes(ge):
    got = recipe.streams()
    assert [g[0] for g in got] == [str(n) for n in ge["names"]]
    for name, data, rate, nch, bps, written in got:
        assert data == ge[name + "/flac"].tobytes(), name
        assert [rate, nch, bps, written] == [int(v) for v in ge[name + "/meta"][[0, 1, 2, 5]]], name
