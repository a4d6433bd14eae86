"""The device FLAC decoder (afp_flac_locate_batch / afp_flac_decode_batch) against the sequential
decoder of tests/flac_reference.py and FFmpeg's stored decodes of the edge corpus
(tests/golden/flac_edges.npz, tools/make_golden_flac_edges.py):
- every corpus stream, in one batched call (with sentinel gaps between the outputs) and file by file:
  FFmpeg's samples and the reference's status;
- 900 seeded random streams built here (random depth, channels, decorrelation, block sizes and codes,
  subframe kinds, orders, LPC precision and shift, Rice parameters, escapes, partition orders, wasted
  bits), in three batched calls, against the reference;
- a fixed-block-size stream of 70,000 frames (4-byte coded numbers) in a batch beside short ones."""
import os

import numpy as np
import pytest
import torch

from audfprint_b200 import _lib, flac
from tests import flac_reference as ref
from tests import flac_writer as fw

pytestmark = pytest.mark.gpu
SENTINEL = 0x5A5A


@pytest.fixture(scope="module")
def ge():
    from tests.conftest import GOLDEN
    return np.load(os.path.join(GOLDEN, "flac_edges.npz"))


def _batch(streams):
    """One locate + decode of `streams` with 37-sample sentinel gaps -> ([(pcm or None, status)], gaps ok)."""
    ctx = _lib.context(0)
    nsamples, status = flac.locate(ctx, streams)
    off, pos = [], 5
    for s, ns in zip(streams, nsamples):
        off.append(pos)
        pos += int(ns) * s.channels + 37
    out = torch.full((pos,), SENTINEL, dtype=torch.int16, device="cuda:0")
    with ctx.after_torch(out):
        st = flac.decode_into(ctx, out, off)
    got = out.cpu().numpy()
    keep = np.zeros(pos, bool)
    res = []
    for s, o, ns, x in zip(streams, off, nsamples, st):
        n = int(ns) * s.channels
        keep[o:o + n] = True
        res.append((got[o:o + n] if not x else None, int(x)))
    return res, bool(np.all(got[~keep] == SENTINEL))


def test_corpus_in_one_call(ge):
    names = [str(n) for n in ge["names"]]
    res, gaps = _batch([flac.parse(ge[n + "/flac"].tobytes()) for n in names])
    assert gaps
    for n, (pcm, st) in zip(names, res):
        assert st == int(ge[n + "/meta"][3]), (n, st)
        if st == 0:
            assert np.array_equal(pcm, ge[n + "/pcm"]), n


def test_corpus_file_by_file(ge):
    ctx = _lib.context(0)
    for n in [str(n) for n in ge["names"]]:
        s = flac.parse(ge[n + "/flac"].tobytes())
        nsamples, status = flac.locate(ctx, [s])
        want = int(ge[n + "/meta"][3])
        if status[0]:
            assert status[0] == want, n
            continue
        out = torch.empty(max(int(nsamples[0]) * s.channels, 1), dtype=torch.int16, device="cuda:0")
        with ctx.after_torch(out):
            st = flac.decode_into(ctx, out, [0])
        assert int(st[0]) == want, n
        if want == 0:
            assert np.array_equal(out.cpu().numpy()[:int(nsamples[0]) * s.channels], ge[n + "/pcm"]), n


def _random_stream(rng):
    """A seeded random FlacStream, or None when the writer cannot code the draw."""
    bps = int(rng.integers(4, 25))
    nch = int(rng.choice([1, 2, 2, 2, 3, 6, 8]))
    chmode = int(rng.choice([1, 8, 9, 10])) if nch == 2 else nch - 1
    nfr = int(rng.integers(1, 4))
    sizes = [int(rng.choice([1, 2, 5, 16, 31, 32, 64, 100, 192, 256, 576, 1024])) for _ in range(nfr)]
    variable = bool(rng.integers(2)) or len(set(sizes[:-1])) > 1
    top = (1 << (bps - 1)) - 1
    n = sum(sizes)
    wasted = int(rng.integers(0, min(bps, 6)))
    amp = int(rng.choice([top, top >> 3, 3]))
    x = rng.integers(-amp - 1, amp + 1, size=(n, nch))
    if rng.integers(3) == 0:
        x = np.cumsum(x, 0).clip(-top - 1, top)
    if nch == 2 and rng.integers(2):
        x[:, 1] = np.clip(x[:, 0] + rng.integers(-5, 5, size=n), -top - 1, top)
    x = (x >> wasted) << wasted

    def spec(bs):
        k = rng.integers(6)
        method = int(rng.integers(2))
        pos = [p for p in range(9) if bs % (1 << p) == 0]
        if bs < 4 or k == 0:
            return {"kind": "verbatim", "wasted": wasted}
        if k == 1:
            return {"kind": "fixed", "order": int(rng.integers(0, min(4, bs) + 1)), "wasted": wasted, "method": method}
        if k == 2:
            po = int(rng.choice(pos))
            o = int(rng.integers(0, min(4, bs >> po) + 1))
            esc = tuple(p for p in range(1 << po) if rng.integers(4) == 0)
            return {"order": o, "po": po, "method": method, "escape": esc, "wasted": wasted}
        o = int(rng.integers(1, min(32, bs) + 1))
        p = int(rng.integers(1, 16))
        c = rng.integers(-(1 << (p - 1)), 1 << (p - 1), size=o).tolist()
        return {"kind": "lpc", "coefs": c, "prec": p, "shift": int(rng.integers(0, 16)), "method": method,
                "wasted": wasted}

    specs = [[spec(bs) for _ in range(nch)] for bs in sizes]
    kw = {"sizes": sizes, "variable": variable, "chmode": chmode, "specs": lambda k: specs[k]}
    if chmode >= 8:
        kw["specs"] = lambda k: [dict(s, wasted=0) for s in specs[k]]
        x = x.copy()
    try:
        data, _ = fw.stream(x, bps, int(rng.choice([8000, 11025, 44100, 12345])), **kw)
    except Exception:
        return None
    return flac.parse(data)


def test_random_streams_equal_the_reference():
    rng = np.random.default_rng(90639)
    for call in range(3):
        streams = [s for s in (_random_stream(rng) for _ in range(300)) if s is not None]
        assert len(streams) > 250
        res, gaps = _batch(streams)
        assert gaps
        for k, (s, (pcm, st)) in enumerate(zip(streams, res)):
            want, wst = ref.decode(s)
            assert st == wst, (call, k, st, wst)
            if st == 0:
                assert np.array_equal(pcm, want), (call, k)


def test_a_stream_of_70000_frames_beside_short_ones(ge):
    saw = ((np.arange(70000 * 16, dtype=np.int64) * 3) % 200 - 100).reshape(-1, 1)
    long_data, _ = fw.stream(saw, 8, 11025, sizes=[16] * 70000, specs=[{"order": 1}])
    names = ["depth16", "ch8", "lpc_0"]
    streams = [flac.parse(ge[n + "/flac"].tobytes()) for n in names]
    streams.insert(1, flac.parse(long_data))
    res, gaps = _batch(streams)
    assert gaps
    want, st = ref.decode(streams[1])
    assert st == 0 and res[1][1] == 0 and np.array_equal(res[1][0], want)
    assert np.array_equal(want, (saw[:, 0] << 8).astype(np.int16))
    for n, (pcm, st) in zip(names, res[:1] + res[2:]):
        assert st == 0 and np.array_equal(pcm, ge[n + "/pcm"]), n
