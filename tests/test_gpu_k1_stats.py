"""A file's spectrogram statistics (floor, mean) and everything computed from them must not depend
on where the file sits: alone, inside a device-resident batch, or inside a host-PCM batch that is
copied and processed in chunks.  K1 writes per-tile partials of those statistics, and the batch
layout decides which CTA computes which tile, whether a tile is staged by a bulk copy or by scalar
loads, and which tiles share a launch.  The per-file statistics are not exported, so the test
compares what they feed: the peaks and hashes of a file in every placement against the file
alone, and the conditioned spectrogram of the file alone across calls.

Covered: files shorter than one frame (512 samples), ragged lengths, a file that starts off a
16-byte boundary (scalar staging throughout), digital silence, a file whose floor bites (exact
zeros inside a track), and a batch whose tile count is not a multiple of K1's grid."""
import numpy as np
import pytest

from audfprint_b200 import Analyzer, _lib
from audfprint_b200.synth import synth_track
from tests import cases

pytestmark = pytest.mark.gpu

N_HOP = 256
FRAMES_PER_TILE = 16


def _tiles(n):
    frames = 1 + n // N_HOP if n >= 1 else 0
    return (frames + FRAMES_PER_TILE - 1) // FRAMES_PER_TILE


@pytest.fixture(scope="module")
def files():
    return [("short100", cases.adversarial_pcm("short100")),
            ("short300", cases.adversarial_pcm("short300")),
            ("short511", cases.adversarial_pcm("short511")),
            ("ragged", cases.adversarial_pcm("ragged")),
            ("zeros", cases.adversarial_pcm("zeros")),
            ("silence_gap", cases.adversarial_pcm("silence_gap")),
            ("track_ragged", synth_track(9001, 7.3)[:80471].copy())]


@pytest.fixture(scope="module")
def alone(files):
    """(sgram, peaks, hashes) of every file fingerprinted on its own, in both precisions."""
    out = {}
    for precision in ("fp64", "fp32"):
        an = Analyzer()
        an.precision = precision
        for name, x in files:
            out[precision, name] = (an.conditioned_sgram(x), an.find_peaks(x, 11025),
                                    an.fingerprint_batch([x])[0])
            # the same file alone twice: the statistics are recomputed from scratch every call
            assert np.array_equal(an.conditioned_sgram(x), out[precision, name][0])
    return out


def _layout(names, sigs, unaligned):
    """Pack signals, each file on a 16-byte boundary except those named in `unaligned`, which
    start 3 samples past one."""
    offs = np.zeros(len(sigs) + 1, np.int64)
    lens = np.array([len(s) for s in sigs], np.int64)
    starts = []
    pos = 0
    for n, s in zip(names, sigs):
        pos = (pos + 7) // 8 * 8 + (3 if n in unaligned else 0)
        starts.append(pos)
        pos += len(s)
    offs[:-1] = starts
    offs[-1] = pos
    buf = np.zeros(pos + 8, np.int16)
    for s, p in zip(sigs, starts):
        buf[p:p + len(s)] = s
    return buf, offs, lens


def _check_batch(an, pcm, offs, lens, names, alone, precision):
    """Fingerprint the batch; the peaks and hashes of every file of `alone` must be its own."""
    ctx = _lib.context(an.device)
    rows, roff = an.fingerprint_packed(pcm, offs, sample_lengths=lens)
    peaks = an._fetch_peaks(ctx, 0, len(lens))
    for i, name in enumerate(names):
        if (precision, name) not in alone:
            continue
        _, pk, h = alone[precision, name]
        assert peaks[i] == pk, (precision, name, "peaks")
        assert np.array_equal(rows[roff[i]:roff[i + 1]], h), (precision, name, "hashes")
    return rows, roff


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_device_batch_matches_alone(files, alone, precision):
    import torch
    an = Analyzer()
    an.precision = precision
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = sms * (2 if precision == "fp64" else 3)
    names = [n for n, _ in files]
    sigs = [x for _, x in files]
    # enough 20 s fillers that every CTA walks several tiles, then a short file so that the
    # tile count is not a multiple of the grid
    k = 0
    while sum(_tiles(len(s)) for s in sigs) < 3 * grid:
        names.append("filler%d" % k)
        sigs.append(synth_track(7000 + k, 20.0))
        k += 1
    if sum(_tiles(len(s)) for s in sigs) % grid == 0:
        names.append("pad")
        sigs.append(synth_track(7999, 1.0))
    assert sum(_tiles(len(s)) for s in sigs) % grid != 0
    buf, offs, lens = _layout(names, sigs, {"ragged"})
    assert (offs[names.index("ragged")] * 2) % 16 != 0
    dev = torch.from_numpy(buf).cuda()
    rows, roff = _check_batch(an, dev, offs, lens, names, alone, precision)
    # every third filler against its own single-file fingerprint
    for i, n in enumerate(names):
        if n.startswith("filler") and i % 3 == 0:
            assert np.array_equal(rows[roff[i]:roff[i + 1]], an.fingerprint_batch([sigs[i]])[0]), n


@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_host_chunked_batch_matches_alone(files, alone, precision):
    an = Analyzer()
    an.precision = precision
    # > 80 MB of host int16 PCM: the library copies and processes it in (two) chunks
    base = synth_track(77, 30.0)
    filler = np.tile(base, 35)
    names, sigs = [], []
    for i, (n, x) in enumerate(files):
        names.append(n)
        sigs.append(x)
        if i in (1, 3, 5):
            names.append("filler%d" % i)
            sigs.append(filler)
    names.append("filler_end")
    sigs.append(filler)
    buf, offs, lens = _layout(names, sigs, {"ragged"})
    assert buf.nbytes > (80 << 20)
    assert (offs[names.index("ragged")] * 2) % 16 != 0
    _check_batch(an, buf, offs, lens, names, alone, precision)
