"""GPU: 24-bit, 32-bit and float WAV and 17-24-bit FLAC through both front-ends, against FFmpeg's own
output (tests/golden/wide_pcm.npz) and against the 16-bit paths."""
import os

import numpy as np
import pytest

from tests import wide_pcm_cases as WC
from tests import wide_pcm_reference as W

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "wide_pcm.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def cases():
    return WC.cases()


def _as_s16(v):
    s = np.rint(np.asarray(v, np.float64) * 32768.0)
    assert np.array_equal(s / 32768.0, v)
    return s.astype(np.int16)


def _write(tmp_path, name, data):
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def test_list_form_equals_the_library(g, cases, tmp_path):
    """Every case through _frontend_sources (WAV payloads and device-decoded FLAC in one call)."""
    from audfprint_b200 import analyzer as A
    names = [c[0] for c in cases]
    srcs = [A._audio_read_raw(_write(tmp_path, "%d.%s" % (k, c[1]), c[4])) for k, c in enumerate(cases)]
    out, off, lens, status = A._frontend_sources([s[0] for s in srcs], [s[1] for s in srcs], [s[2] for s in srcs],
                                                 11025, device=0, resampler="ffmpeg")
    assert not status.any()
    host = out.cpu().numpy()
    for k, name in enumerate(names):
        got = _as_s16(host[off[k]:off[k] + lens[k]])
        assert WC.matches(g, "out_" + name, got), name


def test_per_file_reader_equals_the_library(g, cases, tmp_path):
    from audfprint_b200 import analyzer as A
    for k, (name, src, rate, ch, data, _, _) in enumerate(cases):
        if k % 7 and not name.startswith("special"):
            continue
        p = _write(tmp_path, "%d.%s" % (k, src), data)
        d, sr = A._wav_reader(p, sr=11025, resampler="ffmpeg", device=0)
        assert sr == 11025 and WC.matches(g, "out_" + name, _as_s16(d)), name


def _mixed_round(tmp_path):
    """16-bit WAV, 16-bit FLAC, s24 WAV, f32 WAV, 24-bit FLAC: 2 s stereo at 44.1 kHz each."""
    from tests import ffmpeg_frontend_cases as FC
    rng = np.random.default_rng(9)
    x16 = rng.integers(-32768, 32768, (88200, 2))
    x24 = rng.integers(-(1 << 23), 1 << 23, (88200, 2))
    files = [("a.wav", FC.wav_bytes(x16.reshape(-1), 44100, 2)),
             ("b.flac", FC.flac_bytes(x16[::-1].reshape(-1), 44100, 2)),
             ("c.wav", WC.wav_bytes(WC.payload_of(x24.reshape(-1), W.S24), 44100, 2, 1, 24)),
             ("d.wav", WC.wav_bytes(WC.payload_of(rng.uniform(-1, 1, 2 * 88200), W.F32), 44100, 2, 3, 32)),
             ("e.flac", WC.flac_bytes(x24[::-1], 24, 44100))]
    return [_write(tmp_path, n, d) for n, d in files]


@pytest.mark.parametrize("resampler", ["poly", "ffmpeg"])
def test_mixed_round_is_one_launch_and_keeps_16_bit_bits(tmp_path, resampler):
    from audfprint_b200 import _lib, analyzer as A
    fns = _mixed_round(tmp_path)
    srcs = [A._audio_read_raw(f) for f in fns]
    ctx = _lib.context(0)

    def run(items):
        return A._frontend_sources([s[0] for s in items], [s[1] for s in items], [s[2] for s in items], 11025,
                                   device=0, resampler=resampler)
    ctx.sync()
    n0 = ctx.launch_count()
    out, off, lens, status = run(srcs)
    ctx.sync()
    # locate (2 kernels) + decode (1) + one front-end launch for the five formats
    assert ctx.launch_count() - n0 == 4 and not status.any()
    o16, off16, lens16, _ = run(srcs[:2])
    for k in range(2):
        assert lens[k] == lens16[k]
        assert np.array_equal(out[off[k]:off[k] + lens[k]].cpu().numpy(), o16[off16[k]:off16[k] + lens16[k]].cpu().numpy())
    if resampler == "ffmpeg":
        for k in range(2, 5):
            raw = srcs[k][0]
            pay = raw.tobytes() if isinstance(raw, np.ndarray) else None
            if pay is None:            # the 24-bit FLAC: its samples left-justified
                x = np.frombuffer(srcs[2][0].tobytes(), np.uint8)
                pay = (W.left_justified(x, W.S24).reshape(-1, 2)[::-1]).tobytes()
            fmt = W.S32 if k == 4 else {np.dtype("<f4"): W.F32}.get(raw.dtype, W.S24)
            want = W.frontend(pay, fmt, 2, 44100)
            assert np.array_equal(_as_s16(out[off[k]:off[k] + lens[k]].cpu().numpy()), want), k


def test_poly_mode_takes_the_rule_1_int16(tmp_path, cases):
    """A new-format file in the default front-end is the int16 front-end fed rule (1)'s int16."""
    from audfprint_b200 import analyzer as A
    for k, (name, src, rate, ch, data, fmt, payload) in enumerate(cases):
        if k % 5 and not name.startswith("special"):
            continue
        p = _write(tmp_path, "%d.%s" % (k, src), data)
        d, _ = A._wav_reader(p, sr=11025, device=0)
        s16 = W.as_s16(payload, fmt)
        if src == "flac":                       # the poly front-end keeps today's int16 decode
            s16 = (W.left_justified(payload, W.S32) >> 16).astype(np.int16)
        if len(s16) == 0:
            assert len(d) == 0
            continue
        want = A.pcm_frontend(s16, ch, rate, 11025, device=0)
        assert np.array_equal(d, want), name


@pytest.mark.parametrize("name,rate,fmt", WC.SONGS)
def test_songs_give_the_reference_hashes(g, tmp_path, name, rate, fmt):
    from audfprint_b200 import Analyzer
    p = _write(tmp_path, name + ".wav", WC.song(rate, fmt)[0])
    an = Analyzer(resampler="ffmpeg")
    h = an.wavfile2hashes(p)
    assert np.array_equal(h, g[name + "_hashes"])
    assert np.array_equal(an.wavfiles2hashes([p])[0], h)


def test_list_forms_read_a_24_bit_corpus_as_its_ffmpeg_stream(tmp_path):
    """ingest_files, precompute_files and match_files on 24-bit stereo 44.1 kHz files give what they give
    on 16-bit mono 11025 Hz files holding the int16 stream ffmpeg makes of them."""
    from audfprint_b200 import Analyzer, HashTable, Matcher
    from tests import ffmpeg_frontend_cases as FC
    deep, flat = [], []
    for k in range(4):
        x = FC.song(44100, 30 + k, seconds=8.0).reshape(-1, 2).astype(np.int64) << 8
        x += np.random.default_rng(k).integers(0, 256, x.shape)
        pay = WC.payload_of(x.reshape(-1), W.S24)
        deep.append(_write(tmp_path, "d%d.wav" % k, WC.wav_bytes(pay, 44100, 2, 1, 24)))
        flat.append(_write(tmp_path, "f%d.wav" % k, FC.wav_bytes(W.frontend(pay, W.S24, 2, 44100), 11025, 1)))

    def run(files):
        an = Analyzer(resampler="ffmpeg")
        ht = HashTable(hashbits=18, depth=40, maxtime=1 << 14)
        counts = an.ingest_files(ht, files)
        pre = an.precompute_files(files, str(tmp_path / ("pre_" + os.path.basename(files[0])[0])))
        q = Analyzer(resampler="ffmpeg")
        q.shifts = 4
        lines = Matcher().files_match_to_msgs(q, ht, files)
        return ht, counts, pre, lines
    ht_d, c_d, pre_d, l_d = run(deep)
    ht_f, c_f, pre_f, l_f = run(flat)
    assert [c[1] for c in c_d] == [c[1] for c in c_f]
    assert np.array_equal(ht_d.table, ht_f.table) and np.array_equal(ht_d.counts, ht_f.counts)
    assert len(pre_d) == len(pre_f)

    def outputs(top):
        found = sorted(os.path.join(r, f) for r, _, fs in os.walk(str(tmp_path / top)) for f in fs)
        assert len(found) == 4
        return [open(f, "rb").read() for f in found]
    assert outputs("pre_d") == outputs("pre_f")
    assert repr(l_d).replace(str(tmp_path / "d"), str(tmp_path / "f")) == repr(l_f)
