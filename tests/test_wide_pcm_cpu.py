"""CPU: the NumPy statement of 24-bit, 32-bit, float and deep-FLAC input (tests/wide_pcm_reference.py)
against FFmpeg's own output (tests/golden/wide_pcm.npz, oracle/make_golden_wide_pcm.py), and the RIFF
walk of the default reader (analyzer._wav_parse) on every chunk case and refused coding."""
import os
import struct
import wave

import numpy as np
import pytest

from audfprint_b200 import analyzer as an_mod
from tests import wide_pcm_cases as WC
from tests import wide_pcm_reference as W

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "wide_pcm.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def test_statement_equals_the_library(g):
    cases = WC.cases()
    assert len(cases) > 900
    for name, _, rate, ch, _, fmt, payload in cases:
        assert WC.matches(g, "out_" + name, W.frontend(payload, fmt, ch, rate)), name


def test_specials_take_the_librarys_rules(g):
    """NaN, +-Inf and +-2e9 give -32768 under the packed rule; the last n % 16 frames at equal rates
    take the scalar rule, where they give 0 or wrap."""
    v = np.array([np.nan, np.inf, -np.inf, 2e9, -2e9, 1.5, -1.5, 0.5 / 32768, 1.5 / 32768], np.float32)
    assert W.s16_rule(v).tolist() == [-32768, -32768, -32768, -32768, -32768, 32767, -32768, 0, 2]
    assert W.scalar_s16_rule(v[:5]).tolist() == [0, 0, 0, -32768, 32767]         # low 32 bits of 2^16 1e9
    special = [n for n in g.files if n.startswith("out_special_")]
    assert all(WC.matches(g, n, g[n]) for n in special)
    assert len(special) == 4


def _write(tmp_path, name, data):
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def test_riff_walk_gives_the_payload_ffmpeg_decodes(g, tmp_path):
    for name, data, fmt, ch, payload in WC.chunk_cases():
        p = _write(tmp_path, name + ".wav", data)
        got, code, nch, fs = an_mod._wav_parse(p)
        assert (code, nch) == (fmt, ch) and bytes(got) == bytes(payload), name
        assert fs == struct.unpack_from("<I", data, data.index(b"fmt ") + 12)[0], name
        assert WC.matches(g, "chunk_" + name, W.frontend(got, code, nch, fs)), name
        raw, nch2, fs2 = an_mod._wav_read_raw(p)
        assert (nch2, fs2) == (nch, fs) and raw.tobytes() == bytes(payload), name


def test_riff_walk_keeps_whole_frames(tmp_path):
    p24 = WC.payload_of(np.arange(-300, 300), W.S24)
    p = _write(tmp_path, "cut.wav", WC.wav_bytes(p24[:-5], 8000, 2, 1, 24, data_size=len(p24)))
    got, code, nch, _ = an_mod._wav_parse(p)
    assert code == W.S24 and nch == 2 and bytes(got) == p24[:len(p24) - 6]


def test_sixteen_bit_files_read_as_before(tmp_path):
    rng = np.random.default_rng(3)
    x = rng.integers(-32768, 32768, 2 * 501).astype("<i2")
    p = str(tmp_path / "s.wav")
    with wave.open(p, "wb") as w:
        w.setnchannels(2)
        w.setsampwidth(2)
        w.setframerate(44100)
        w.writeframes(x.tobytes())
    raw, nch, fs = an_mod._wav_read_raw(p)
    assert raw.dtype == np.dtype("<i2") and np.array_equal(raw, x) and (nch, fs) == (2, 44100)
    ext = _write(tmp_path, "x.wav", WC.wav_bytes(x.tobytes(), 44100, 2, 1, 16, extensible=True, mask=3))
    raw, nch, fs = an_mod._wav_read_raw(ext)
    assert raw.dtype == np.dtype("<i2") and np.array_equal(raw, x)


def _raised(fn, *a):
    try:
        fn(*a)
    except Exception as e:          # noqa: BLE001 - the point is to compare what is raised
        return type(e), str(e)
    return None


def test_refused_codings_keep_their_message(tmp_path):
    """8-bit PCM, 64-bit float, A-law and mu-law (plain or EXTENSIBLE) stay unreadable, with the message
    the wave module gave them."""
    pay = bytes(64)
    cases = {
        "u8": (WC.wav_bytes(pay, 8000, 1, 1, 8), (OSError, "only 16-bit PCM WAV is supported, got 1-byte samples")),
        "u8x": (WC.wav_bytes(pay, 8000, 1, 1, 8, extensible=True, mask=4),
                (OSError, "only 16-bit PCM WAV is supported, got 1-byte samples")),
        "f64": (WC.wav_bytes(pay, 8000, 1, 3, 64), (wave.Error, "unknown format: 3")),
        "f64x": (WC.wav_bytes(pay, 8000, 1, 3, 64, extensible=True, mask=4),
                 (wave.Error, "unknown extended format: 00000003-0000-0010-8000-00aa00389b71")),
        "alaw": (WC.wav_bytes(pay, 8000, 1, 6, 8), (wave.Error, "unknown format: 6")),
        "mulaw": (WC.wav_bytes(pay, 8000, 1, 7, 8), (wave.Error, "unknown format: 7")),
        "mulawx": (WC.wav_bytes(pay, 8000, 1, 7, 8, extensible=True, mask=4),
                   (wave.Error, "unknown extended format: 00000007-0000-0010-8000-00aa00389b71")),
        "adpcm": (WC.wav_bytes(pay, 8000, 1, 2, 4), (wave.Error, "unknown format: 2")),
        # FFmpeg decodes a 32-bit container with fewer valid bits as packed 24-bit samples: garbage
        "valid24_s32x": (WC.wav_bytes(pay, 8000, 1, 1, 32, extensible=True, valid_bits=24, mask=4),
                         (OSError, "32-bit PCM WAV with 24 valid bits is not supported")),
    }
    for name, (data, want) in cases.items():
        p = _write(tmp_path, name + ".wav", data)
        assert _raised(an_mod._wav_read_raw, p) == want, name
        assert _raised(an_mod._wav_reader, p, 11025, 1) == want, name
    # the wave module's own messages for these, as the parent read them
    for name in ("u8", "alaw", "mulawx", "f64", "f64x"):
        p = str(tmp_path / (name + ".wav"))
        got = _raised(wave.open, p, "rb")
        if got is not None:
            assert got == cases[name][1], name


def test_planner_counts_the_payload_bytes(tmp_path):
    from audfprint_b200 import Analyzer
    an = Analyzer()
    sizes = {}
    for name, fmt, tag, bits, ext in WC.WAV_KINDS:
        x = WC.signal("noise", 1000, 2, fmt, bits, np.random.default_rng(1), None)
        p = _write(tmp_path, name + ".wav", WC.wav_bytes(WC.payload_of(x.reshape(-1), fmt), 11025, 2, tag, bits, ext,
                                                         mask=3 if ext else 0))
        sizes[name] = an._read_item(0, p, 1, False)[3]
    assert sizes == {"s24": 6000, "s24x": 6000, "s32": 8000, "s32x": 8000, "f32": 8000, "f32x": 8000}
