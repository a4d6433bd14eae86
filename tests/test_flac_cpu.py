"""FLAC input on the host: format dispatch by content, the metadata block parser, the int16
conversion rule against FFmpeg's stored output, and the fixture bit writer against the stored bytes
(tests/golden/flac.npz, tools/make_golden_flac.py)."""
import os
import sys
import wave

import numpy as np
import pytest

from audfprint_b200 import analyzer as an_mod
from audfprint_b200 import flac
from tests import flac_writer as fw
from tests.conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden_flac as recipe  # noqa: E402


@pytest.fixture(scope="module")
def gf():
    return np.load(os.path.join(GOLDEN, "flac.npz"))


def _bytes(gf, name):
    return gf[name + "/flac"].tobytes()


def test_parser_reads_streaminfo_and_skips_other_blocks(gf):
    s = flac.parse(_bytes(gf, "w_blocks"))          # PADDING, SEEKTABLE, VORBIS_COMMENT, APPLICATION
    assert (s.sample_rate, s.channels, s.bits_per_sample, s.max_blocksize, s.total_samples) == (11025, 1, 16, 3000,
                                                                                                 3000)
    plain = flac.parse(_bytes(gf, "w_total0"))
    assert plain.total_samples == 0 and np.array_equal(s.frames, plain.frames)
    for typ in (5, 6, 7, 126):                       # CUESHEET, PICTURE, reserved types: skipped
        data = b"fLaC" + fw.streaminfo(4096, 4096, 11025, 1, 16, 5000, last=False) + \
            fw.block_header(typ, 3, True) + b"xyz" + s.frames.tobytes()
        assert np.array_equal(flac.parse(data).frames, s.frames)


def test_parser_skips_id3v2(gf):
    a, b = flac.parse(_bytes(gf, "w_id3")), flac.parse(_bytes(gf, "w_total0"))
    assert np.array_equal(a.frames, b.frames)
    assert flac.is_flac(_bytes(gf, "w_id3")) and flac.id3v2_end(_bytes(gf, "w_id3")) == 310
    footer = b"ID3\x04\x00\x10\x00\x00\x00\x02ab" + b"3DI" + bytes(7) + _bytes(gf, "w_total0")
    assert flac.is_flac(footer)


@pytest.mark.parametrize("case", ["truncated", "type127", "not_first", "short_info", "two_info", "past_end"])
def test_malformed_block_chains_are_unreadable(case):
    si = fw.streaminfo(4096, 4096, 11025, 1, 16, 0, last=False)
    body = {
        "truncated": si[:20],
        "type127": si + fw.block_header(127, 0, True),
        "not_first": fw.block_header(1, 4, False) + bytes(4) + fw.streaminfo(4096, 4096, 11025, 1, 16, 0),
        "short_info": fw.block_header(0, 33, True) + bytes(33),
        "two_info": si + fw.streaminfo(4096, 4096, 11025, 1, 16, 0),
        "past_end": si + fw.block_header(1, 100, True) + bytes(10),
    }[case]
    with pytest.raises(IOError):
        flac.parse(b"fLaC" + body)


def _raised(f, *a):
    try:
        f(*a)
    except Exception as e:
        return type(e), str(e)
    return None


def test_dispatch_by_content(gf, tmp_path):
    fn = str(tmp_path / "a.wav")                    # a FLAC file whatever its name says
    with open(fn, "wb") as f:
        f.write(_bytes(gf, "w_id3"))
    s, nch, fs = an_mod._audio_read_raw(fn)
    assert isinstance(s, flac.FlacStream) and (nch, fs) == (1, 11025)
    w = str(tmp_path / "b.flac")                    # a WAV file whatever its name says
    with wave.open(w, "wb") as f:
        f.setnchannels(2)
        f.setsampwidth(2)
        f.setframerate(8000)
        f.writeframes(np.arange(10, dtype=np.int16).tobytes())
    raw, nch, fs = an_mod._audio_read_raw(w)
    assert np.array_equal(raw, np.arange(10)) and (nch, fs) == (2, 8000)
    # anything else fails as a non-WAV always has: Ogg-FLAC, ID3v2 before something that is not FLAC
    for name, data in (("ogg", b"OggS\x00\x02" + bytes(40) + b"\x7fFLAC"), ("id3mp3", b"ID3\x04\x00\x00\x00\x00\x00\x00"
                                                                               + b"\xff\xfb\x90" + bytes(40))):
        p = str(tmp_path / name)
        with open(p, "wb") as f:
            f.write(data)
        got = _raised(an_mod._audio_read_raw, p)
        assert got is not None and got == _raised(an_mod._wav_read_raw, p), name


def test_conversion_rule_is_ffmpegs(gf):
    """x << (16 - b) up to 16 bits, x >> (b - 16) above: FFmpeg's `-ac 1 -ar 11025 -f s16le` output."""
    names = [n[:-len("/source")] for n in gf.files if n.endswith("/source")]
    assert {"w_depth4", "w_depth8", "w_depth12", "w_depth20", "w_depth24", "ff_s24_mono"} <= set(names)
    for name in names:
        x = gf[name + "/source"].astype(np.int64)
        b = int(gf[name + "/meta"][2])
        rule = (x << (16 - b)) if b <= 16 else (x >> (b - 16))
        assert np.array_equal(rule.astype(np.int16), gf[name + "/ffmpeg_s16"]), name


def test_writer_makes_the_stored_bytes(gf):
    cases = recipe.writer_cases()
    assert [c[0] for c in cases] == [str(n) for n in gf["writer_names"]]
    for name, pcm, bps, rate, status, kw in cases:
        assert fw.stream(pcm, bps, rate, **kw)[0] == _bytes(gf, name), name
