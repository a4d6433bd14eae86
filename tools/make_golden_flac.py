"""Recipe of tests/golden/flac.npz: FLAC files and FFmpeg's decode of each.

Files come from two encoders:
  - FFmpeg's own FLAC encoder (the FFmpeg 8.0 libraries vendored in the opencv-python-headless wheel,
    driven through ctypes as oracle/ffdecode.py drives the decoder), from seeded PCM: compression
    levels 0-12, every ch_mode, every lpc_type, small / default / 65535-sample frames, 1, 2, 6 and 8
    channels, s16 and 24-bit input, digital silence, full-scale noise, a file shorter than one block,
    and the bundled query (tests/golden/bundled.npz);
  - the bit writer of tests/flac_writer.py, for what FFmpeg's encoder does not emit (variable block
    size, escape partitions, LPC order 32, explicit header codes, 4-20-bit depths, wasted bits with a
    side channel, an ID3v2 prefix, STREAMINFO with 0 samples, metadata blocks FFmpeg does not write, a
    sync pattern inside a frame's samples) and damaged copies.
Every decodable file is decoded by FFmpeg (oracle/ffdecode.py at the file's rate and channels, s16)
and that decode, which must equal the source PCM converted to int16 (x << (16 - b) up to 16 bits,
x >> (b - 16) above), is stored beside the file (`name/pcm`, or `name/pcm_of` naming the file whose
`pcm` holds the same samples).  Mono 11025 Hz files of 8, 12, 20 and 24 bits also
store FFmpeg's `-ac 1 -ar 11025 -f s16le` output, which pins the conversion.

    python tools/make_golden_flac.py        (needs the opencv-python-headless wheel)
Stores only data; nothing of FFmpeg is copied."""
from __future__ import annotations

import ctypes as C
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ffdecode                  # noqa: E402
from tests import flac_writer as fw          # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "flac.npz")
AV_SAMPLE_FMT_S16, AV_SAMPLE_FMT_S32 = 1, 2
AVERROR_EAGAIN, AVERROR_EOF = -11, -541478725


def convert(x, bps):
    """The int16 ffmpeg's FLAC decoder and libswresample make of a bps-bit sample."""
    x = np.asarray(x, np.int64)
    return (x << (16 - bps) if bps <= 16 else x >> (bps - 16)).astype(np.int16)


def source(seed, n, nch, bps, kind="music"):
    """Seeded int PCM (n, nch) at bps bits: sines plus noise, silence or full-scale noise."""
    rng = np.random.default_rng(seed)
    top = (1 << (bps - 1)) - 1
    if kind == "silence":
        return np.zeros((n, nch), np.int64)
    if kind == "noise":
        return rng.integers(-top - 1, top + 1, size=(n, nch))
    t = np.arange(n)[:, None] / 11025.0
    f = rng.uniform(80, 3000, size=(4, nch))
    x = sum(np.sin(2 * np.pi * f[k] * t + k) / (k + 1) for k in range(4)) * 0.35
    x += rng.normal(0, 0.02, size=(n, nch))
    return np.clip(np.round(x * top), -top - 1, top).astype(np.int64)


# ---- FFmpeg's encoder through ctypes ----------------------------------------------------------
_frame_fields = None


def _probe_frame_fields(u, s, c, f):
    """Offsets of AVFrame.ch_layout and AVFrame.sample_rate (no accessor exists), found in a frame
    the pcm_s16le decoder fills for a 3-channel 37011 Hz WAV, by their known values."""
    global _frame_fields
    if _frame_fields:
        return _frame_fields
    import wave
    with tempfile.TemporaryDirectory() as d:
        fn = os.path.join(d, "probe.wav")
        with wave.open(fn, "wb") as w:
            w.setnchannels(3)
            w.setsampwidth(2)
            w.setframerate(37011)
            w.writeframes(np.zeros(6144, np.int16).tobytes())
        fmt = C.c_void_p()
        assert f.avformat_open_input(C.byref(fmt), fn.encode(), None, None) == 0
        f.avformat_find_stream_info(fmt, None)
        dec = C.c_void_p()
        idx = f.av_find_best_stream(fmt, 1, -1, -1, C.byref(dec), 0)
        streams = ffdecode._rd(fmt.value, 48, C.c_void_p)
        st = ffdecode._rd(streams, 8 * idx, C.c_void_p)
        ctx = C.c_void_p(c.avcodec_alloc_context3(dec))
        par = ffdecode._rd(st, 16, C.c_void_p)
        # AVCodecParameters {codec_type, codec_id, codec_tag, extradata, extradata_size, coded_side_data,
        # nb_coded_side_data, format}: audio, PCM_S16LE, s16
        assert (ffdecode._rd(par, 0, C.c_int), ffdecode._rd(par, 4, C.c_int), ffdecode._rd(par, 44, C.c_int)) == \
            (1, 0x10000, AV_SAMPLE_FMT_S16), "AVCodecParameters layout"
        c.avcodec_parameters_to_context(ctx, par)
        assert c.avcodec_open2(ctx, dec, None) == 0
        pkt, frm = C.c_void_p(c.av_packet_alloc()), C.c_void_p(u.av_frame_alloc())
        assert f.av_read_frame(fmt, pkt) >= 0
        c.avcodec_send_packet(ctx, pkt)
        assert c.avcodec_receive_frame(ctx, frm) == 0
        raw = C.string_at(frm.value, 1024)
        # a plain WAV has no channel mask: the layout is {UNSPEC, 3 channels, 0}
        chl = [o for o in range(120, 1000, 8) if raw[o:o + 16] == (3 << 32).to_bytes(16, "little")]
        rate = [o for o in range(120, 1000, 4) if raw[o:o + 4] == (37011).to_bytes(4, "little")]
        assert len(chl) == 1 and len(rate) == 1, (chl, rate)
        c.av_packet_free(C.byref(pkt))
        u.av_frame_free(C.byref(frm))
        c.avcodec_free_context(C.byref(ctx))
        f.avformat_close_input(C.byref(fmt))
    _frame_fields = (chl[0], rate[0])
    return _frame_fields


def ff_encode(pcm, rate, bps, level=5, frame_size=0, opts=None):
    """FLAC file bytes FFmpeg's encoder makes of int (n, nch) pcm: 'fLaC', a STREAMINFO written here
    (FFmpeg's own is final only at the end of the stream; MD5 0 = not given) and FFmpeg's frames."""
    u, s, c, f = ffdecode._load()
    vp = C.c_void_p
    c.avcodec_find_encoder_by_name.restype = vp
    c.avcodec_send_frame.argtypes = [vp, vp]
    c.avcodec_receive_packet.argtypes = [vp, vp]
    u.av_opt_set_int.argtypes = [vp, C.c_char_p, C.c_int64, C.c_int]
    c.avcodec_parameters_alloc.restype = vp
    c.avcodec_parameters_from_context.argtypes = [vp, vp]
    c.avcodec_parameters_free.argtypes = [C.POINTER(vp)]
    u.av_opt_set_chlayout.argtypes = [vp, C.c_char_p, C.POINTER(ffdecode.AVChannelLayout), C.c_int]
    u.av_dict_set.argtypes = [C.POINTER(vp), C.c_char_p, C.c_char_p, C.c_int]
    u.av_frame_get_buffer.argtypes = [vp, C.c_int]
    chl_off, rate_off = _probe_frame_fields(u, s, c, f)
    pcm = np.asarray(pcm, np.int64).reshape(len(pcm), -1)
    n, nch = pcm.shape
    enc = c.avcodec_find_encoder_by_name(b"flac")
    ctx = vp(c.avcodec_alloc_context3(enc))
    sfmt = AV_SAMPLE_FMT_S16 if bps <= 16 else AV_SAMPLE_FMT_S32
    lay = ffdecode.AVChannelLayout()
    u.av_channel_layout_default(C.byref(lay), nch)
    assert u.av_opt_set_int(ctx, b"ar", rate, 0) >= 0
    assert u.av_opt_set_chlayout(ctx, b"ch_layout", C.byref(lay), 0) >= 0
    # the sample format has no option: it goes in through AVCodecParameters.format (offset 44, checked on
    # a decoder's parameters in _probe_frame_fields)
    par = vp(c.avcodec_parameters_alloc())
    assert c.avcodec_parameters_from_context(par, ctx) >= 0
    C.c_int.from_address(par.value + 44).value = sfmt
    assert c.avcodec_parameters_to_context(ctx, par) >= 0
    c.avcodec_parameters_free(C.byref(par))
    assert u.av_opt_set_int(ctx, b"compression_level", level, 0) >= 0
    if bps > 16:
        assert u.av_opt_set_int(ctx, b"bits_per_raw_sample", bps, 0) >= 0
    if frame_size:
        assert u.av_opt_set_int(ctx, b"frame_size", frame_size, 0) >= 0
    d = vp()
    for k, v in (opts or {}).items():
        u.av_dict_set(C.byref(d), k.encode(), str(v).encode(), 0)
    assert c.avcodec_open2(ctx, enc, C.byref(d)) == 0, "avcodec_open2"
    fs = C.c_int64()
    u.av_opt_get_int(ctx, b"frame_size", 0, C.byref(fs))
    fs = int(fs.value)
    pkt = vp(c.av_packet_alloc())
    frames, sizes = [], []

    def drain():
        while True:
            r = c.avcodec_receive_packet(ctx, pkt)
            if r in (AVERROR_EAGAIN, AVERROR_EOF):
                return
            assert r == 0, r
            frames.append(C.string_at(ffdecode._rd(pkt.value, 24, vp), ffdecode._rd(pkt.value, 32, C.c_int)))
            c.av_packet_unref(pkt)
    wide = pcm << (32 - bps) if bps > 16 else pcm
    for start in range(0, n, fs):
        blk = wide[start:start + fs]
        frm = vp(u.av_frame_alloc())
        C.c_int.from_address(frm.value + 112).value = len(blk)
        C.c_int.from_address(frm.value + 116).value = sfmt
        C.memmove(frm.value + chl_off, C.byref(lay), C.sizeof(lay))
        C.c_int.from_address(frm.value + rate_off).value = rate
        assert u.av_frame_get_buffer(frm, 0) == 0
        data = np.ascontiguousarray(blk, np.int16 if sfmt == AV_SAMPLE_FMT_S16 else np.int32)
        C.memmove(ffdecode._rd(frm.value, 0, vp), data.ctypes.data, data.nbytes)
        assert c.avcodec_send_frame(ctx, frm) == 0
        sizes.append(len(blk))
        drain()
        C.memset(frm.value + chl_off, 0, C.sizeof(lay))
        u.av_frame_free(C.byref(frm))
    c.avcodec_send_frame(ctx, None)
    drain()
    c.av_packet_free(C.byref(pkt))
    c.avcodec_free_context(C.byref(ctx))
    head = b"fLaC" + fw.streaminfo(fs if n >= fs else n, fs, rate, nch, bps, n)
    return head + b"".join(frames)


def ff_decode(data, rate, nch, as_query=False):
    with tempfile.TemporaryDirectory() as d:
        fn = os.path.join(d, "x.flac")
        with open(fn, "wb") as fh:
            fh.write(data)
        if as_query:
            return ffdecode.decode(fn)
        return ffdecode.decode(fn, rate, nch).reshape(-1)


def writer_cases():
    """The bit writer's files: (name, pcm, bps, rate, status, tests.flac_writer.stream keywords)."""
    cases = []

    def wadd(name, pcm, bps, rate, status=0, **kw):
        cases.append((name, pcm, bps, rate, status, kw))

    stereo = source(1, 2000, 2, 16)
    x = source(20, 4096, 1, 16)
    sizes = [1000, 37, 1500, 1, 900, 16, 642]
    wadd("w_variable", x, 16, 11025, sizes=sizes, variable=True,
         specs=lambda k: [{"kind": "verbatim"}] if sizes[k] < 4 else [{"order": k % 5, "po": 0}])
    e = x.copy()
    e[2048:3072] = 0
    wadd("w_escape", e, 16, 11025, specs=[{"po": 2, "escape": (0, 2), "method": 1}])
    taps = np.round(np.hanning(34)[1:-1] / np.hanning(34)[1:-1].sum() * 2048).astype(np.int64)
    wadd("w_lpc32", x, 16, 11025, specs=[{"kind": "lpc", "coefs": taps.tolist(), "prec": 12, "shift": 11, "po": 3}])
    wadd("w_codes_bs6_sr12", source(21, 2000, 1, 16), 16, 22000, sizes=[200] * 10, sr_code=12)
    wadd("w_codes_bs7_sr13", source(22, 3000, 1, 16), 16, 11025, sizes=[1000] * 3, sr_code=13)
    wadd("w_codes_sr14", source(23, 2000, 2, 16), 16, 44100, sizes=[1024, 976], sr_code=14, bs_code=lambda k: 7)
    for b in (4, 8, 12, 20, 24):
        wadd("w_depth%d" % b, source(30 + b, 2000, 1, b), b, 11025)
    ws = source(40, 2000, 2, 16) & ~3
    wadd("w_wasted_side", ws, 16, 11025, chmode=8, specs=[{"wasted": 2}, {"wasted": 2, "order": 1}])
    wadd("w_right_side", stereo, 16, 11025, chmode=9)
    wadd("w_mid_side", stereo, 16, 11025, chmode=10, specs=[{"kind": "lpc", "coefs": [3, -1], "prec": 4, "shift": 1},
                                                            {"order": 3}])
    wadd("w_id3", x[:3000], 16, 11025, id3=300)
    wadd("w_total0", x[:3000], 16, 11025, total=0)
    vc = b"\x04\x00\x00\x00test" + b"\x00\x00\x00\x00"
    blocks = (fw.block_header(1, 20, False) + bytes(20) + fw.block_header(3, 0, False) +
              fw.block_header(4, len(vc), False) + vc + fw.block_header(2, 8, True) + b"abcdtest")
    wadd("w_blocks", x[:3000], 16, 11025, blocks=blocks)
    # a sync pattern inside a frame: 8-bit VERBATIM samples are whole bytes of the frame, so frame 0's
    # samples spell the header frame 1 will carry (sync, codes, number 1, right CRC-8)
    hdr1 = fw.frame(np.zeros((1024, 1), np.int64), 1, 8, 11025)[:6]
    p8 = source(41, 3072, 1, 8)
    p8[500:506, 0] = np.frombuffer(hdr1, np.uint8).astype(np.int8)
    wadd("w_planted_sync", p8, 8, 11025, sizes=[1024] * 3, specs=[{"kind": "verbatim"}])
    # refused: a reserved subframe type in frames 1-2 (CRCs right), a 28-bit stream
    wadd("c_subframe_reserved", x[:3000], 16, 11025, status=4, sizes=[1024, 1024, 952],
         specs=lambda k: [{"sub_type": 2 if k else None}])
    wadd("c_depth28", source(42, 1000, 1, 28), 28, 11025, status=1)
    return cases


def main():
    out, names, decodes = {}, [], {}

    def add(name, data, pcm, bps, rate, status=0, keep_pcm=True):
        pcm = np.asarray(pcm, np.int64).reshape(len(pcm), -1)
        out[name + "/flac"] = np.frombuffer(data, np.uint8)
        out[name + "/meta"] = np.array([rate, pcm.shape[1], bps, status], np.int64)
        if status == 0:
            want = convert(pcm, bps).reshape(-1)
            got = ff_decode(data, rate, pcm.shape[1])
            assert np.array_equal(got, want), name
            if keep_pcm:
                # one copy of each distinct decode: the other files with the same PCM name its owner
                key = got.tobytes()
                if key in decodes:
                    out[name + "/pcm_of"] = np.array(decodes[key])
                else:
                    decodes[key] = name
                    out[name + "/pcm"] = got
            if pcm.shape[1] == 1 and rate == 11025 and bps != 16:
                out[name + "/source"] = pcm.reshape(-1).astype(np.int32)
                out[name + "/ffmpeg_s16"] = ff_decode(data, rate, 1, as_query=True)
        names.append(name)

    n = 2000
    # ---- FFmpeg's encoder
    stereo = source(1, n, 2, 16)
    for lvl in range(13):
        add("ff_level%d" % lvl, ff_encode(stereo, 11025, 16, level=lvl), stereo, 16, 11025)
    for m in ("indep", "left_side", "right_side", "mid_side"):
        add("ff_chmode_" + m, ff_encode(stereo, 44100, 16, opts={"ch_mode": m}), stereo, 16, 44100)
    for t in ("none", "fixed", "levinson", "cholesky"):
        add("ff_lpc_" + t, ff_encode(stereo, 11025, 16, opts={"lpc_type": t}), stereo, 16, 11025)
    x = source(2, 2000, 1, 16)
    add("ff_frame16", ff_encode(x, 11025, 16, frame_size=16), x, 16, 11025)
    # a 65535-sample frame needs that many samples: a sawtooth, which both encoders store in little space
    x = ((np.arange(66000, dtype=np.int64) * 7) % 1000 - 500).reshape(-1, 1)
    add("ff_frame65535", ff_encode(x, 11025, 16, frame_size=65535), x, 16, 11025)
    for nch in (1, 6, 8):
        x = source(3 + nch, 800, nch, 16)
        add("ff_ch%d" % nch, ff_encode(x, 48000, 16), x, 16, 48000)
    x24 = source(9, n, 1, 24)
    add("ff_s24_mono", ff_encode(x24, 11025, 24, level=8), x24, 24, 11025)
    x24s = source(10, n, 2, 24)
    add("ff_s24_stereo", ff_encode(x24s, 44100, 24), x24s, 24, 44100)
    z = source(0, 9000, 2, 16, "silence")
    add("ff_silence", ff_encode(z, 11025, 16), z, 16, 11025)
    nz = source(11, 3000, 1, 16, "noise")
    add("ff_noise", ff_encode(nz, 11025, 16), nz, 16, 11025)
    sh = source(12, 100, 1, 16)
    add("ff_short", ff_encode(sh, 11025, 16), sh, 16, 11025)
    # the bundled query (its PCM is in bundled.npz); the tests encode the bundled tracks with the bit writer
    gb = np.load(os.path.join(ROOT, "tests", "golden", "bundled.npz"))
    add("bundled_query", ff_encode(gb["query/pcm"], 11025, 16), gb["query/pcm"], 16, 11025, keep_pcm=False)

    # ---- the bit writer
    for name, pcm, bps, rate, status, kw in writer_cases():
        add(name, fw.stream(pcm, bps, rate, **kw)[0], pcm, bps, rate, status)

    # ---- damaged files
    x = source(20, 3072, 1, 16)
    good, lens = fw.stream(x, 16, 11025, sizes=[1024] * 3)
    f1 = len(good) - sum(lens) + lens[0]                   # frames 1 and 2 (the last) start here
    f2 = f1 + lens[1]
    bad = bytearray(good)
    bad[f1 + 60] ^= 0x10
    add("c_residual_bit", bytes(bad), x, 16, 11025, status=3)
    bad = bytearray(good)
    bad[f1 + 2] ^= 0x01                                    # sample-rate code 0 -> 1: the CRC-8 fails
    add("c_header_bit", bytes(bad), x, 16, 11025, status=2)
    add("c_truncated", good[:-10], x, 16, 11025, status=5)
    bad = bytearray(good)
    bad[f2 + 2] &= 0x0F                                    # block-size code 0 (reserved), CRC-8 made right
    hl = 6                                                 # header: 4 bytes, 1-byte number, CRC-8
    bad[f2 + hl - 1] = fw.crc8(bad[f2:f2 + hl - 1])
    add("c_reserved", bytes(bad), x, 16, 11025, status=4)

    out["names"] = np.array(names)
    out["writer_names"] = np.array([c[0] for c in writer_cases()])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(names), "files")


if __name__ == "__main__":
    main()
