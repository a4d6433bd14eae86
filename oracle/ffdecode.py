"""TEST INFRASTRUCTURE (golden generation only) - decode the reference's bundled
tests/data/*.mp3 the way the reference's own reader does.

The reference reads audio by piping `ffmpeg -i FILE -f s16le -ac 1 -ar 11025 -`
(audio_read.py:196-203, FFmpegAudioFile) and converting the int16 stream to
float32 / 32768 (audio_read.py:102-116, buf_to_float).  The image has no
`ffmpeg` executable, but the opencv-python-headless wheel vendors complete
FFmpeg 8.0 shared libraries (libavformat 62 / libavcodec 62 / libswresample 6,
mp3float decoder included).  This module drives those libraries through ctypes
with what the command line above makes `ffmpeg` do:

  demux (avformat) -> decode (avcodec, planar float) -> ONE libswresample
  context with library-default options converting rate, channel layout and
  sample format at once (what the auto-inserted `aresample` filter is) ->
  interleaved s16, flushed at end of stream.

Nothing of the product imports this file; it only produces the PCM that
oracle/make_golden_bundled.py feeds to the live reference, and the small PCM
fixtures the GPU parity tests read.  Struct fields are reached only where no
accessor exists; the offsets used are those of the FFmpeg 5.1-8.0 public
headers and are asserted against values known through accessors.
"""
from __future__ import annotations

import ctypes as C
import glob
import os

import numpy as np

AVMEDIA_TYPE_AUDIO = 1
AV_SAMPLE_FMT_S16 = 1
AVERROR_EOF = -541478725           # FFERRTAG('E','O','F',' ')
AVERROR_EAGAIN = -11


class AVRational(C.Structure):
    _fields_ = [("num", C.c_int), ("den", C.c_int)]


class AVChannelLayout(C.Structure):
    _fields_ = [("order", C.c_int), ("nb_channels", C.c_int), ("mask", C.c_uint64), ("opaque", C.c_void_p)]


_libs = None


def _load():
    global _libs
    if _libs is not None:
        return _libs
    import cv2  # noqa: F401  (maps the vendored libraries with their rpath)
    d = os.path.join(os.path.dirname(os.path.dirname(cv2.__file__)), "opencv_python_headless.libs")

    def lib(stem):
        hits = glob.glob(os.path.join(d, stem + "-*"))
        if not hits:
            raise RuntimeError("no vendored " + stem + " under " + d)
        return C.CDLL(hits[0], mode=C.RTLD_GLOBAL)
    u, s, c, f = lib("libavutil"), lib("libswresample"), lib("libavcodec"), lib("libavformat")
    vp, i, p = C.c_void_p, C.c_int, C.POINTER
    f.avformat_open_input.argtypes = [p(vp), C.c_char_p, vp, vp]
    f.avformat_find_stream_info.argtypes = [vp, vp]
    f.av_find_best_stream.argtypes = [vp, i, i, i, p(vp), i]
    f.av_read_frame.argtypes = [vp, vp]
    f.avformat_close_input.argtypes = [p(vp)]
    c.avcodec_alloc_context3.restype = vp
    c.avcodec_alloc_context3.argtypes = [vp]
    c.avcodec_parameters_to_context.argtypes = [vp, vp]
    c.avcodec_open2.argtypes = [vp, vp, vp]
    c.avcodec_send_packet.argtypes = [vp, vp]
    c.avcodec_receive_frame.argtypes = [vp, vp]
    c.avcodec_free_context.argtypes = [p(vp)]
    c.av_packet_alloc.restype = vp
    c.av_packet_unref.argtypes = [vp]
    c.av_packet_free.argtypes = [p(vp)]
    u.av_frame_alloc.restype = vp
    u.av_frame_unref.argtypes = [vp]
    u.av_frame_free.argtypes = [p(vp)]
    u.av_opt_set_q.argtypes = [vp, C.c_char_p, AVRational, i]
    u.av_opt_get_int.argtypes = [vp, C.c_char_p, i, p(C.c_int64)]
    u.av_get_sample_fmt_name.restype = C.c_char_p
    u.av_get_sample_fmt_name.argtypes = [i]
    u.av_opt_get_chlayout.argtypes = [vp, C.c_char_p, i, p(AVChannelLayout)]
    u.av_channel_layout_default.argtypes = [p(AVChannelLayout), i]
    u.av_sample_fmt_is_planar.argtypes = [i]
    s.swr_alloc_set_opts2.argtypes = [p(vp), p(AVChannelLayout), i, i, p(AVChannelLayout), i, i, i, vp]
    s.swr_init.argtypes = [vp]
    s.swr_convert.argtypes = [vp, p(vp), i, p(vp), i]
    s.swr_get_out_samples.argtypes = [vp, i]
    s.swr_free.argtypes = [p(vp)]
    _libs = (u, s, c, f)
    return _libs


def _rd(ptr, off, ctype):
    return ctype.from_address(ptr + off).value


def decode(path: str, sr: int = 11025, channels: int = 1) -> np.ndarray:
    """int16 PCM, shape (n,) for channels == 1 else (n, channels): the byte
    stream `ffmpeg -i path -f s16le -ac channels -ar sr -` writes."""
    u, s, c, f = _load()
    fmt = C.c_void_p()
    if f.avformat_open_input(C.byref(fmt), os.fsencode(path), None, None) < 0:
        raise IOError("avformat_open_input failed: " + path)
    ctx = C.c_void_p()
    swr = C.c_void_p()
    pkt = C.c_void_p(c.av_packet_alloc())
    frm = C.c_void_p(u.av_frame_alloc())
    out = []
    try:
        if f.avformat_find_stream_info(fmt, None) < 0:
            raise IOError("no stream info: " + path)
        dec = C.c_void_p()
        idx = f.av_find_best_stream(fmt, AVMEDIA_TYPE_AUDIO, -1, -1, C.byref(dec), 0)
        if idx < 0:
            raise IOError("no audio stream: " + path)
        # AVFormatContext.streams (offset 48 after 5 pointers + ctx_flags + nb_streams);
        # AVStream {av_class, index, id, codecpar, priv_data, time_base}
        nb_streams = _rd(fmt.value, 44, C.c_uint)
        assert 0 <= idx < nb_streams <= 64, "AVFormatContext layout"
        streams = _rd(fmt.value, 48, C.c_void_p)
        st = _rd(streams, 8 * idx, C.c_void_p)
        assert _rd(st, 8, C.c_int) == idx, "AVStream layout"
        codecpar = _rd(st, 16, C.c_void_p)
        tb = AVRational.from_address(st + 32)
        assert tb.num > 0 and tb.den > 0, "AVStream.time_base"
        ctx = C.c_void_p(c.avcodec_alloc_context3(dec))
        if c.avcodec_parameters_to_context(ctx, codecpar) < 0:
            raise IOError("avcodec_parameters_to_context")
        # ffmpeg sets pkt_timebase so that the demuxer's skip-samples side data
        # (encoder delay of the MP3) is applied by the decoder
        u.av_opt_set_q(ctx, b"pkt_timebase", AVRational(tb.num, tb.den), 0)
        if c.avcodec_open2(ctx, dec, None) < 0:
            raise IOError("avcodec_open2")

        def setup_swr():
            rate = C.c_int64()
            lay = AVChannelLayout()
            assert u.av_opt_get_int(ctx, b"ar", 0, C.byref(rate)) >= 0
            assert u.av_opt_get_chlayout(ctx, b"ch_layout", 0, C.byref(lay)) >= 0
            # the sample format has no option accessor: take it from the first frame
            # (AVFrame.format, offset 116) and check it names a real format
            sfmt = C.c_int(_rd(frm.value, 116, C.c_int))
            assert u.av_get_sample_fmt_name(sfmt.value), "AVFrame.format"
            olay = AVChannelLayout()
            u.av_channel_layout_default(C.byref(olay), channels)
            if s.swr_alloc_set_opts2(C.byref(swr), C.byref(olay), AV_SAMPLE_FMT_S16, sr,
                                     C.byref(lay), sfmt.value, int(rate.value), 0, None) < 0:
                raise IOError("swr_alloc_set_opts2")
            if s.swr_init(swr) < 0:
                raise IOError("swr_init")
            return sfmt.value, lay.nb_channels, int(rate.value)

        info = None

        def pull(in_ptrs, n_in):
            cap = s.swr_get_out_samples(swr, n_in) + 64
            buf = np.empty((cap, channels), np.int16)
            op = (C.c_void_p * 1)(buf.ctypes.data)
            n = s.swr_convert(swr, op, cap, in_ptrs, n_in)
            if n < 0:
                raise IOError("swr_convert")
            if n:
                out.append(buf[:n].copy())

        def drain_decoder():
            nonlocal info
            while True:
                r = c.avcodec_receive_frame(ctx, frm)
                if r in (AVERROR_EAGAIN, AVERROR_EOF):
                    return r
                if r < 0:
                    raise IOError("avcodec_receive_frame %d" % r)
                if info is None:
                    info = setup_swr()
                # AVFrame {data[8], linesize[8], extended_data, width, height, nb_samples, format}
                nb = _rd(frm.value, 112, C.c_int)
                assert _rd(frm.value, 116, C.c_int) == info[0] and 0 < nb <= 1 << 16, "AVFrame layout"
                ext = _rd(frm.value, 96, C.c_void_p)
                planes = info[1] if u.av_sample_fmt_is_planar(info[0]) else 1
                ip = (C.c_void_p * max(planes, 1))(*[_rd(ext, 8 * k, C.c_void_p) for k in range(planes)])
                pull(ip, nb)
                u.av_frame_unref(frm)

        while f.av_read_frame(fmt, pkt) >= 0:
            # AVPacket {buf, pts, dts, data, size, stream_index}
            if _rd(pkt.value, 36, C.c_int) == idx:
                r = c.avcodec_send_packet(ctx, pkt)
                if r < 0 and r != AVERROR_EAGAIN:
                    c.av_packet_unref(pkt)
                    continue            # ffmpeg logs the error and goes on
                drain_decoder()
            c.av_packet_unref(pkt)
        c.avcodec_send_packet(ctx, None)
        drain_decoder()
        if swr:
            pull(None, 0)               # flush the resampler tail
    finally:
        if swr:
            s.swr_free(C.byref(swr))
        if ctx:
            c.avcodec_free_context(C.byref(ctx))
        c.av_packet_free(C.byref(pkt))
        u.av_frame_free(C.byref(frm))
        f.avformat_close_input(C.byref(fmt))
    pcm = np.concatenate(out) if out else np.zeros((0, channels), np.int16)
    return pcm[:, 0].copy() if channels == 1 else pcm


def audio_read(filename, sr=None, channels=None):
    """Signature of the reference's audio_read.audio_read (audio_read.py:56-99):
    float32 in [-1, 1) and the sampling rate."""
    pcm = decode(filename, sr or 11025, channels or 1)
    return (pcm.astype(np.float32) / 32768.0), (sr or 11025)


if __name__ == "__main__":
    import sys
    for pth in sys.argv[1:]:
        x = decode(pth)
        print(pth, x.shape, x.dtype, int(np.abs(x).max()) if len(x) else 0, "%.2f s" % (len(x) / 11025.0))
