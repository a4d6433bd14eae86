"""Analyzer — drop-in mirror of audfprint_analyze.Analyzer whose arithmetic
runs in libafp.so (sm_90a CUDA) through the C ABI of include/afp.h.

Same attribute names, method names, argument meaning and error behaviour as the
reference class (audfprint_analyze.py:115-457); the module-level helpers
landmarks2hashes / hashes2landmarks and the .afpt/.afpk codecs (:81-112,
:460-514) are provided too.  Host code here is bookkeeping only: parameter
tables, buffer packing, result unpacking.  Nothing in this file computes a
spectrogram, a peak or a hash on the CPU.
"""
from __future__ import annotations

import ctypes as C
import os
import struct
import time
import wave

import numpy as np

from . import _lib, flac

# Special extensions of precomputed files (audfprint_analyze.py:29-32)
PRECOMPEXT = '.afpt'
PRECOMPPKEXT = '.afpk'

DENSITY = 20.0
OVERSAMP = 1
N_FFT = 512
N_HOP = 256
HPF_POLE = 0.98

# hash layout (audfprint_analyze.py:69-78): bin1 in 8 bits, signed bin difference in 6, frame gap in 6
F1_BITS, DF_BITS, DT_BITS = 8, 6, 6
B1_SHIFT, DF_SHIFT = DF_BITS + DT_BITS, DT_BITS
B1_MASK, DF_MASK, DT_MASK = (1 << F1_BITS) - 1, (1 << DF_BITS) - 1, (1 << DT_BITS) - 1


def landmarks2hashes(landmarks):
    """(time, bin1, bin2, dtime) rows -> int32 (L,2) [time, hash]
    (audfprint_analyze.py:81-96).  Pure bit packing of values the device
    produced; kept on the host for API parity (<1 % of the reference's time)."""
    lm = np.asarray(landmarks, dtype=np.int64).reshape(-1, 4)
    t, f1, f2, dt = lm[:, 0], lm[:, 1], lm[:, 2], lm[:, 3]
    packed = ((f1 & B1_MASK) << B1_SHIFT) | (((f2 - f1) & DF_MASK) << DF_SHIFT) | (dt & DT_MASK)
    return np.stack([t, packed], axis=1).astype(np.int32)


def hashes2landmarks(hashes):
    """Inverse of landmarks2hashes (audfprint_analyze.py:99-112): list of
    (time, bin1, bin2, dtime) tuples."""
    h = np.asarray(hashes, dtype=np.int64).reshape(-1, 2)
    word = h[:, 1]
    f1 = (word >> B1_SHIFT) & B1_MASK
    df = (word >> DF_SHIFT) & DF_MASK
    df = df - ((df >> (DF_BITS - 1)) << DF_BITS)          # sign-extend the 6-bit difference
    return list(zip(h[:, 0].tolist(), f1.tolist(), (f1 + df).tolist(), (word & DT_MASK).tolist()))


def resample_taps(up, down):
    """The low-pass scipy.signal.resample_poly designs for (up, down) (window ('kaiser', 5.0),
    half length 10 * max(up, down), cut-off 1 / max(up, down), scaled by `up`): float64 (2*half+1,)."""
    from scipy.signal import firwin
    max_rate = max(up, down)
    half = 10 * max_rate
    return np.ascontiguousarray(firwin(2 * half + 1, 1.0 / max_rate, window=('kaiser', 5.0)) * up, dtype=np.float64)


# sample formats of the front-ends (afp.h AFP_PCM_*), by name
SAMPLE_FORMATS = {'s16': _lib.PCM_I16, 's24': _lib.PCM_S24, 's32': _lib.PCM_S32, 'f32': _lib.PCM_F32}
_WIDTH = {_lib.PCM_I16: 2, _lib.PCM_S24: 3, _lib.PCM_S32: 4, _lib.PCM_F32: 4}


def _as_payload(raw, sample_format):
    """One file's samples -> (payload bytes as uint8, AFP_PCM_* code).  sample_format None: int16 as
    pcm_frontend has always taken it (values converted to int16).  Otherwise 's16', 's24', 's32' or 'f32':
    `raw` holds the data chunk's little-endian bytes, in any array type (a 24-bit file as uint8 bytes)."""
    if sample_format is None:
        return np.ascontiguousarray(raw, dtype=np.int16).reshape(-1).view(np.uint8), _lib.PCM_I16
    if sample_format not in SAMPLE_FORMATS:
        raise ValueError("sample_format must be one of %s" % ", ".join(sorted(SAMPLE_FORMATS)))
    code = SAMPLE_FORMATS[sample_format]
    b = np.ascontiguousarray(raw).reshape(-1).view(np.uint8)
    return b[:len(b) // _WIDTH[code] * _WIDTH[code]], code


def pcm_frontend(raw, channels, src_rate, dst_rate=None, device=None, to_host=True, resampler='poly',
                 sample_format=None):
    """Interleaved int16 PCM -> mono float32 at dst_rate, on the device: pcm_frontend_batch of one file
    (channel mean, 1/32768 scaling, polyphase resampling).  Returns a NumPy array, or with
    to_host=False a torch CUDA tensor that Analyzer.fingerprint_packed takes as it is.
    resampler='ffmpeg' gives instead the bits `ffmpeg -ac 1 -ar dst_rate` gives, v / 32768
    (mono or stereo, and rates with out / gcd <= 1024).
    sample_format 's24', 's32' or 'f32' (or 's16') takes `raw` as a WAV data chunk's bytes of that
    format (_as_payload)."""
    out, _, lens = pcm_frontend_batch([raw], [channels], [src_rate], src_rate if dst_rate is None else dst_rate,
                                      device=device, resampler=resampler, sample_formats=[sample_format])
    out = out[:int(lens[0])]
    return out.cpu().numpy() if to_host else out


_GUID_TAIL = b"\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"      # KSDATAFORMAT_SUBTYPE_* after Data1
_WAVE_PCM, _WAVE_FLOAT, _WAVE_EXTENSIBLE = 1, 3, 0xFFFE


def _wav_format(fmt):
    """A fmt chunk -> (AFP_PCM_* code, channels, rate).  Raises for the codings the front-ends do not
    take, with the message the wave module gave them: 8-bit PCM, 64-bit float, A-law, mu-law, ADPCM..."""
    if len(fmt) < 16:
        raise EOFError
    tag, nch, fs, _, _, bits = struct.unpack_from('<HHIIHH', fmt)
    sub = tag
    if tag == _WAVE_EXTENSIBLE:
        if len(fmt) < 40:
            raise EOFError
        guid = fmt[24:40]
        sub = int.from_bytes(guid[:4], 'little') if guid[4:] == _GUID_TAIL else None
        if sub not in (_WAVE_PCM, _WAVE_FLOAT) or (sub == _WAVE_FLOAT and bits != 32):
            import uuid
            raise wave.Error('unknown extended format: %s' % uuid.UUID(bytes_le=guid))
        valid = struct.unpack_from('<H', fmt, 18)[0]
        if sub == _WAVE_PCM and bits == 32 and 0 < valid < 32:
            # ffmpeg reads such a file as packed 24-bit samples, which it is not
            raise IOError("32-bit PCM WAV with %d valid bits is not supported" % valid)
    elif tag not in (_WAVE_PCM, _WAVE_FLOAT) or (tag == _WAVE_FLOAT and bits != 32):
        raise wave.Error('unknown format: %r' % (tag,))
    width = (bits + 7) // 8
    if not width:
        raise wave.Error('bad sample width')
    if not nch:
        raise wave.Error('bad # of channels')
    if sub == _WAVE_FLOAT:
        return _lib.PCM_F32, nch, fs
    if width not in (2, 3, 4):
        raise IOError("only 16-bit PCM WAV is supported, got %d-byte samples" % width)
    return {2: _lib.PCM_I16, 3: _lib.PCM_S24, 4: _lib.PCM_S32}[width], nch, fs


def _wav_parse(filename):
    """Walk a RIFF WAVE file's chunks (padded to even sizes; unknown ones skipped) to its fmt and data
    chunks -> (payload uint8, AFP_PCM_* code, channels, rate): the data chunk's bytes as they are, cut to
    the whole frames present (a data size past the end of the file reads to the end).  Samples are not
    converted: 16-bit, 24-bit and 32-bit PCM and 32-bit float, plain or WAVE_FORMAT_EXTENSIBLE.  Raises
    for other files, with the wave module's messages."""
    with open(filename, 'rb') as f:
        data = f.read()
    if len(data) < 8:
        raise EOFError
    if data[:4] != b'RIFF':
        raise wave.Error('file does not start with RIFF id')
    if data[8:12] != b'WAVE':
        raise wave.Error('not a WAVE file')
    pos, form = 12, None
    while pos + 8 <= len(data):
        cid, size = data[pos:pos + 4], int.from_bytes(data[pos + 4:pos + 8], 'little')
        body = data[pos + 8:pos + 8 + size]
        if cid == b'fmt ':
            form = _wav_format(body)
        elif cid == b'data':
            if form is None:
                raise wave.Error('data chunk before fmt chunk')
            code, nch, fs = form
            frame = _WIDTH[code] * nch
            payload = np.frombuffer(body, np.uint8)
            return payload[:len(payload) // frame * frame], code, nch, fs
        pos += 8 + size + (size & 1)
    raise wave.Error('fmt chunk and/or data chunk missing')


def _wav_read_raw(filename):
    """The host half of _wav_reader: parse a WAV (_wav_parse) -> (interleaved samples, channels, rate).
    The samples are the payload's bytes as they are, typed by format: int16, int32 or float32 arrays, a
    24-bit file as uint8 (n, 3).  Raises what _wav_reader raises for a file it cannot read."""
    payload, code, nch, fs = _wav_parse(filename)
    if code == _lib.PCM_S24:
        return payload.reshape(-1, 3), nch, fs
    return payload.view({_lib.PCM_I16: '<i2', _lib.PCM_S32: '<i4', _lib.PCM_F32: '<f4'}[code]), nch, fs


def _raw_format(raw):
    """The sample_format name of an array _wav_read_raw returns."""
    if raw.dtype == np.uint8:
        return 's24'
    return {np.dtype('<i2'): 's16', np.dtype('<i4'): 's32', np.dtype('<f4'): 'f32'}[raw.dtype]


def _audio_read_raw(filename):
    """The host half of the default reader, by content rather than extension: a native FLAC stream
    (after optional ID3v2 tags) -> (flac.FlacStream, channels, rate); anything else goes to
    _wav_read_raw, which reads a RIFF WAV or raises what it raises for other files."""
    with open(filename, 'rb') as f:
        head = f.read(10)
        if head[:3] == b'ID3' or head[:4] == flac.MAGIC:
            data = head + f.read()
            if flac.is_flac(data):
                stream = flac.parse(data)
                return stream, stream.channels, stream.sample_rate
    return _wav_read_raw(filename)


def _check_resampler(resampler):
    if resampler not in ('poly', 'ffmpeg'):
        raise ValueError("resampler must be 'poly' or 'ffmpeg'")
    return resampler


def swr_length(nframes, src_rate, dst_rate):
    """Samples the 'ffmpeg' front-end (afp_swr_frontend_batch) yields for nframes input frames (host
    arithmetic, no device).  Raises AfpError for a rate the front-end refuses."""
    n = C.c_int64(0)
    rc = _lib.load().afp_swr_length(int(nframes), int(src_rate), int(dst_rate), C.byref(n))
    if rc == -3:
        raise _lib.AfpError("the ffmpeg front-end does not take %d Hz -> %d Hz" % (src_rate, dst_rate))
    if rc:
        raise ValueError("afp_swr_length: %d frames, %d Hz -> %d Hz" % (nframes, src_rate, dst_rate))
    return int(n.value)


# the channel masks ffmpeg gives a WAV that names none: FC for mono, FL|FR for stereo
_DEFAULT_WAV_MASKS = {1: 0x4, 2: 0x3}


def _wav_channel_mask(filename):
    """dwChannelMask of a WAVE_FORMAT_EXTENSIBLE file, or None for any other WAV."""
    with open(filename, 'rb') as f:
        if f.read(12)[8:12] != b'WAVE':
            return None
        while True:
            head = f.read(8)
            if len(head) < 8:
                return None
            cid, size = head[:4], int.from_bytes(head[4:], 'little')
            if cid == b'fmt ':
                fmt = f.read(size)
                if size >= 24 and int.from_bytes(fmt[:2], 'little') == 0xFFFE:
                    return int.from_bytes(fmt[20:24], 'little')
                return None
            f.seek(size + (size & 1), 1)


def _swr_check(filename, raw, nch, fs, sr):
    """Raise for a file the 'ffmpeg' front-end cannot give ffmpeg's bits for: more than two channels,
    a WAV whose channel mask is not the default layout, or a rate afp_swr_frontend_batch refuses."""
    if nch > 2:
        raise ValueError("%s: the ffmpeg front-end takes mono or stereo, not %d channels" % (filename, nch))
    if isinstance(raw, np.ndarray) and _wav_channel_mask(filename) not in (None, 0, _DEFAULT_WAV_MASKS[nch]):
        raise ValueError("%s: the ffmpeg front-end takes only the default channel layout" % filename)
    swr_length(0, fs, sr)


def _wav_reader(filename, sr=None, channels=None, device=None, resampler='poly'):
    """PCM-WAV and FLAC reader standing in for audio_read.audio_read (audio_read.py:56-68; ffmpeg
    decoding of other formats is out of scope, SURVEY §2 #9).  Returns (float32 samples in [-1,1), sr)
    like the reference reader does (audio_read.py:139-145).  A WAV is parsed on the host; a FLAC file's
    frames are decoded on the device to the samples ffmpeg's decoder gives.  The arithmetic the
    reference hands to ffmpeg - down-mix to mono, resampling to `sr` - runs on the device
    (_frontend_sources, SURVEY.md 8f-2).  No two resamplers agree bit for bit, so parity statements in
    this repo are made on 11025 Hz PCM.  With resampler='ffmpeg' the down-mix and resampling are
    ffmpeg's own, bit for bit (afp_swr_frontend_batch_bytes)."""
    raw, nch, fs = _audio_read_raw(filename)
    sr = fs if sr is None else sr
    if _check_resampler(resampler) == 'ffmpeg':
        _swr_check(filename, raw, nch, fs, sr)
    if isinstance(raw, np.ndarray) and raw.dtype == np.int16 and nch == 1 and fs == sr:
        # nothing to do but the reader's own scaling (exact in float32, the bits the device gives)
        return raw.astype(np.float32) * np.float32(1.0 / 32768.0), fs
    out, _, lens, status = _frontend_sources([raw], [nch], [fs], sr, device, resampler)
    if status[0]:
        raise flac.failure(status[0])
    return out[:int(lens[0])].cpu().numpy(), sr


_TAPS = {}


def taps_table(pairs):
    """The designs of the distinct resampling pairs among `pairs` ((up, down) per file; (1, 1) needs
    none), in order of first appearance -> (pair_rates int32 (P,2), tap_offsets int64 (P+1,),
    taps float64): what afp_pcm_frontend_batch takes.  Each design is resample_taps(up, down),
    computed once per process."""
    uniq = []
    for ud in pairs:
        ud = (int(ud[0]), int(ud[1]))
        if ud != (1, 1) and ud not in uniq:
            uniq.append(ud)
    designs = []
    for ud in uniq:
        if ud not in _TAPS:
            _TAPS[ud] = resample_taps(*ud)
        designs.append(_TAPS[ud])
    off = np.zeros(len(uniq) + 1, np.int64)
    off[1:] = np.cumsum([len(t) for t in designs])
    taps = np.ascontiguousarray(np.concatenate(designs)) if designs else np.zeros(1, np.float64)
    return np.array(uniq, np.int32).reshape(-1, 2), off, taps


def pcm_frontend_batch(raws, channels, src_rates, dst_rate, device=None, resampler='poly', sample_formats=None):
    """Many files' interleaved int16 PCM -> mono float32 at dst_rate in ONE device buffer
    (_frontend_packed: one upload of the packed payloads, one launch, one synchronise).
    Returns (out torch CUDA float32, offsets int64 [n+1], lengths int64 [n]): file i is
    out[offsets[i]:offsets[i] + lengths[i]], starting on a 16-byte boundary - the layout
    Analyzer.fingerprint_packed(out, offsets, sample_lengths=lengths) takes as it is.
    resampler='ffmpeg': ffmpeg's down-mix and resampler (pcm_frontend).
    sample_formats: None (every file int16, values converted as pcm_frontend converts them), or one
    pcm_frontend sample_format per file; files of every format share the one call."""
    if sample_formats is None:
        sample_formats = [None] * len(raws)
    pays, fmts, nfr = _payloads(raws, sample_formats, channels)
    packed, boff = _pack_payloads(pays)
    return _frontend_packed(_lib.context(device), packed, boff, nfr, channels, src_rates, dst_rate, resampler, fmts)


def _payloads(raws, sample_formats, channels):
    """Files' samples -> (payload bytes, AFP_PCM_* codes, frames) per file (_as_payload)."""
    pays = [_as_payload(r, f) for r, f in zip(raws, sample_formats)]
    nfr = [len(b) // _WIDTH[k] // max(1, int(c)) for (b, k), c in zip(pays, channels)]
    return [b for b, _ in pays], [k for _, k in pays], nfr


def _pack_payloads(payloads, extra=()):
    """Payload bytes of many files -> (one uint8 buffer, byte offset int64 [n]), every file on a 4-byte
    boundary; `extra` byte counts get aligned places after them (filled by the caller)."""
    if len(payloads) == 1 and not extra:          # nothing to align: the bytes go up as they are, uncopied
        return payloads[0], np.array([0, len(payloads[0])], np.int64)
    sizes = [len(b) for b in payloads] + list(extra)
    boff = np.zeros(len(sizes) + 1, np.int64)
    boff[1:] = np.cumsum([(n + 3) // 4 * 4 for n in sizes])
    packed = np.zeros(int(boff[-1]), np.uint8)
    for b, o in zip(payloads, boff):
        packed[o:o + len(b)] = b
    return packed, boff


def _frontend_packed(ctx, pcm, inoff, nfr, channels, src_rates, dst_rate, resampler='poly', formats=None):
    """The byte-form front-end (afp_pcm_frontend_batch_bytes, or afp_swr_frontend_batch_bytes for
    'ffmpeg') over files packed in `pcm`, a host uint8 array or device uint8 tensor: file i's nfr[i]
    frames of channels[i] channels, AFP_PCM_* formats[i], start at byte inoff[i].  formats None: `pcm`
    is a host int16 array or device int16 tensor, `inoff` counts int16 values, and every file is
    AFP_PCM_I16.  -> (out, offsets, lengths) as pcm_frontend_batch returns them."""
    import torch
    from math import gcd
    n = len(nfr)
    inoff = np.ascontiguousarray(inoff, dtype=np.int64)
    if formats is None:
        pcm = pcm.view(np.uint8) if isinstance(pcm, np.ndarray) else pcm.view(torch.uint8)
        inoff, formats = 2 * inoff, np.full(n, _lib.PCM_I16, np.int32)
    fmt = np.ascontiguousarray(formats, dtype=np.int32)
    ch = np.array([int(c) for c in channels], np.int32)
    nfr = np.ascontiguousarray(nfr, dtype=np.int64)
    P = C.POINTER(C.c_int64)
    ptr, on_host = _lib.ptr_of(pcm)
    plen = len(pcm) if isinstance(pcm, np.ndarray) else pcm.numel()
    if _check_resampler(resampler) == 'ffmpeg':
        rates = np.array([int(fs) for fs in src_rates], np.int32)
        fn, own = ctx.lib.afp_swr_frontend_batch_bytes, [rates.ctypes.data, int(dst_rate)]
    else:
        up, down = np.ones(n, np.int32), np.ones(n, np.int32)
        for i, fs in enumerate(src_rates):
            if dst_rate is not None and int(dst_rate) != int(fs):
                g = gcd(int(dst_rate), int(fs))
                up[i], down[i] = int(dst_rate) // g, int(fs) // g
        rates, toff, taps = taps_table(zip(up, down))
        fn, own = ctx.lib.afp_pcm_frontend_batch_bytes, [up.ctypes.data, down.ctypes.data, len(rates),
                                                         rates.ctypes.data, toff.ctypes.data_as(P), taps.ctypes.data]
    args = [ctx.h, ptr if plen else None, on_host, plen, n, inoff.ctypes.data_as(P), fmt.ctypes.data,
            nfr.ctypes.data_as(P), ch.ctypes.data] + own
    off, lens = np.zeros(n + 1, np.int64), np.zeros(n, np.int64)
    ctx.check(fn(*args, None, 0, off.ctypes.data_as(P), lens.ctypes.data_as(P)))
    # 16 bytes of zeros past the last file, as Analyzer._pack leaves
    out = torch.zeros(int(off[-1]) + 4, dtype=torch.float32, device=torch.device("cuda", ctx.device))
    with ctx.after_torch(out, pcm):       # the zeros (and a device pcm) land before the library's stream
        ctx.check(fn(*args, out.data_ptr(), out.numel(), None, None))
    return out, off, lens


def _flac_format(stream, resampler):
    """The AFP_PCM_* format a FLAC file is decoded to for `resampler`: int16, or for 17-24 bits in
    'ffmpeg' mode the full-depth int32 ffmpeg's decoder gives (flac.decode_into_bytes)."""
    return _lib.PCM_S32 if resampler == 'ffmpeg' and stream.bits_per_sample > 16 else _lib.PCM_I16


def _frontend_sources(sources, channels, src_rates, dst_rate, device=None, resampler='poly'):
    """The front-end over files given as WAV samples (what _wav_read_raw returns, or int16 PCM) or as
    flac.FlacStream.  Without FLAC files: pcm_frontend_batch of the WAV payloads, each in its own
    format (_raw_format).  With them, the round's buffer is built on the device: the WAV payloads go up
    in one copy, the FLAC files are located (one call) and decoded into their places after them (one
    call; _flac_format), and one front-end call runs over all (_frontend_packed).
    -> (out, offsets, lengths, status int32 [n]): 0, or the AFP_FLAC_* code of a FLAC file the device
    refused, which then has no samples."""
    n = len(sources)
    status = np.zeros(n, np.int32)
    fl = [k for k, s in enumerate(sources) if isinstance(s, flac.FlacStream)]
    if not fl:
        return pcm_frontend_batch(sources, channels, src_rates, dst_rate, device=device, resampler=resampler,
                                  sample_formats=[_raw_format(s) for s in sources]) + (status,)
    import torch
    ctx = _lib.context(device)
    wav = [k for k, s in enumerate(sources) if not isinstance(s, flac.FlacStream)]
    fmts, nfr = np.zeros(n, np.int32), np.zeros(n, np.int64)
    pays, fmts[wav], nfr[wav] = _payloads([sources[k] for k in wav], [_raw_format(sources[k]) for k in wav],
                                          [channels[k] for k in wav])
    nsamples = flac.locate(ctx, [sources[k] for k in fl])[0]
    for j, k in enumerate(fl):
        fmts[k], nfr[k] = _flac_format(sources[k], resampler), nsamples[j]
    packed, boff = _pack_payloads(pays, [int(nfr[k]) * int(channels[k]) * _WIDTH[int(fmts[k])] for k in fl])
    inoff = np.zeros(n, np.int64)
    inoff[wav] = boff[:len(wav)]
    inoff[fl] = boff[len(wav):n]
    pcm = torch.empty(max(len(packed), 1), dtype=torch.uint8, device=torch.device("cuda", ctx.device))
    wav_len = int(boff[len(wav)])
    if wav_len:
        pcm[:wav_len].copy_(torch.from_numpy(packed[:wav_len]))
    with ctx.after_torch(pcm):            # the payload copy lands before the decode writes after it
        status[fl] = flac.decode_into_bytes(ctx, pcm, inoff[fl], resampler == 'ffmpeg')
    nfr[status != 0] = 0
    return _frontend_packed(ctx, pcm, inoff, nfr, channels, src_rates, dst_rate, resampler, fmts) + (status,)


class _ChunkPlanner(object):
    """Greedy chunking in list order: a chunk grows while its frames stay within max_frames and its
    bytes within max_bytes; a file over either cap goes alone."""

    def __init__(self, max_frames, max_bytes):
        self.max_frames, self.max_bytes = max_frames, max_bytes
        self.n = self.frames = self.nbytes = 0

    def add(self, frames, nbytes):
        """Account one more file; True when it has to start a new chunk (the open one is full)."""
        new = self.n > 0 and (self.frames + frames > self.max_frames or self.nbytes + nbytes > self.max_bytes)
        if new:
            self.n = self.frames = self.nbytes = 0
        self.n += 1
        self.frames += frames
        self.nbytes += nbytes
        return new


def plan_chunks(frames, nbytes, max_frames, max_bytes):
    """[start, end) of the chunks _ChunkPlanner makes of a list (what wavfiles2hashes does while it
    reads): where a chunk ends depends only on the files before it."""
    planner, out, start = _ChunkPlanner(max_frames, max_bytes), [], 0
    for i, (f, b) in enumerate(zip(frames, nbytes)):
        if planner.add(f, b):
            out.append((start, i))
            start = i
    if len(frames) > start:
        out.append((start, len(frames)))
    return out


def _peak_rows(peaks):
    """A peak list ((col, bin) pairs) -> contiguous int32 (n, 2)."""
    return np.ascontiguousarray(np.asarray(peaks, dtype=np.int32).reshape(-1, 2))


def precompute_name(filename, precompdir, hashes_not_peaks=True, strip_prefix=None):
    """Output file of `precompute` for `filename` (audfprint.py:76-93): `strip_prefix` removed when
    the name starts with it, '.', '..' and empty components dropped (so absolute and relative names
    land inside `precompdir`), the extension replaced by .afpt (hashes) or .afpk (peaks)."""
    if strip_prefix and filename[:len(strip_prefix)] == strip_prefix:
        tail = filename[len(strip_prefix):]
    else:
        tail = filename
    relname = '/'.join([comp for comp in tail.split('/') if comp not in ('.', '..', '')])
    return os.path.join(precompdir, os.path.splitext(relname)[0] + (PRECOMPEXT if hashes_not_peaks else PRECOMPPKEXT))


def _ensure_dir(dirname):
    """Create `dirname` if it is missing (audfprint.py:55-60, failures ignored as there)."""
    if not os.path.exists(dirname):
        try:
            os.makedirs(dirname)
        except OSError:
            pass


def _precompute_write(filename, opfname, hashes_not_peaks, output, dur):
    """Write one precompute result as the reference's saver does (magic, then int32 pairs) and return
    its message (audfprint.py:105-115)."""
    if len(output) == 0:
        return "Zero length analysis for " + filename + " -- not saving."
    _ensure_dir(os.path.split(opfname)[0])
    with open(opfname, 'wb') as f:
        f.write(HASH_MAGIC if hashes_not_peaks else PEAK_MAGIC)
        np.ascontiguousarray(np.asarray(output, dtype='<i4').reshape(-1, 2)).tofile(f)
    return "wrote " + opfname + " ( %d %s, %.3f sec)" % (len(output), "hashes" if hashes_not_peaks else "peaks", dur)


def next_precompute_round(opnames, start, skip_existing, exists, max_files):
    """The precompute round that starts at file `start` of a list whose output names are `opnames`
    -> (end, skipped): files [start, end) are analysed together, those in `skipped` are not.

    The round gives what the per-file loop gives as long as every existence check sees the disk the
    loop would see.  Outputs are written in list order after the round, so with skip_existing a file
    whose output name an earlier file of the same round has closes the round before it: the earlier
    file writes (or, with an empty analysis, does not) before the later one is checked.  Without
    skip_existing a later file of the same name simply overwrites the earlier one's output.
    `exists(name)` is the check (os.path.isfile)."""
    seen, skipped = set(), []
    i = start
    while i < len(opnames) and i - start < max_files:
        name = opnames[i]
        if skip_existing:
            if name in seen:
                break
            if exists(name):
                skipped.append(i)
            seen.add(name)
        i += 1
    return i, skipped


class DeviceHashes(object):
    """One file's hashes left on the device by Analyzer._hashes_of_files(rows_on_device=True):
    `rows` is a torch CUDA int32 (n, 2) view, `last_time` the time of its last row (np.int32)."""
    __slots__ = ("rows", "last_time")

    def __init__(self, rows, last_time):
        self.rows, self.last_time = rows, last_time

    def __len__(self):
        return int(self.rows.shape[0])


def _as_pcm(d):
    """Normalise one signal to a contiguous int16 or float32 1-D array."""
    a = np.asarray(d)
    if a.ndim != 1:
        raise ValueError("signal must be 1-D")
    if a.dtype == np.int16:
        return np.ascontiguousarray(a), _lib.PCM_I16
    if a.dtype != np.float32:
        # the reference reader yields float32 (audio_read.py:145); wider input is narrowed
        a = a.astype(np.float32)
    return np.ascontiguousarray(a), _lib.PCM_F32


class Analyzer(object):
    """Parameters + methods of the reference Analyzer (audfprint_analyze.py:115-151)."""

    # attribute -> default, as set by audfprint_analyze.py:118-147
    _REFERENCE_DEFAULTS = dict(target_sr=11025, n_fft=N_FFT, n_hop=N_HOP, shifts=1, f_sd=30.0,
                               maxpksperframe=5, maxpairsperpeak=3, targetdf=31, mindt=2, targetdt=63,
                               soundfiledur=0.0, soundfiletotaldur=0.0, soundfilecount=0,
                               fail_on_error=True)

    def __init__(self, density=DENSITY, device=None, resampler='poly'):
        self.density = density
        for attr, default in self._REFERENCE_DEFAULTS.items():
            setattr(self, attr, default)
        # not in the reference: which GPU, the pluggable file reader, and the arithmetic of the
        # spectrogram kernel: 'fp64' (default, results bit-identical to the reference) or 'fp32'
        # (opt-in: K1 at HBM speed, magnitudes within 1e-5, a few files per thousand differ)
        self.device = device
        self.precision = 'fp64'
        self.reader = _wav_reader
        # how the default reader down-mixes and resamples: 'poly' (the channel mean and a
        # resample_poly FIR) or 'ffmpeg' (ffmpeg's own arithmetic, so files at any supported rate
        # give the reference's hashes)
        self.resampler = _check_resampler(resampler)

    # objects are pickled into worker processes by the reference CLI
    # (audfprint.py:218-223,249-265): carry only plain attributes
    def __getstate__(self):
        st = dict(self.__dict__)
        if st.get("reader") is _wav_reader:
            st["reader"] = None
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self.__dict__.setdefault("precision", "fp64")
        self.__dict__.setdefault("resampler", "poly")
        if self.reader is None:
            self.reader = _wav_reader

    # ---- device configuration -------------------------------------------------
    def _a_dec(self):
        # audfprint_analyze.py:277, same expression -> same double
        return float((1 - 0.01 * (self.density * np.sqrt(self.n_hop / 352.8) / 35)) ** (1 / OVERSAMP))

    def _configure(self, shifts):
        if self.n_fft != N_FFT or self.n_hop != N_HOP:
            raise ValueError("libafp is compiled for n_fft=512, n_hop=256")
        ctx = _lib.context(self.device)
        if self.precision not in ('fp64', 'fp32'):
            raise ValueError("precision must be 'fp64' or 'fp32'")
        fp32 = 1 if self.precision == 'fp32' else 0
        key = (float(self.density), float(self.f_sd), int(self.maxpksperframe), int(self.maxpairsperpeak),
               int(self.targetdf), int(self.mindt), int(self.targetdt), int(shifts), fp32)
        if ctx.analyzer_key != key:
            p = _lib.AnalyzerParams(self._a_dec(), HPF_POLE ** (1 / OVERSAMP), int(self.maxpksperframe),
                                    int(self.maxpairsperpeak), int(self.targetdf), int(self.mindt),
                                    int(self.targetdt), int(shifts), fp32)
            # the very doubles the reference multiplies by (audfprint_analyze.py:279, :187-192)
            win = np.ascontiguousarray(np.hanning(self.n_fft + 2)[1:-1], dtype=np.float64)
            npts = self.n_fft // 2
            gauss = np.ascontiguousarray(
                np.exp(-0.5 * ((np.arange(-npts, npts + 1) / self.f_sd) ** 2)), dtype=np.float64)
            ctx.check(ctx.lib.afp_set_analyzer(ctx.h, C.byref(p), win.ctypes.data, gauss.ctypes.data,
                                               float(self.f_sd)))
            ctx.analyzer_key = key
        return ctx

    # ---- batch entry points (the throughput path) -------------------------------
    def fingerprint_packed(self, pcm, sample_offsets, shifts=None, fetch=True, host_rows=None,
                           sample_lengths=None):
        """Fingerprint nfiles signals packed in one buffer.

        pcm             int16/float32 numpy array (host) or torch tensor (CUDA or pinned host)
        sample_offsets  int64 [nfiles+1] start of each file in `pcm`
        sample_lengths  int64 [nfiles] or None (= offsets[i+1]-offsets[i]); lets files be
                        padded to 16-byte boundaries (TMA staging)
        returns (rows int32 (U,2), row_offsets int64 (nfiles+1)) — rows of file i
        are rows[row_offsets[i]:row_offsets[i+1]], sorted by (time, hash).
        With fetch=False nothing is copied back (results stay in the workspace)."""
        shifts = self.shifts if shifts is None else shifts
        shifts = max(1, int(shifts))
        ctx = self._configure(shifts)
        off = np.ascontiguousarray(sample_offsets, dtype=np.int64)
        nfiles = len(off) - 1
        lens = None if sample_lengths is None else np.ascontiguousarray(sample_lengths, dtype=np.int64)
        lens_p = None if lens is None else lens.ctypes.data_as(C.POINTER(C.c_int64))
        ptr, on_host = _lib.ptr_of(pcm)
        if isinstance(pcm, np.ndarray):
            dtype = {np.dtype(np.int16): _lib.PCM_I16, np.dtype(np.float32): _lib.PCM_F32}[pcm.dtype]
        else:
            dtype = _lib.PCM_I16 if pcm.element_size() == 2 else _lib.PCM_F32
        total = C.c_int64(-1)
        # torch tensors: written on torch's stream, read (and host_rows written) on the context's; with
        # fetch=False the call returns while the device still reads pcm, which after_torch keeps alive
        with ctx.after_torch(pcm, host_rows):
            ctx.check(ctx.lib.afp_fingerprint_batch(ctx.h, ptr, dtype, on_host, nfiles,
                                                    off.ctypes.data_as(C.POINTER(C.c_int64)), lens_p,
                                                    C.byref(total) if fetch else None))
            if not fetch:
                return None, None
            rows = host_rows if host_rows is not None else np.empty((max(int(total.value), 0), 2), np.int32)
            roff = np.empty(nfiles + 1, np.int64)
            rptr, r_on_host = _lib.ptr_of(rows)
            ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, rptr, r_on_host, roff.ctypes.data_as(C.POINTER(C.c_int64))))
        if host_rows is not None:
            rows = rows[:int(total.value)]
        return rows, roff

    # frames of log-spectrogram workspace per device call (2 KB each): 8 M frames = 16 GB
    max_frames_per_call = 8 << 20

    def fingerprint_batch(self, signals, shifts=None):
        """List of 1-D signals (int16 or float) -> list of int32 (U,2) hash arrays.
        Long lists are cut into device calls of at most `max_frames_per_call` frames."""
        out = []
        for start, end in self._signal_chunks(signals, max(1, int(self.shifts if shifts is None else shifts))):
            packed, starts, lens = self._pack(signals[start:end])
            rows, roff = self.fingerprint_packed(packed, starts, shifts, sample_lengths=lens)
            out += [rows[roff[i]:roff[i + 1]] for i in range(end - start)]
        return out

    def ingest_batch(self, hashtable, names, signals, on_device=True):
        """Fingerprint many signals and add them to the table (batched Analyzer.ingest,
        audfprint_analyze.py:430-457).  Returns the hash counts.
        With on_device (default) the hashes never leave the GPU: every device call of at most
        `max_frames_per_call` frames fingerprints its files and HashTable.store_batch inserts
        them straight from the workspace into the device-resident table (bit-identical to
        per-track store() calls from the same `random` state).  on_device=False keeps the
        round-1 path: hashes to the host, one store() per file."""
        if not on_device:
            hashes = self.fingerprint_batch(signals, self.shifts)
            for name, sig, h in zip(names, signals, hashes):
                hashtable.store(name, h)
                self._account(len(sig) / self.target_sr)
            return [len(h) for h in hashes]
        nsh = max(1, int(self.shifts))
        counts, pending = [], None
        for start, end in self._signal_chunks(signals, nsh):
            packed, starts, lens = self._pack(signals[start:end])
            self.fingerprint_packed(packed, starts, nsh, fetch=False, sample_lengths=lens)
            # the host-side RNG replay of the previous call's overflow runs while the GPU
            # fingerprints this one
            counts += hashtable.store_batch_finish(pending)
            pending = hashtable.store_batch_begin(names[start:end])
        counts += hashtable.store_batch_finish(pending)
        for sig in signals:
            self._account(len(sig) / self.target_sr)
        return counts

    def _signal_chunks(self, signals, nsh):
        """[start, end) of the device calls that fingerprint `signals` at nsh shifts: at most
        max_frames_per_call frames each, a longer signal alone."""
        frames = [nsh * (1 + len(x) // self.n_hop) for x in signals]
        return plan_chunks(frames, [0] * len(frames), self.max_frames_per_call, float('inf'))

    @staticmethod
    def _pack(signals):
        """Signals -> one packed PCM buffer, every file on a 16-byte boundary (TMA bulk copies)."""
        arrs = [_as_pcm(s) for s in signals]
        kinds = set(k for _, k in arrs)
        if len(kinds) > 1:
            arrs = [(a.astype(np.float32) * np.float32(1.0 / 32768.0) if k == _lib.PCM_I16 else a, _lib.PCM_F32)
                    for a, k in arrs]
        lens = np.array([len(a) for a, _ in arrs], np.int64)
        al = 16 // arrs[0][0].dtype.itemsize
        starts = np.zeros(len(arrs) + 1, np.int64)
        starts[1:] = np.cumsum((lens + al - 1) // al * al)
        packed = np.zeros(int(starts[-1]) + al, arrs[0][0].dtype)
        for (a, _), s in zip(arrs, starts[:-1]):
            packed[s:s + len(a)] = a
        return packed, starts, lens

    # ---- reference methods -------------------------------------------------------
    def find_peaks(self, d, sr):
        """Waveform -> list of (time_frame, freq_bin) (audfprint_analyze.py:255-308)."""
        if len(d) == 0:
            return []
        a, dtype = _as_pcm(d)
        ctx = self._configure(1)
        off = np.array([0, len(a)], np.int64)
        ctx.check(ctx.lib.afp_fingerprint_batch(ctx.h, a.ctypes.data, dtype, 1, 1,
                                                off.ctypes.data_as(C.POINTER(C.c_int64)), None, None))
        return self._fetch_peaks(ctx, 0, 1)[0]

    def _fetch_peaks(self, ctx, shift, nfiles):
        poff = np.empty(nfiles + 1, np.int64)
        ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, shift, None, 1, poff.ctypes.data_as(C.POINTER(C.c_int64))))
        rows = np.empty((int(poff[-1]), 2), np.int32)
        ctx.check(ctx.lib.afp_fetch_peaks(ctx.h, shift, rows.ctypes.data, 1, None))
        return [[(int(c), int(b)) for c, b in rows[poff[i]:poff[i + 1]]] for i in range(nfiles)]

    def peaks2landmarks(self, pklist):
        """(col, bin) list -> (col, bin1, bin2, dt) list (audfprint_analyze.py:310-343)."""
        if len(pklist) == 0:
            return []
        rows = np.ascontiguousarray(np.array(pklist, dtype=np.int32).reshape(-1, 2))
        ctx = self._configure(1)
        n = C.c_int64(0)
        ctx.check(ctx.lib.afp_landmarks_from_peaks(ctx.h, rows.ctypes.data, len(rows), 1, C.byref(n)))
        out = np.empty((int(n.value), 4), np.int32)
        ctx.check(ctx.lib.afp_fetch_landmarks(ctx.h, out.ctypes.data, 1))
        return [tuple(int(v) for v in r) for r in out]

    def spreadpeaksinvector(self, vector, width=4.0):
        """Blurred copy of `vector`: every local maximum spread by a Gaussian of SD `width`, max
        over the bumps (audfprint_analyze.py:153-160 over spreadpeaks :162-197).  The product
        path fuses this into the peak kernel (afp_peaks.cu `spread`); this entry point runs the
        same arithmetic on the device for a stand-alone vector (afp_spread_peaks)."""
        v = np.ascontiguousarray(vector, dtype=np.float64).ravel()
        n = len(v)
        out = np.zeros(n, np.float64)
        if n == 0:
            return out
        ctx = _lib.context(self.device)
        # the very doubles the reference caches in __sp_vals (:187-192)
        tab = np.ascontiguousarray(np.exp(-0.5 * ((np.arange(-n, n + 1) / width) ** 2)), dtype=np.float64)
        ctx.check(ctx.lib.afp_spread_peaks(ctx.h, v.ctypes.data, n, tab.ctypes.data, float(width), None,
                                           out.ctypes.data))
        return out

    def _read(self, filename):
        try:
            if self.reader is _wav_reader:
                d, sr = _wav_reader(filename, sr=self.target_sr, channels=1,
                                    resampler=_check_resampler(self.resampler))
            else:
                d, sr = self.reader(filename, sr=self.target_sr, channels=1)
        except Exception as e:
            self._read_failed(filename, e)
            d, sr = [], self.target_sr
        return d, sr

    def _read_failed(self, filename, e):
        """What the reference does with a file it cannot read: raise IOError, or report and skip it."""
        message = "wavfile2peaks: Error reading " + filename
        if self.fail_on_error:
            print(e)
            raise IOError(message)
        print(message, "skipping")

    def _list_form(self, run):
        """A list form's bookkeeping around run() -> (results, durations): the durations go to
        `last_batch_durations`, and if run() raises, soundfiledur / soundfiletotaldur / soundfilecount
        are left as they were.  The per-file calls run the same drivers on one file without it."""
        saved = (self.soundfiledur, self.soundfiletotaldur, self.soundfilecount)
        try:
            results, self.last_batch_durations = run()
        except BaseException:
            self.soundfiledur, self.soundfiletotaldur, self.soundfilecount = saved
            raise
        return results

    def _account(self, dur):
        self.soundfiledur = dur
        self.soundfiletotaldur += dur
        self.soundfilecount += 1

    def wavfile2peaks(self, filename, shifts=None):
        """Soundfile -> peaks, or list of peak lists when shifts > 1
        (audfprint_analyze.py:345-383): the driver of wavfiles2peaks run on the one file."""
        return self._peaks_of_files([filename], shifts)[0][0]

    def wavfile2hashes(self, filename):
        """Soundfile -> int32 (U,2) [time, hash] rows (audfprint_analyze.py:385-426): the driver of
        wavfiles2hashes run on the one file, so a malformed .afpk file stays counted when it raises,
        as in the reference."""
        return self._hashes_of_files([filename])[0][0]

    # bytes of raw PCM (WAV payload bytes: 2, 3 or 4 a sample; decoded FLAC at _flac_format's width; or a
    # custom reader's float32) that wavfiles2hashes stages per device call
    max_pcm_bytes_per_call = 1 << 30

    def wavfiles2hashes(self, filenames):
        """List form of wavfile2hashes: per file exactly what wavfile2hashes returns ([] included),
        with soundfiledur / soundfiletotaldur / soundfilecount left as the per-file loop leaves them
        and the files' durations in `last_batch_durations`.

        WAVs read by the default reader are parsed on the host (_wav_read_raw); the raw PCM of a
        chunk of files is staged once, down-mixed and resampled by ONE front-end call into a device
        buffer (_frontend_sources), and fingerprinted there in place (fingerprint_packed).  FLAC files
        are decoded on the device into the same staging buffer first; one the device refuses is an
        unreadable file.  A custom
        `reader` is called per file and its output packed as it is.  Runs of .afpk files are loaded
        on the host and hashed by ONE afp_fingerprint_from_peaks call per chunk; .afpt files are
        loaded as they are.  Chunks follow max_frames_per_call and max_pcm_bytes_per_call (a file
        over a cap goes alone); the results do not depend on where they fall.

        Files are read in list order.  With fail_on_error, the first unreadable file raises the
        IOError wavfile2hashes raises, and nothing is returned: unlike the per-file loop, which has
        already returned the earlier files' hashes by then, the counters are left as they were.  A
        malformed precomputed file raises what wavfile2hashes raises for it, the same way."""
        return self._list_form(lambda: self._hashes_of_files(filenames))

    def _hashes_of_files(self, filenames, rows_on_device=False):
        """The driver of wavfile2hashes and wavfiles2hashes -> (hashes, durations) per file; with
        rows_on_device the fingerprinted files' hashes stay on the device (afp_fetch_hashes into a
        torch tensor) as DeviceHashes."""
        def collect(kind, idx, results):
            # the reference returns [] when a WAV has no peaks (:401-402)
            self._collect_hashes(idx, results, rows_on_device, kind == 'pcm' and self.shifts < 2)
        return self._analyse_files(filenames, False, max(1, int(self.shifts)), collect, list)

    def _analyse_files(self, filenames, peaks_mode, nsh, collect, empty):
        """The file driver: read `filenames` in rounds (_file_rounds), run each device round at nsh
        shifts and hand it to `collect(kind, indices, results)`, which puts the round's results at
        their indices.  A file whose result is known on the host takes it as it is, or `empty()` when
        it has no samples.  -> (results, durations).  The files are counted after the last round.
        When a file raises nothing is counted, except a malformed .afpk file, which the reference
        counts before it raises (_peaks_round); the list forms then restore the counters (_list_form)."""
        n = len(filenames)
        results, durs = [None] * n, [0.0] * n
        for kind, items in self._file_rounds(filenames, peaks_mode, nsh, False):
            if kind == 'host':
                for i, value, dur in items:
                    results[i], durs[i] = (empty() if value is None else value), dur
                continue
            refused = []
            if kind == 'pcm':
                refused = self._fingerprint_pcm(items, nsh, durs)
                self._refuse(filenames, items, refused)
            else:
                self._peaks_round(items, durs)
            collect(kind, [it[0] for it in items], results)
            for k, _ in refused:
                results[items[k][0]] = empty()          # an unreadable file has no samples
        for dur in durs:
            self._account(dur)
        return results, durs

    def _file_rounds(self, filenames, peaks_mode, nsh, in_order):
        """Read `filenames` in list order and group them into rounds of one kind, each one device call:
          ('pcm',   [(i, pcm, nsamples, dur)])  audio for one front-end + fingerprint call (dur None
                                                until the front-end gives the resampled length)
          ('peaks', [(i, rows int32 (n,2), dur)]) .afpk files for one afp_fingerprint_from_peaks
          ('host',  [(i, value, dur)])         files whose result is known on the host: .afpt hashes
                                                (.afpk peaks with peaks_mode), None for audio without samples
        A round closes when a cap (max_frames_per_call, max_pcm_bytes_per_call) is reached.  With
        in_order (a caller that stores in list order) it also closes when the kind changes, so rounds
        come in list order; otherwise a round of each device kind stays open across the other files
        and host files pass through as rounds of one.  When reading a file raises, the open rounds
        (files before it) are yielded first, then the exception propagates, so a caller can finish the
        earlier files as the per-file loop does.  Audio files count nsh frames per hop against
        max_frames_per_call."""
        open_ = {}                                 # kind -> (items, planner) of its open round
        try:
            for i, fn in enumerate(filenames):
                k, item, frames, nbytes = self._read_item(i, fn, nsh, peaks_mode)
                if k == 'host' and not in_order:
                    yield k, [item]
                    continue
                if in_order and open_ and k not in open_:
                    for kind, (items, _) in list(open_.items()):
                        yield kind, items
                    open_.clear()
                if k not in open_:
                    open_[k] = ([], _ChunkPlanner(self.max_frames_per_call, self.max_pcm_bytes_per_call))
                    open_[k][1].add(frames, nbytes)
                elif open_[k][1].add(frames, nbytes):
                    yield k, open_[k][0]
                    open_[k] = ([], open_[k][1])
                open_[k][0].append(item)
        except Exception:
            for kind, (items, _) in list(open_.items()):
                yield kind, items
            raise
        for kind, (items, _) in list(open_.items()):
            yield kind, items

    def _read_item(self, i, fn, nsh, peaks_mode):
        """One file of _file_rounds -> (kind, item, frames, bytes).  Raises for a file it cannot read
        (_read_failed, fail_on_error), before anything is counted."""
        ext = os.path.splitext(fn)[1]
        if ext == PRECOMPEXT and not peaks_mode:
            hashes = hashes_load(fn)
            return 'host', (i, hashes, np.max(hashes, axis=0)[0] * self.n_hop / self.target_sr), 0, 0
        if ext == PRECOMPPKEXT:
            peaks = peaks_load(fn)
            dur = np.max(peaks, axis=0)[0] * self.n_hop / self.target_sr        # raises for an empty file
            if peaks_mode:
                return 'host', (i, peaks, dur), 0, 0
            rows = _peak_rows(peaks)
            return 'peaks', (i, rows, dur), max(1, int(rows[-1, 0]) + 1), rows.nbytes
        if self.reader is _wav_reader:
            try:
                raw, nch, fs = _audio_read_raw(fn)
                if fs < 1:
                    # no rate to resample from: the device front-end would refuse it (down < 1)
                    raise ValueError("%s: sample rate %d" % (fn, fs))
                nframes = len(raw) // nch if isinstance(raw, np.ndarray) else self._flac_frames(raw)
                if _check_resampler(self.resampler) == 'ffmpeg':
                    _swr_check(fn, raw, nch, fs, self.target_sr)
                    nout = swr_length(nframes, fs, self.target_sr)
                else:
                    nout = -(-nframes * self.target_sr // fs)      # ceil(nframes * up / down)
            except Exception as e:
                self._read_failed(fn, e)
                raw, nch, fs, nframes, nout = np.zeros(0, np.int16), 1, self.target_sr, 0, 0
            if nout == 0:
                return 'host', (i, None, 0.0), 0, 0
            if isinstance(raw, np.ndarray):
                nbytes = raw.nbytes                   # the payload as it goes up: 2, 3 or 4 bytes a sample
            else:                                     # decoded FLAC
                nbytes = _WIDTH[_flac_format(raw, self.resampler)] * nframes * nch
            return 'pcm', (i, (raw, nch, fs), nout, None), nsh * (1 + nout // self.n_hop), nbytes
        d, sr = self._read(fn)
        if len(d) == 0:
            return 'host', (i, None, len(d) / sr), 0, 0
        a = _as_pcm(d)[0]
        return 'pcm', (i, a, len(d), len(d) / sr), nsh * (1 + len(d) // self.n_hop), a.nbytes

    def _flac_frames(self, stream):
        """Samples per channel of a FLAC file for the round planner: STREAMINFO's count, or when that
        is 0 (unknown) the count the device finds by locating the file's frames.  Raises for a file
        the device refuses."""
        if stream.total_samples:
            return stream.total_samples
        nsamples, status = flac.locate(_lib.context(self.device), [stream])
        if status[0]:
            raise flac.failure(status[0])
        return int(nsamples[0])

    def _fingerprint_pcm(self, items, shifts, durs):
        """Fingerprint one 'pcm' round in one device call at `shifts`; the results stay in the
        workspace.  Each file's duration goes to durs[i].  Returns [(position in items, AFP_FLAC_*
        code)] of the FLAC files the device refused; they are fingerprinted as files without samples,
        and the caller reports them (_refuse)."""
        idx = [it[0] for it in items]
        if self.reader is _wav_reader:
            raws = [it[1] for it in items]
            out, off, lens, status = _frontend_sources([r[0] for r in raws], [r[1] for r in raws],
                                                       [r[2] for r in raws], self.target_sr, device=self.device,
                                                       resampler=_check_resampler(self.resampler))
            for i, ln in zip(idx, lens):
                durs[i] = int(ln) / self.target_sr
            self.fingerprint_packed(out, off, shifts, fetch=False, sample_lengths=lens)
            return [(k, int(c)) for k, c in enumerate(status) if c]
        for it in items:
            durs[it[0]] = it[3]
        packed, starts, lens = self._pack([it[1] for it in items])
        self.fingerprint_packed(packed, starts, shifts, fetch=False, sample_lengths=lens)
        return []

    def _refuse(self, filenames, items, refused):
        """Report the files _fingerprint_pcm refused as unreadable, in list order: under fail_on_error
        the first raises _read_failed's IOError."""
        for k, code in refused:
            self._read_failed(filenames[items[k][0]], flac.failure(code))

    def _fingerprint_peaks(self, arrays):
        """wavfile2hashes of many .afpk peak lists (int32 (n,2) each, n >= 1) in ONE
        afp_fingerprint_from_peaks call; the results stay in the workspace.  When a file's peaks are
        malformed, raises what the per-file call raises for it, with the file's position in
        `arrays` as the exception's `file_index`."""
        ctx = self._configure(max(1, int(self.shifts)))
        n = len(arrays)
        off = np.zeros(n + 1, np.int64)
        off[1:] = np.cumsum([len(a) for a in arrays])
        rows = np.ascontiguousarray(np.concatenate(arrays), dtype=np.int32) if off[-1] else None
        status = np.zeros(max(n, 1), np.int32)
        rc = ctx.lib.afp_fingerprint_from_peaks(ctx.h, rows.ctypes.data if rows is not None else None, 1, n,
                                                off.ctypes.data_as(C.POINTER(C.c_int64)), status.ctypes.data, None)
        if rc:
            try:
                ctx.check(rc)
            except Exception as e:
                if status.any():
                    e.file_index = int(np.flatnonzero(status)[0])
                raise

    def _peaks_round(self, items, durs, before=None):
        """Fingerprint one 'peaks' round of _file_rounds (_fingerprint_peaks); file i's duration goes
        to durs[i].  A malformed file raises, counted first as the per-file call counts it: the
        reference's wavfile2peaks counts the file before its peaks are hashed.  `before(k)`, when
        given, finishes the k files before it ahead of that count."""
        for i, _, dur in items:
            durs[i] = dur
        try:
            self._fingerprint_peaks([it[1] for it in items])
        except Exception as e:
            k = getattr(e, 'file_index', None)
            if k is None:
                raise
            if before is not None:
                before(k)
            self._account(durs[items[k][0]])
            raise

    def _collect_hashes(self, idx, results, rows_on_device, empty_as_list):
        """Put the hashes of the last device call's files at their indices `idx` of `results`; with
        empty_as_list a file without hashes gets []."""
        ctx = _lib.context(self.device)
        roff = np.empty(len(idx) + 1, np.int64)
        ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, None, 1, roff.ctypes.data_as(C.POINTER(C.c_int64))))
        total = int(roff[-1])
        if rows_on_device:
            import torch
            rows = torch.empty((max(total, 1), 2), dtype=torch.int32, device=torch.device("cuda", ctx.device))
            with ctx.after_torch(rows):   # torch's pending reads of rows' memory come first
                ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, C.c_void_p(rows.data_ptr()), 0, None))
            ends = np.maximum(roff[1:] - 1, 0)
            last = rows[torch.from_numpy(ends).to(rows.device), 0].cpu().numpy() if total else np.zeros(len(idx), np.int32)
        else:
            rows = np.empty((total, 2), np.int32)
            ctx.check(ctx.lib.afp_fetch_hashes(ctx.h, rows.ctypes.data, 1, None))
        for k, i in enumerate(idx):
            lo, hi = int(roff[k]), int(roff[k + 1])
            if empty_as_list and hi == lo:
                results[i] = []
            elif rows_on_device:
                results[i] = DeviceHashes(rows[lo:hi], last[k])
            else:
                results[i] = rows[lo:hi]

    def wavfiles2peaks(self, filenames, shifts=None):
        """List form of wavfile2peaks: per file exactly what wavfile2peaks(filename, shifts) returns,
        with the counters and `last_batch_durations` as wavfiles2hashes leaves them.

        Audio goes through the batched front-end and ONE fingerprint call per chunk, at 1 shift when
        `shifts` is None or < 2, else at self.shifts with min(shifts, self.shifts) peak lists per
        file (`shifts` empty lists for audio without samples); one afp_fetch_peaks per shift serves
        the whole chunk.  .afpk files are loaded on the host; .afpt files are read as audio, as the
        reference reads them.  Failures behave as in wavfiles2hashes."""
        return self._list_form(lambda: self._peaks_of_files(filenames, shifts))

    def _peaks_of_files(self, filenames, shifts):
        """The driver of wavfile2peaks and wavfiles2peaks -> (peaks, durations) per file."""
        multi = not (shifts is None or shifts < 2)
        # NB the reference takes the offsets from self.shifts (audfprint_analyze.py:375)
        nsh = max(1, int(self.shifts)) if multi else 1

        def collect(kind, idx, results):
            ctx = _lib.context(self.device)
            per_shift = [self._fetch_peaks(ctx, s, len(idx)) for s in range(min(shifts, nsh) if multi else 1)]
            for k, i in enumerate(idx):
                results[i] = [p[k] for p in per_shift] if multi else per_shift[0][k]
        return self._analyse_files(filenames, True, nsh, collect,
                                   (lambda: [[] for _ in range(shifts)]) if multi else list)

    def ingest(self, hashtable, filename):
        """Read a file and add it to the table (audfprint_analyze.py:430-457)."""
        hashes = self.wavfile2hashes(filename)
        hashtable.store(filename, hashes)
        return self.soundfiledur, len(hashes)

    def ingest_files(self, hashtable, filenames):
        """List form of the reference's `new` / `add` loop (audfprint.py:173-187): returns
        [self.ingest(hashtable, f) for f in filenames], and leaves the table (table, counts, names,
        hashesperid), the counters and the `random` state exactly as that loop leaves them.

        Audio chunks are fingerprinted on the device and stored from the workspace in place
        (HashTable.store_batch_begin(names, None)); runs of .afpk files go through ONE
        afp_fingerprint_from_peaks call per chunk and are stored the same way; .afpt files and files
        without samples (unreadable under fail_on_error = False, empty, no peaks) are stored from host
        rows.  A name takes its id in list order whatever its file yields.  The host replay of
        random.randint for one round's full buckets runs while the device fingerprints the next round.

        With fail_on_error, an unreadable or malformed file raises what the per-file loop raises, after
        the files before it (those of its own round included) have been stored: a table cannot be
        rolled back cheaply, so the state is the loop's state at that point, not the state before."""
        n = len(filenames)
        out, durs = [None] * n, [0.0] * n
        pending = [None]          # (store token, indices) of the round begun and not yet finished

        def finish():
            if pending[0] is not None:
                token, idx = pending[0]
                pending[0] = None
                for i, cnt in zip(idx, hashtable.store_batch_finish(token)):
                    out[i] = (durs[i], cnt)
                    self._account(durs[i])

        def begin(idx, hashes):
            finish()
            pending[0] = (hashtable.store_batch_begin([filenames[i] for i in idx], hashes), idx)

        try:
            for kind, items in self._file_rounds(filenames, False, max(1, int(self.shifts)), True):
                idx = [it[0] for it in items]
                if kind == 'host':
                    for i, _, dur in items:
                        durs[i] = dur
                    begin(idx, [[] if it[1] is None else it[1] for it in items])
                    continue
                if kind == 'pcm':
                    refused = self._fingerprint_pcm(items, self.shifts, durs)
                    if refused and self.fail_on_error:
                        # the loop stores the files before the refused one; it is not counted
                        k = refused[0][0]
                        if k:
                            self._fingerprint_pcm(items[:k], self.shifts, durs)
                            begin(idx[:k], None)
                        finish()
                    self._refuse(filenames, items, refused)
                else:
                    def before(k):
                        # the loop stores the files before the malformed one
                        if k:
                            self._fingerprint_peaks([it[1] for it in items[:k]])
                            begin(idx[:k], None)
                        finish()
                    self._peaks_round(items, durs, before)
                begin(idx, None)
            finish()
        except BaseException:
            finish()
            raise
        return out

    # files analysed together by one precompute_files round
    max_files_per_precompute = 4096

    def precompute_file(self, filename, precompdir, type='hashes', skip_existing=False, strip_prefix=None):
        """`precompute` of one file (file_precompute + file_precompute_peaks_or_hashes,
        audfprint.py:70-127): writes `precompdir`/name.afpt (type 'hashes') or .afpk (any other
        type: peaks) and returns the one-message list the reference returns."""
        print(time.ctime(), "precomputing", type, "for", filename, "...")
        return self._precompute_one(filename, precompdir, type, skip_existing, strip_prefix)

    def _precompute_one(self, filename, precompdir, type, skip_existing, strip_prefix):
        hashes = type == 'hashes'
        opfname = precompute_name(filename, precompdir, hashes, strip_prefix)
        if skip_existing and os.path.isfile(opfname):
            return ["file " + opfname + " exists (and --skip-existing); skipping"]
        output = self.wavfile2hashes(filename) if hashes else self.wavfile2peaks(filename)
        return [_precompute_write(filename, opfname, hashes, output, self.soundfiledur)]

    def precompute_files(self, filenames, precompdir, type='hashes', skip_existing=False, strip_prefix=None):
        """List form of precompute_file: one message list per file, and the very files the per-file
        loop writes, byte for byte, including two effects of its order: with skip_existing a file
        whose output an earlier file of the list wrote is skipped, and a later file with the same
        output name overwrites an earlier one.

        The list is cut into rounds (next_precompute_round) of at most max_files_per_precompute
        files; each round prints file_precompute's "precomputing" line for its files in list order,
        analyses the files it does not skip with ONE wavfiles2hashes / wavfiles2peaks call, and
        writes them in list order.  When that call raises (fail_on_error), the round runs file by
        file instead, so that the files before the failing one are written and the per-file
        exception is raised, as in the loop."""
        hashes = type == 'hashes'
        n = len(filenames)
        opnames = [precompute_name(f, precompdir, hashes, strip_prefix) for f in filenames]
        msgs = [None] * n
        start = 0
        while start < n:
            end, skipped = next_precompute_round(opnames, start, skip_existing, os.path.isfile,
                                                 max(1, int(self.max_files_per_precompute)))
            for i in range(start, end):
                print(time.ctime(), "precomputing", type, "for", filenames[i], "...")
            skipped = set(skipped)
            todo = [i for i in range(start, end) if i not in skipped]
            try:
                names = [filenames[i] for i in todo]
                outs = self.wavfiles2hashes(names) if hashes else self.wavfiles2peaks(names)
            except Exception:
                for i in range(start, end):
                    msgs[i] = self._precompute_one(filenames[i], precompdir, type, skip_existing, strip_prefix)
                start = end
                continue
            durs = self.last_batch_durations
            for i in range(start, end):
                if i in skipped:
                    msgs[i] = ["file " + opnames[i] + " exists (and --skip-existing); skipping"]
            for k, i in enumerate(todo):
                msgs[i] = [_precompute_write(filenames[i], opnames[i], hashes, outs[k], durs[k])]
            start = end
        return msgs

    # ---- parity probes -------------------------------------------------------------
    def stft_magnitude(self, d):
        """|STFT| (257, T) float64 — np.abs(stft.stft(...)) of the reference."""
        a, dtype = _as_pcm(d)
        ctx = self._configure(1)
        T = 1 + len(a) // self.n_hop
        out = np.empty((T, 257), np.float64)
        ctx.check(ctx.lib.afp_stft_mag(ctx.h, a.ctypes.data, dtype, 1, len(a), out.ctypes.data, 1))
        return out.T

    def conditioned_sgram(self, d):
        """log / mean / high-pass spectrogram (256, T) float64 (audfprint_analyze.py:280-295)."""
        a, dtype = _as_pcm(d)
        ctx = self._configure(1)
        T = 1 + len(a) // self.n_hop
        out = np.empty((T, 256), np.float64)
        ctx.check(ctx.lib.afp_sgram(ctx.h, a.ctypes.data, dtype, 1, len(a), out.ctypes.data, 1))
        return out.T


# ---- precomputed-file codecs (byte-compatible, audfprint_analyze.py:460-514) --------
HASH_FMT = '<2i'
HASH_MAGIC = b'audfprinthashV00'
PEAK_FMT = '<2i'
PEAK_MAGIC = b'audfprintpeakV00'


def _pairs_save(fname, magic, pairs):
    arr = np.asarray(pairs, dtype='<i4').reshape(-1, 2)
    with open(fname, 'wb') as f:
        f.write(magic)
        f.write(arr.tobytes())


def _pairs_load(fname, magic, what):
    with open(fname, 'rb') as f:
        got = f.read(len(magic))
        if got != magic:
            raise IOError('%s is not a %s file (magic %s)' % (fname, what, got))
        data = f.read()
    n = len(data) // struct.calcsize(HASH_FMT)
    arr = np.frombuffer(data[:n * 8], dtype='<i4').reshape(-1, 2)
    return [(int(a), int(b)) for a, b in arr]


def hashes_save(hashfilename, hashes):
    _pairs_save(hashfilename, HASH_MAGIC, hashes)


def hashes_load(hashfilename):
    return _pairs_load(hashfilename, HASH_MAGIC, 'hash')


def peaks_save(peakfilename, peaks):
    _pairs_save(peakfilename, PEAK_MAGIC, peaks)


def peaks_load(peakfilename):
    return _pairs_load(peakfilename, PEAK_MAGIC, 'peak')


def glob2hashtable(pattern, density=20.0):
    """Build a hash table from the files matching a glob pattern (audfprint_analyze.py:560-579):
    the files are read on the host, fingerprinted in one batched device call and inserted in
    glob order."""
    import glob
    import time
    from .hash_table import HashTable
    analyzer = Analyzer(density=density)
    ht = HashTable()
    files = glob.glob(pattern)
    t0 = time.time()
    signals = [analyzer._read(fn)[0] for fn in files]
    counts = analyzer.ingest_batch(ht, files, signals)
    total = analyzer.soundfiletotaldur
    if total > 0:
        print("Added", sum(counts), "(", sum(counts) / total, "hashes/sec) at ", (time.time() - t0) / total, "x RT")
    return ht
