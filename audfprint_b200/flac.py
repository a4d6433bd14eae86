"""FLAC input: the host half (recognising a FLAC file, reading its metadata blocks) and the calls of
the device decoder (afp_flac_locate_batch / afp_flac_decode_batch_bytes, include/afp.h).

The host only finds where the frames start and what STREAMINFO says; locating, checking and decoding
the frames run on the device.  Native FLAC only: Ogg-FLAC (an Ogg container) is not recognised and
reads as an unreadable file, like any other format but PCM and float WAV.  The STREAMINFO MD5 signature is
not checked, as ffmpeg does not check it by default."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

MAGIC = b'fLaC'
# per-file codes of the device decoder (afp.h AFP_FLAC_*)
STATUS_TEXT = {1: "bits per sample outside 4-24", 2: "broken frame chain", 3: "frame CRC-16 mismatch",
               4: "reserved code", 5: "truncated last frame", 6: "subframe data does not fit its frame"}

STREAMINFO, LAST_TYPE = 0, 126      # block types 1-126 are skipped; 127 is invalid


class FlacStream(object):
    """One FLAC file as the device decoder takes it: the bytes of its frames (everything after the
    metadata blocks) and the STREAMINFO fields."""
    __slots__ = ("frames", "sample_rate", "channels", "bits_per_sample", "max_blocksize", "total_samples")

    def __init__(self, frames, sample_rate, channels, bits_per_sample, max_blocksize, total_samples):
        self.frames = frames
        self.sample_rate, self.channels, self.bits_per_sample = sample_rate, channels, bits_per_sample
        self.max_blocksize, self.total_samples = max_blocksize, total_samples


def id3v2_end(data, pos=0):
    """Offset after the ID3v2 tags that start at `pos` (none: `pos`), as ffmpeg's demuxer skips them."""
    while len(data) >= pos + 10 and data[pos:pos + 3] == b'ID3':
        size = 0
        for b in data[pos + 6:pos + 10]:
            if b & 0x80:
                return pos               # not a synchsafe size: not a tag
            size = (size << 7) | b
        pos += 10 + size + (10 if data[pos + 5] & 0x10 else 0)      # footer flag
    return pos


def is_flac(data):
    """True when `data` (the file's first bytes, enough to hold its ID3v2 tags) is a native FLAC stream."""
    pos = id3v2_end(data)
    return data[pos:pos + 4] == MAGIC


def parse(data):
    """A whole FLAC file's bytes -> FlacStream.  Raises IOError for a malformed metadata block chain:
    no STREAMINFO first, a STREAMINFO that is not 34 bytes or repeats, the invalid block type 127, or a
    block that runs past the end of the file."""
    pos = id3v2_end(data)
    if data[pos:pos + 4] != MAGIC:
        raise IOError("not a FLAC stream")
    pos += 4
    info, last = None, False
    while not last:
        if pos + 4 > len(data):
            raise IOError("FLAC metadata: truncated block header")
        last, typ = bool(data[pos] & 0x80), data[pos] & 0x7F
        length = int.from_bytes(data[pos + 1:pos + 4], 'big')
        pos += 4
        if pos + length > len(data):
            raise IOError("FLAC metadata: block of type %d runs past the end of the file" % typ)
        if typ == STREAMINFO:
            if info is not None or length != 34:
                raise IOError("FLAC metadata: malformed STREAMINFO")
            info = data[pos:pos + 34]
        elif typ > LAST_TYPE:
            raise IOError("FLAC metadata: invalid block type %d" % typ)
        elif info is None:
            raise IOError("FLAC metadata: the first block is not STREAMINFO")
        pos += length
    if info is None:
        raise IOError("FLAC metadata: no STREAMINFO")
    max_bs = int.from_bytes(info[2:4], 'big')
    word = int.from_bytes(info[10:18], 'big')
    rate, ch, bps, total = word >> 44, ((word >> 41) & 7) + 1, ((word >> 36) & 31) + 1, word & ((1 << 36) - 1)
    if rate < 1:
        raise IOError("FLAC STREAMINFO: sample rate 0")
    return FlacStream(np.frombuffer(data, np.uint8)[pos:], rate, ch, bps, max_bs, total)


def read(filename):
    """parse() of a file."""
    with open(filename, 'rb') as f:
        return parse(f.read())


def _table(streams):
    """Packed frame bytes and the afp_flac_stream table of a list of FlacStream."""
    tab = (_lib.FlacStream * max(len(streams), 1))()
    off = 0
    for k, s in enumerate(streams):
        tab[k] = _lib.FlacStream(off, len(s.frames), s.sample_rate, s.channels, s.bits_per_sample, s.max_blocksize)
        off += len(s.frames)
    packed = np.concatenate([s.frames for s in streams]) if off else np.zeros(1, np.uint8)
    return np.ascontiguousarray(packed), off, tab


def locate(ctx, streams):
    """afp_flac_locate_batch over `streams` -> (samples per channel int64 [n], status int32 [n]).
    The batch stays located for decode_into."""
    packed, nbytes, tab = _table(streams)
    n = len(streams)
    nsamples = np.zeros(max(n, 1), np.int64)
    status = np.zeros(max(n, 1), np.int32)
    rc = ctx.lib.afp_flac_locate_batch(ctx.h, packed.ctypes.data, 1, nbytes, n, tab,
                                       nsamples.ctypes.data_as(C.POINTER(C.c_int64)), status.ctypes.data)
    _check_files(ctx, rc, status)
    return nsamples[:n], status[:n]


def decode_into(ctx, out, out_offsets):
    """decode_into_bytes of the last located batch into the device int16 tensor `out`, every file int16:
    file i at out[out_offsets[i]:].  -> status int32 [n]."""
    import torch
    return decode_into_bytes(ctx, out.view(torch.uint8), 2 * np.asarray(out_offsets, dtype=np.int64), False)


def decode_into_bytes(ctx, out, out_offsets, full_depth):
    """afp_flac_decode_batch_bytes of the last located batch into the device uint8 tensor `out` (the
    caller orders it against torch with ctx.after_torch): file i at byte out_offsets[i], int16, or with
    full_depth a file of 17-24 bits as int32 x << (32 - bits).  -> status int32 [n]."""
    off = np.ascontiguousarray(out_offsets, dtype=np.int64)
    n = len(off)
    status = np.zeros(max(n, 1), np.int32)
    rc = ctx.lib.afp_flac_decode_batch_bytes(ctx.h, out.data_ptr(), out.numel(),
                                             off.ctypes.data_as(C.POINTER(C.c_int64)), int(bool(full_depth)),
                                             status.ctypes.data)
    _check_files(ctx, rc, status)
    return status[:n]


def _check_files(ctx, rc, status):
    """Raise for a failure that is not a file's own (those are in `status`)."""
    if rc and not status.any():
        ctx.check(rc)


def failure(code):
    """The IOError of a file the device refused with AFP_FLAC_* `code`."""
    return IOError("FLAC: " + STATUS_TEXT.get(int(code), "status %d" % code))


def decode(stream, device=None):
    """One file -> its interleaved int16 samples (host), decoded on the device.  Raises failure()."""
    import torch
    ctx = _lib.context(device)
    nsamples, status = locate(ctx, [stream])
    if status[0]:
        raise failure(status[0])
    n = int(nsamples[0]) * stream.channels
    out = torch.empty(max(n, 1), dtype=torch.int16, device=torch.device("cuda", ctx.device))
    with ctx.after_torch(out):
        status = decode_into(ctx, out, [0])
    if status[0]:
        raise failure(status[0])
    return out[:n].cpu().numpy()
