"""A small FLAC bit writer for test fixtures: native FLAC streams built construct by construct, for the
constructs FFmpeg's encoder does not emit (variable block size, escape partitions, LPC order 32,
explicit block-size and sample-rate header codes, 4-20-bit depths, wasted bits, ID3v2 prefixes,
STREAMINFO without a sample count) and for damaged files.  tools/make_golden_flac.py writes its
output to tests/golden/flac.npz, where FFmpeg's decode of each file is stored beside it;
tests/test_flac_cpu.py checks that this writer still produces the stored bytes."""
from __future__ import annotations

import numpy as np

_STD_BS = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, 256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12, 8192: 13,
           16384: 14, 32768: 15}
_STD_SR = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
           96000: 11}
_SS = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6, 32: 7}


def _crc_table(poly, width):
    top, mask, tab = 1 << (width - 1), (1 << width) - 1, []
    for i in range(256):
        c = i << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) & mask if c & top else (c << 1) & mask
        tab.append(c)
    return tab


_T8, _T16 = _crc_table(0x07, 8), _crc_table(0x8005, 16)


def crc8(data):
    c = 0
    for b in data:
        c = _T8[c ^ b]
    return c


def crc16(data):
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _T16[(c >> 8) ^ b]
    return c


class Bits(object):
    """MSB-first bit string."""

    def __init__(self):
        self.parts = []

    def u(self, v, n):
        if n:
            self.parts.append(format(int(v) & ((1 << n) - 1), "0%db" % n))

    def unary(self, q):
        self.parts.append("0" * int(q) + "1")

    def tobytes(self):
        s = "".join(self.parts)
        s += "0" * (-len(s) % 8)
        return int(s, 2).to_bytes(len(s) // 8, "big") if s else b""


def utf8_number(v):
    if v < 0x80:
        return bytes([v])
    for n in range(2, 8):
        if v < 1 << (5 * n + 1) or n == 7:
            break
    out = []
    for _ in range(n - 1):
        out.append(0x80 | (v & 0x3F))
        v >>= 6
    lead = (0xFF00 >> n) & 0xFF
    return bytes([lead | v] + out[::-1])


def _width(r):
    """Bits of the smallest signed field that holds every value of r (0 when all are 0)."""
    m = int(max(np.max(r), -np.min(r) - 1)) if len(r) else 0
    return 0 if not np.any(r) else m.bit_length() + 1


def residual(w, r, order, bs, po=0, method=0, escape=(), *, rice=None, esc_width=None):
    """Rice-coded residual r (the block's residual after `order` warm-up samples); partitions listed in
    `escape` are written raw.  rice: a Rice parameter per partition (None: chosen from the partition's
    mean); esc_width: the escape partitions' sample width (None: the narrowest that holds them).  A
    method above 1 or a partition order that does not divide the block writes only what fits, for
    streams a decoder must refuse."""
    w.u(method, 2)
    w.u(po, 4)
    kbits, esc = (5, 31) if method else (4, 15)
    psize = bs >> po
    i = 0
    for p in range(1 << po):
        n = max(psize - (order if p == 0 else 0), 0)
        part = np.asarray(r[i:i + n], np.int64)
        i += n
        if p in escape:
            nb = _width(part) if esc_width is None else esc_width
            w.u(esc, kbits)
            w.u(nb, 5)
            for v in part:
                w.u(int(v), nb)
            continue
        mean = float(np.mean(np.abs(part))) if len(part) else 0.0
        k = min(max(int(np.log2(mean + 1.0)), 0), esc - 1) if rice is None or rice[p] is None else rice[p]
        w.u(k, kbits)
        for v in part:
            v = int(v)
            u = (v << 1) if v >= 0 else ((-v) << 1) - 1
            w.unary(u >> k)
            w.u(u & ((1 << k) - 1), k)


def subframe(w, x, sbps, kind="fixed", order=2, coefs=None, prec=12, shift=10, wasted=0, po=0, method=0,
             escape=(), sub_type=None, *, rice=None, esc_width=None, raw=None, pad=0, prec_code=None):
    """One subframe of the int64 samples x at sbps bits.  kind: constant, verbatim, fixed (order 0-4),
    lpc (coefs quantised ints, precision prec, shift).  sub_type overrides the 6-bit type code.
    rice / esc_width: see residual(); raw: the residual to write instead of x's (x then gives only the
    warm-up samples), pad: the subframe header's padding bit, prec_code: the 4-bit precision code
    instead of prec - 1."""
    x = np.asarray(x, np.int64)
    bs = len(x)
    w.u(pad, 1)
    code = {"constant": 0, "verbatim": 1, "fixed": 8 + order, "lpc": 32 + (len(coefs or [1]) - 1)}[kind]
    w.u(code if sub_type is None else sub_type, 6)
    if wasted:
        assert not np.any(x & ((1 << wasted) - 1))
        w.u(1, 1)
        w.unary(wasted - 1)
        x = x >> wasted
        sbps -= wasted
    else:
        w.u(0, 1)
    if kind == "constant":
        assert np.all(x == x[0])
        w.u(int(x[0]), sbps)
    elif kind == "verbatim":
        for v in x:
            w.u(int(v), sbps)
    elif kind == "fixed":
        for v in x[:order]:
            w.u(int(v), sbps)
        r = x.copy()
        for _ in range(order):
            r = np.diff(r)
        residual(w, r if raw is None else raw, order, bs, po, method, escape, rice=rice, esc_width=esc_width)
    else:
        c = np.asarray(coefs, np.int64)
        p = len(c)
        for v in x[:p]:
            w.u(int(v), sbps)
        w.u(prec - 1 if prec_code is None else prec_code, 4)
        w.u(shift, 5)
        for v in c:
            w.u(int(v), prec)
        pred = np.zeros(max(bs - p, 0), np.int64)
        for j in range(p):
            pred += c[j] * x[p - 1 - j:bs - 1 - j]
        r = x[p:] - (pred >> shift) if raw is None else raw
        residual(w, r, p, bs, po, method, escape, rice=rice, esc_width=esc_width)


def frame(block, number, bps, rate, variable=False, chmode=None, bs_code=None, sr_code=None, specs=None, *,
          ss_code=None, reserved=0, tail=b""):
    """One frame of the int64 block (bs, nch): its header, subframes and CRC-16.  chmode 8-10 codes the
    first two channels as left/side, right/side or mid/side.  specs: one dict of subframe() keywords
    per channel.  ss_code: the sample-size code (None: the code of bps, 0 for a depth without one);
    reserved: the header's reserved bit; tail: bytes after the subframes, before the CRC-16."""
    block = np.asarray(block, np.int64)
    bs, nch = block.shape
    chmode = nch - 1 if chmode is None else chmode
    if bs_code is None:
        bs_code = _STD_BS.get(bs, 6 if bs <= 256 else 7)
    if sr_code is None:
        sr_code = _STD_SR.get(rate, 0)
    if ss_code is None:
        ss_code = _SS.get(bps, 0)
    hdr = bytearray([0xFF, 0xF8 | int(variable), (bs_code << 4) | sr_code, (chmode << 4) | (ss_code << 1) | reserved])
    hdr += utf8_number(number)
    if bs_code == 6:
        hdr += bytes([bs - 1])
    elif bs_code == 7:
        hdr += (bs - 1).to_bytes(2, "big")
    if sr_code == 12:
        hdr += bytes([rate // 1000])
    elif sr_code == 13:
        hdr += rate.to_bytes(2, "big")
    elif sr_code == 14:
        hdr += (rate // 10).to_bytes(2, "big")
    hdr.append(crc8(hdr))
    chans = [block[:, c] for c in range(nch)]
    side = [False] * nch
    if chmode == 8:
        chans[1], side[1] = chans[0] - chans[1], True
    elif chmode == 9:
        chans[0], side[0] = chans[0] - chans[1], True
    elif chmode == 10:
        chans[0], chans[1] = (block[:, 0] + block[:, 1]) >> 1, block[:, 0] - block[:, 1]
        side[1] = True
    w = Bits()
    specs = specs or [{}] * nch
    for c in range(nch):
        subframe(w, chans[c], bps + side[c], **specs[c])
    body = bytes(hdr) + w.tobytes() + tail
    out = bytearray(body)
    out += crc16(out).to_bytes(2, "big")
    return bytes(out)


def streaminfo(min_bs, max_bs, rate, nch, bps, total, last=True):
    w = Bits()
    w.u(min_bs, 16)
    w.u(max_bs, 16)
    w.u(0, 24)
    w.u(0, 24)
    w.u(rate, 20)
    w.u(nch - 1, 3)
    w.u(bps - 1, 5)
    w.u(total, 36)
    w.u(0, 64)
    w.u(0, 64)
    return block_header(0, 34, last) + w.tobytes()


def block_header(typ, length, last):
    return bytes([(0x80 if last else 0) | typ]) + length.to_bytes(3, "big")


def stream(pcm, bps, rate, sizes=None, variable=False, total=None, blocks=b"", id3=0, *, first=0, max_bs=None,
           **frame_kw):
    """A whole FLAC file of the int (n, nch) pcm cut into blocks of `sizes` (default 4096).  blocks:
    metadata blocks after STREAMINFO (header bytes included, the last one flagged); id3: bytes of an
    ID3v2 tag body put in front; first: the first frame's number (fixed block size) or sample number
    (variable); max_bs: STREAMINFO's largest block size (None: the largest of `sizes`).  frame_kw goes to
    every frame; a callable value is called with the frame index."""
    pcm = np.asarray(pcm, np.int64)
    pcm = pcm if pcm.ndim == 2 else pcm.reshape(len(pcm), -1)
    n = len(pcm)
    if sizes is None:
        sizes = [4096] * (n // 4096) + ([n % 4096] if n % 4096 else [])
    assert sum(sizes) == n
    frames, pos = [], 0
    for k, bs in enumerate(sizes):
        kw = {key: (v(k) if callable(v) else v) for key, v in frame_kw.items()}
        frames.append(frame(pcm[pos:pos + bs], first + (pos if variable else k), bps, rate, variable, **kw))
        pos += bs
    top = max(sizes, default=0) if max_bs is None else max_bs
    out = b"fLaC" + streaminfo(min(sizes, default=0) if variable else top, top, rate, pcm.shape[1], bps,
                               n if total is None else total, last=not blocks) + blocks
    if id3:
        size = bytes([(id3 >> 21) & 127, (id3 >> 14) & 127, (id3 >> 7) & 127, id3 & 127])
        out = b"ID3\x04\x00\x00" + size + bytes(id3) + out
    return out + b"".join(frames), [len(f) for f in frames]
