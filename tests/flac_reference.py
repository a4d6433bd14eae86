"""A sequential integer FLAC decoder: the statement the device decoder (csrc/afp_flac.cu) is held to.

Written from the format (RFC 9639) and from what FFmpeg 8.0's decoder does with streams whose CRCs are
right: whatever FFmpeg refuses in such a frame (and so drops, where the file is then unreadable here,
DESIGN section 8), this decoder refuses too.  All arithmetic is on Python ints; a subframe's samples are
32-bit words, as in every decoder, so they wrap to int32.

decode(stream) -> (interleaved int16 samples, status), with the device's AFP_FLAC_* codes.  A Record
passed in collects which constructs were decoded, so that a corpus can show it reaches every edge.

Frames are delimited as the device delimits them (DESIGN section 5): a frame runs from its header to the
next header that is consistent with STREAMINFO, has a right CRC-8 and a number that follows on, at which
the CRC-16 of the frame's bytes is 0.  Statuses where no frame decodes:
  CHAIN      no header at byte 0; or at a point where the CRC-16 is 0, a header that does not follow on;
             or the file ends with a CRC-16 that is not 0 after passing a header that did not follow on;
  CRC        the file ends with a CRC-16 that is not 0 after passing a header that follows on;
  RESERVED   a reserved code in the first header, or in a header (right CRC-8) where the CRC-16 is 0;
  TRUNCATED  the file ends with a CRC-16 that is not 0 and no header was passed in the last frame;
and in a frame's subframes RESERVED (padding bit, subframe type, LPC precision code 15, residual method)
or CORRUPT (everything else FFmpeg refuses, and data that runs past the frame)."""
from __future__ import annotations

from collections import defaultdict

import numpy as np

OK, DEPTH, CHAIN, CRC, RESERVED, TRUNCATED, CORRUPT = range(7)

_BS = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, **{c: 256 << (c - 8) for c in range(8, 16)}}
_SR = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000,
       11: 96000}
_SS = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}
INT_MAX = (1 << 31) - 1


class Record(object):
    """Decoded constructs: axis name -> set of values seen."""

    def __init__(self):
        self.seen = defaultdict(set)

    def add(self, axis, value):
        self.seen[axis].add(value)


class _NoRecord(object):
    def add(self, axis, value):
        pass


class Refused(Exception):
    def __init__(self, status, why):
        Exception.__init__(self, why)
        self.status = status


def _crc8(data):
    c = 0
    for b in data:
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
    return c


def _crc16_table():
    t = []
    for i in range(256):
        c = i << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
        t.append(c)
    return t


_T16 = _crc16_table()


def _crc16(c, data):
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _T16[(c >> 8) ^ b]
    return c


def _wrap32(v):
    return ((v + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def header(data, pos, s):
    """The frame header at data[pos:] against FlacStream s -> ("ok", fields), ("reserved", None) when
    its CRC-8 is right but a code is reserved, or ("none", None)."""
    n = len(data)
    if n - pos < 6 or data[pos] != 0xFF or data[pos + 1] & 0xFE != 0xF8:
        return "none", None
    variable = data[pos + 1] & 1
    bs_code, sr_code = data[pos + 2] >> 4, data[pos + 2] & 15
    ch_code, ss_code, bit = data[pos + 3] >> 4, (data[pos + 3] >> 1) & 7, data[pos + 3] & 1
    q = pos + 4
    # UTF-8-style coded number; FFmpeg's reader takes lead bytes up to 0xFD (6 bytes, 31 bits)
    lead = data[q]
    if lead < 0x80:
        extra, v = 0, lead
    else:
        extra = next((e for e in range(1, 6) if lead >> (6 - e) == (0xFF >> (6 - e)) - 1), None)
        if extra is None:
            return "none", None
        v = lead & ((1 << (6 - extra)) - 1)
    q += 1
    if n - q < extra + 1:
        return "none", None
    for b in data[q:q + extra]:
        if b & 0xC0 != 0x80:
            return "none", None
        v = (v << 6) | (b & 0x3F)
    q += extra
    if bs_code == 6:
        if n - q < 2:
            return "none", None
        bs = data[q] + 1
        q += 1
    elif bs_code == 7:
        if n - q < 3:
            return "none", None
        bs = (data[q] << 8 | data[q + 1]) + 1
        q += 2
    else:
        bs = _BS.get(bs_code, 0)
    rate = _SR.get(sr_code, s.sample_rate)
    width = {12: 1, 13: 2, 14: 2}.get(sr_code, 0)
    if width:
        if n - q < width + 1:
            return "none", None
        raw = int.from_bytes(data[q:q + width], "big")
        rate = raw * 1000 if sr_code == 12 else raw * 10 if sr_code == 14 else raw
        q += width
    if n - q < 1 or _crc8(data[pos:q]) != data[q]:
        return "none", None
    if bs_code == 0 or sr_code == 15 or ch_code > 10 or ss_code == 3 or bit or bs > 65535:
        return "reserved", None
    bps = _SS.get(ss_code, s.bits_per_sample)
    nch = ch_code + 1 if ch_code < 8 else 2
    if bps != s.bits_per_sample or nch != s.channels or rate != s.sample_rate or \
            (s.max_blocksize >= 16 and bs > s.max_blocksize):
        return "none", None
    return "ok", dict(variable=variable, number=v, bs=bs, chmode=ch_code, nbytes=q + 1 - pos, bs_code=bs_code,
                      sr_code=sr_code, ss_code=ss_code, numlen=extra + 1)


def frames(data, s):
    """[(start, end, header fields)] of the frames of FlacStream s's bytes; raises Refused."""
    n = len(data)
    kind, h = header(data, 0, s)
    if kind != "ok":
        raise Refused(RESERVED if kind == "reserved" else CHAIN, "no frame at the start")
    a = np.frombuffer(data, np.uint8)
    sync = np.flatnonzero((a[:-1] == 0xFF) & (a[1:] & 0xFE == 0xF8)) if n > 1 else []
    out, start, crc, last = [], 0, 0, 0
    seen = passed = False
    for p in sync:
        p = int(p)
        if p == 0:
            continue
        kind, g = header(data, p, s)
        if kind == "none":
            continue
        crc = _crc16(crc, data[last:p])
        last = p
        if kind == "reserved":
            if crc == 0:
                raise Refused(RESERVED, "reserved code in the header at %d" % p)
            continue
        follows = g["variable"] == h["variable"] and g["number"] == h["number"] + (h["bs"] if h["variable"] else 1)
        passed = True
        if crc == 0:
            if not follows:
                raise Refused(CHAIN, "header at %d does not follow on" % p)
            out.append((start, p, h))
            start, h, crc = p, g, 0
            seen = passed = False
        elif follows:
            seen = True
    if _crc16(crc, data[last:]) != 0:
        raise Refused(CRC if seen else CHAIN if passed else TRUNCATED, "last frame does not end in its CRC-16")
    out.append((start, n, h))
    return out


class Bits(object):
    """MSB-first reader of bits [8 * lo, 8 * hi) of data; a read past the end refuses the frame."""

    def __init__(self, data, lo, hi):
        self.b = np.unpackbits(np.frombuffer(data[lo:hi], np.uint8)).tobytes().translate(_ASCII).decode()
        self.pos = 0

    def u(self, n):
        if self.pos + n > len(self.b):
            raise Refused(CORRUPT, "subframe data runs past the frame")
        self.pos += n
        return int(self.b[self.pos - n:self.pos], 2) if n else 0

    def s(self, n):
        x = self.u(n)
        return x - (1 << n) if n and x >> (n - 1) else x

    def unary(self):
        one = self.b.find("1", self.pos)
        if one < 0:
            raise Refused(CORRUPT, "unary code runs past the frame")
        q = one - self.pos
        self.pos = one + 1
        return q


_ASCII = bytes.maketrans(b"\x00\x01", b"01")


def residual(br, bs, order, rec):
    method = br.u(2)
    if method > 1:
        raise Refused(RESERVED, "residual method %d" % method)
    po = br.u(4)
    psize = bs >> po
    if psize << po != bs:
        raise Refused(CORRUPT, "partition order %d does not divide %d" % (po, bs))
    if order > psize:
        raise Refused(CORRUPT, "order %d above the partition size %d" % (order, psize))
    rec.add("po", po)
    if order == psize:
        rec.add("first_partition_empty", order)
    kbits = 5 if method else 4
    out = []
    for part in range(1 << po):
        k = br.u(kbits)
        n = psize - (order if part == 0 else 0)
        if k == (1 << kbits) - 1:
            nb = br.u(5)
            rec.add("escape%d" % method, nb)
            out += [br.s(nb) for _ in range(n)]
            continue
        rec.add("rice%d" % method, k)
        # FFmpeg's Rice reader: a quotient of `limit` is refused, one of limit - 1 is followed by a single
        # bit b and means u = b + 1, and u = 2^32 - 1 (residual -2^31) is refused
        limit = (INT_MAX >> (k - 1)) + 2 if k > 1 else INT_MAX
        for _ in range(n):
            q = br.unary()
            if q > 57:
                rec.add("unary_long", min(q, 65))
            if q >= limit:
                raise Refused(CORRUPT, "Rice quotient %d at k=%d" % (q, k))
            if q == limit - 1:
                rec.add("quotient_limit", k)
                u = br.u(1) + 1
            else:
                u = (q << k) | br.u(k)
            if u == 0xFFFFFFFF:
                raise Refused(CORRUPT, "residual -2^31")
            v = (u >> 1) ^ -(u & 1)
            if v in (-INT_MAX, INT_MAX):
                rec.add("residual_extreme", v)
            out.append(v)
    return out


def subframe(br, bs, sbps, rec):
    """One subframe's bs samples at sbps bits (int32 words)."""
    if br.u(1):
        raise Refused(RESERVED, "subframe padding bit")
    typ = br.u(6)
    wasted = 0
    if br.u(1):
        wasted = br.unary() + 1
        if wasted >= sbps:
            raise Refused(CORRUPT, "%d wasted bits of %d" % (wasted, sbps))
        rec.add("wasted", (sbps, wasted))
    b = sbps - wasted
    if typ == 0:
        rec.add("subframe", ("constant", 0))
        x = [br.s(b)] * bs
    elif typ == 1:
        rec.add("subframe", ("verbatim", 0))
        x = [br.s(b) for _ in range(bs)]
    elif 8 <= typ <= 12:
        order = typ - 8
        if order > bs:
            raise Refused(CORRUPT, "FIXED order above the block size")
        rec.add("subframe", ("fixed", order))
        if order == bs:
            rec.add("fixed_bs_eq_order", order)
        x = [br.s(b) for _ in range(order)]
        x += residual(br, bs, order, rec)
        # the order-th difference of the signal is the residual: undo it with binomial weights
        w = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}[order]
        for i in range(order, bs):
            x[i] = _wrap32(x[i] + sum(c * x[i - 1 - j] for j, c in enumerate(w)))
    elif typ >= 32:
        order = typ - 31
        if order > bs:
            raise Refused(CORRUPT, "LPC order above the block size")
        x = [br.s(b) for _ in range(order)]
        pc = br.u(4)
        if pc == 15:
            raise Refused(RESERVED, "LPC precision code 15")
        shift = br.s(5)
        if shift < 0:
            raise Refused(CORRUPT, "negative LPC shift")
        coef = [br.s(pc + 1) for _ in range(order)]
        rec.add("subframe", ("lpc", order))
        rec.add("prec", pc + 1)
        rec.add("shift", shift)
        if any(c == -(1 << pc) for c in coef):
            rec.add("coef_min", pc + 1)
        x += residual(br, bs, order, rec)
        for i in range(order, bs):
            acc = sum(c * x[i - 1 - j] for j, c in enumerate(coef))
            if abs(acc) >= 1 << 31:
                rec.add("lpc_sum_wide", True)
            x[i] = _wrap32(x[i] + (acc >> shift))
    else:
        raise Refused(RESERVED, "subframe type %d" % typ)
    return [_wrap32(v << wasted) for v in x]


def _to_int16(v, bps):
    v = v << (16 - bps) if bps <= 16 else v >> (bps - 16)
    return ((v + 32768) & 0xFFFF) - 32768


def decode_frame(data, lo, hi, h, s, rec):
    """One frame's samples, interleaved int16 (a list)."""
    bps, bs, nch, cm = s.bits_per_sample, h["bs"], s.channels, h["chmode"]
    br = Bits(data, lo + h["nbytes"], hi - 2)
    chans = []
    for c in range(nch):
        side = (cm == 8 and c == 1) or (cm == 9 and c == 0) or (cm == 10 and c == 1)
        if side:
            rec.add("side_depth", bps + 1)
        chans.append(subframe(br, bs, bps + side, rec))
    if cm == 8:                     # left, side
        chans[1] = [_wrap32(a - d) for a, d in zip(*chans)]
    elif cm == 9:                   # side, right
        chans[0] = [_wrap32(d + b) for d, b in zip(*chans)]
    elif cm == 10:                  # mid, side: right = mid - side / 2 (floor), left = right + side
        right = [_wrap32(m - (d >> 1)) for m, d in zip(*chans)]
        chans = [[_wrap32(r + d) for r, d in zip(right, chans[1])], right]
    out = [0] * (bs * nch)
    for c in range(nch):
        out[c::nch] = [_to_int16(v, bps) for v in chans[c]]
    return out


def decode(s, rec=None):
    """FlacStream s (audfprint_b200.flac.parse) -> (int16 interleaved samples, AFP_FLAC_* status)."""
    rec = rec or _NoRecord()
    empty = np.zeros(0, np.int16)
    if not 4 <= s.bits_per_sample <= 24:
        return empty, DEPTH
    data = np.asarray(s.frames, np.uint8).tobytes()
    if len(data) == 0:
        return empty, OK
    try:
        spans = frames(data, s)
        out = []
        for lo, hi, h in spans:
            rec.add("bs_code", h["bs_code"])
            rec.add("sr_code", h["sr_code"])
            rec.add("ss_code", (h["ss_code"], s.bits_per_sample))
            rec.add("numlen", ("variable" if h["variable"] else "fixed", h["numlen"]))
            if h["bs_code"] in (6, 7):
                rec.add("bs%d" % h["bs_code"], h["bs"])
            rec.add("chmode", h["chmode"])
            out += decode_frame(data, lo, hi, h, s, rec)
    except Refused as e:
        rec.add("refused", e.status)
        return empty, e.status
    rec.add("depth", s.bits_per_sample)
    rec.add("frames", min(len(spans), 1 << 17).bit_length())
    return np.asarray(out, np.int16), OK
