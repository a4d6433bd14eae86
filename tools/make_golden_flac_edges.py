"""Recipe of tests/golden/flac_edges.npz: small FLAC streams at the edges of the format, each with what
FFmpeg 8.0's decoder makes of it.

The streams come from the bit writer of tests/flac_writer.py (seeded PCM, explicit codes) and cover
every depth 4-24, channel counts 1-8, the three stereo decorrelations at every depth with full-scale
and odd negative sides, wasted bits on every subframe type, FIXED orders 0-4, every LPC order,
precision and shift with extreme coefficients, every Rice parameter and escape width of both methods,
partition orders up to 15, long unary runs, extreme residuals and FFmpeg's Rice quotient limit, every
block-size and sample-rate code, coded numbers across every length boundary, chain edges and one
damaged stream (CRCs right) per refusal rule.

For each stream `name`: name/flac (bytes), name/meta = [rate, channels, bps, status, ffmpeg samples,
written samples] (status: tests/flac_reference.py's; ffmpeg samples: interleaved int16 FFmpeg returned,
-1 when it stopped with an error, -2 for the 3- and 4-channel streams, see main(); written samples: interleaved, as the frames' block sizes say), and
name/pcm, FFmpeg's decode (oracle/ffdecode.py at the stream's rate and channels, s16), when status is 0.

    python tools/make_golden_flac_edges.py        (needs the opencv-python-headless wheel)
writes the same bytes each time.  Stores only data; nothing of FFmpeg is copied."""
from __future__ import annotations

import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import flac                 # noqa: E402
from tests import flac_reference as ref         # noqa: E402
from tests import flac_writer as fw             # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "flac_edges.npz")


def extremes(rng, n, nch, bps):
    """Seeded PCM (n, nch) at bps bits that visits both full-scale ends, -1, 0 and 1."""
    top = (1 << (bps - 1)) - 1
    x = rng.integers(-top - 1, top + 1, size=(n, nch))
    pat = np.array([top, -top - 1, -1, 0, 1, top, top, -top - 1, -top - 1])
    for c in range(nch):
        x[:len(pat), c] = np.roll(pat, c)[:n]
    x[-4:] = np.array([top, -top - 1, top, -top - 1])[:, None]
    return x


def cases():
    """(name, pcm, bps, rate, tests.flac_writer.stream keywords) of every stream, in order."""
    rng = np.random.default_rng(2026)
    out = []

    def add(name, pcm, bps, rate=11025, **kw):
        pcm = np.asarray(pcm, np.int64)
        out.append((name, pcm.reshape(-1, 1) if pcm.ndim == 1 else pcm, bps, rate, kw))

    # ---- depths, channel counts, decorrelation
    for b in range(4, 25):
        add("depth%d" % b, extremes(rng, 96, 1, b), b, sizes=[48, 48],
            specs=lambda k: [{"order": 2} if k == 0 else {"kind": "verbatim"}])
        if b in fw._SS:
            add("depth%d_ss0" % b, extremes(rng, 40, 1, b), b, sizes=[40], ss_code=0)
        top = (1 << (b - 1)) - 1
        lr = np.concatenate([[[top, -top - 1], [-top - 1, top], [-top - 1, 0], [0, top], [-3, 0], [-top, 2]],
                             extremes(rng, 58, 2, b)])
        for cm in (8, 9, 10):
            add("depth%d_chmode%d" % (b, cm), lr, b, sizes=[32, 32], chmode=cm,
                specs=lambda k: [{"order": 1}, {"kind": "verbatim" if k else "fixed", "order": 2}])
    for nch in range(1, 9):
        add("ch%d" % nch, extremes(rng, 80, nch, 16), 16, sizes=[40, 40])

    # ---- wasted bits: 1 .. sbps - 1 on every subframe type, the side channel's included
    for kind in ("constant", "verbatim", "fixed", "lpc"):
        frames = []
        for w in range(1, 16):
            v = rng.integers(-(1 << (15 - w)), 1 << (15 - w), size=32) << w
            frames.append(np.full(32, v[0]) if kind == "constant" else v)
        spec = {"kind": kind, "order": 2, "coefs": [1, 1, -1], "prec": 3, "shift": 0}
        add("wasted_" + kind, np.concatenate(frames), 16, sizes=[32] * 15,
            specs=lambda k, s=spec: [dict(s, wasted=k + 1)])
    left, right = [], []
    for w in range(1, 17):
        s = rng.integers(1 - (1 << (16 - w)), 1 << (16 - w), size=32) << w if w < 16 else np.zeros(32, np.int64)
        a = np.clip(rng.integers(-32768, 32768, size=32), -32768 + np.maximum(s, 0), 32767 + np.minimum(s, 0))
        left.append(a)
        right.append(a - s)
    for kind in ("verbatim", "fixed"):
        add("wasted_side_" + kind, np.stack([np.concatenate(left), np.concatenate(right)], 1), 16, sizes=[32] * 16,
            chmode=8, specs=lambda k, kd=kind: [{}, {"kind": kd, "order": 1, "wasted": k + 1}])
    # ---- FIXED orders 0-4 with bs == order, and a first partition with psize == order
    x = rng.integers(-3000, 3000, size=(2 + 3 + 4 + 64 + 64, 1))
    add("fixed_bs_eq_order", x, 16, sizes=[2, 3, 4, 64, 64], max_bs=64,
        specs=lambda k: [{"order": [2, 3, 4, 4, 1][k], "po": [0, 0, 0, 4, 6][k]}])
    for o in range(5):
        add("fixed_order%d" % o, extremes(rng, 64, 1, 16) >> 2, 16, sizes=[32, 32],
            specs=[{"order": o, "po": 1, "method": 1}])

    # ---- LPC: every order, precision and shift; extreme coefficients, 24-bit data, sums past 2^31
    combos = [(o, 1 + (o * 7) % 15, o % 16) for o in range(1, 33)]
    combos += [(1 + (p % 4), p, s) for p, s in zip(range(1, 16), range(15, 0, -1))]
    combos += [(2, 15, s) for s in range(16)]
    lpc_frames, lpc_specs = [], []
    for o, p, s in combos:
        c = [-(1 << (p - 1)) if j % 2 == 0 else (1 << (p - 1)) - 1 for j in range(o)]
        xx = extremes(rng, 64, 1, 24)[:, 0]
        while True:        # the residual must fit in 32 bits: halve the data until it does
            pred = np.array([sum(c[j] * int(xx[i - 1 - j]) for j in range(o)) >> s for i in range(o, 64)])
            if np.max(np.abs(xx[o:] - pred)) < (1 << 31) - 1:
                break
            xx = xx >> 1
        lpc_frames.append(xx)
        lpc_specs.append({"kind": "lpc", "coefs": c, "prec": p, "shift": s, "method": 1})
    for i in range(0, len(lpc_frames), 16):
        add("lpc_%d" % (i // 16), np.concatenate(lpc_frames[i:i + 16]), 24, sizes=[64] * len(lpc_frames[i:i + 16]),
            specs=lambda k, sp=lpc_specs[i:i + 16]: [sp[k]])

    # ---- Rice: every k of both methods, escape widths 0-31, partition orders 0-15, long unary runs
    for method, ks in ((0, range(15)), (1, range(31))):
        r = rng.integers(-40, 40, size=(32 * len(ks), 1))
        add("rice_m%d" % method, r, 24, sizes=[32] * len(ks),
            specs=lambda k, m=method: [{"order": 0, "method": m, "po": 1, "rice": [k, 0]}])
    for method in (0, 1):
        frames = []
        for w in range(32):
            frames.append(rng.integers(-(1 << max(w - 1, 0)), 1 << max(w - 1, 0), size=32) if w else np.zeros(32, int))
        add("escape_m%d" % method, np.concatenate(frames).reshape(-1, 1), 24, sizes=[32] * 32,
            specs=lambda k, m=method: [{"order": 0, "method": m, "po": 0, "escape": (0,), "esc_width": k}])
    saw = (np.arange(2 ** 17, dtype=np.int64) * 5) % 251 - 125
    sizes = [2 << p for p in range(15)] + [32768]
    add("partition_orders", saw[:sum(sizes)], 8, sizes=sizes, specs=lambda k: [{"order": 1, "po": k, "method": k % 2}])
    big = rng.integers(-200, 200, size=(256, 1))
    big[::7] = 40
    add("unary_long", big, 16, sizes=[128, 128], specs=[{"order": 0, "rice": [0]}])
    for name, v in (("residual_min_plus1", -(1 << 31) + 1), ("residual_max", (1 << 31) - 1),
                    ("residual_min", -(1 << 31))):
        x = rng.integers(-100, 100, size=(96, 1))
        add(name, x, 24, sizes=[32, 32, 32], specs=lambda k, v=v: [
            {"order": 0, "method": 1, "raw": np.r_[x[32:64, 0][:5], v, x[32:64, 0][6:]]} if k == 1 else {}])
    for k, q in ((14, 1 << 18), (14, (1 << 18) + 1), (30, 4), (30, 5), (20, 4095)):
        u = q << k
        raw = np.zeros(32, np.int64)
        raw[3] = u >> 1 if u % 2 == 0 else -((u + 1) >> 1)
        raw[9] = 5
        add("quotient_k%d_q%d" % (k, q), np.zeros((96, 1), np.int64), 16, sizes=[32, 32, 32],
            specs=lambda f, raw=raw, k=k: [{"order": 0, "method": 1, "rice": [k], "raw": raw} if f == 1 else {}])

    # ---- header codes
    std_bs = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, **{c: 256 << (c - 8) for c in range(8, 16)}}
    for code, bs in std_bs.items():
        add("bs_code%d" % code, saw[:bs + 16], 8, sizes=[bs, 16], max_bs=bs, specs=[{"order": 1, "po": 0}])
    for code, vals in ((6, (1, 2, 256)), (7, (1, 256, 65535))):
        for v in vals:
            add("bs%d_%d" % (code, v), saw[:v + min(v, 16)], 8, sizes=[v, min(v, 16)], bs_code=code, max_bs=max(v, 16),
                specs=[{"kind": "verbatim"}] if v < 4 else [{"order": 1}])
    rates = {0: 11025, 1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100,
             10: 48000, 11: 96000, 12: 255000, 13: 65535, 14: 655350}
    for code, rate in rates.items():
        add("sr_code%d" % code, extremes(rng, 64, 1, 16), 16, rate, sizes=[32, 32], sr_code=code)
    # coded numbers: fixed-mode files of 130 and 2050 frames, then first numbers at each length boundary
    add("frames130", saw[:130 * 16], 8, sizes=[16] * 130, specs=[{"order": 1}])
    add("frames2050", np.repeat(saw[:2050], 16)[:2050 * 16], 8, sizes=[16] * 2050, specs=[{"kind": "constant"}])
    for bits in (16, 21, 26, 31):
        top = bits == 31           # the last frame's number stays below 2^31
        add("fixed_first_2^%d" % bits, saw[:64], 8, sizes=[16] * 4, first=(1 << bits) - 2 - 2 * top)
        add("variable_first_2^%d" % bits, saw[:64], 8, sizes=[16] * 4, variable=True, first=(1 << bits) - 32 - 32 * top)
    add("variable_first_0", saw[:64], 8, sizes=[16, 16, 32], variable=True)
    add("variable_first_2^11", saw[:64], 8, sizes=[16] * 4, variable=True, first=(1 << 11) - 32)
    add("variable_first_2^36", saw[:64], 8, sizes=[16] * 4, variable=True, first=(1 << 36) - 64)

    # ---- chain edges
    for pos in (1, 100, 250):
        p8 = rng.integers(-128, 128, size=(768, 1))
        hdr = fw.frame(np.zeros((256, 1), np.int64), 1, 8, 11025)[:6]    # frame 1's header, inside frame 0
        p8[pos:pos + 6, 0] = np.frombuffer(hdr, np.uint8).astype(np.int8)
        add("planted_%d" % pos, p8, 8, sizes=[256] * 3, specs=[{"kind": "verbatim"}])
    for t in range(1, 6):
        tail = b"\xff\xf8\x69\x08\x00"[:t]
        add("tail%d" % t, saw[:64], 8, sizes=[32, 32], tail=lambda k, tail=tail: tail if k else b"")
    add("one_frame", saw[:100], 8, sizes=[100])
    add("empty", np.zeros((0, 2), np.int64), 16, sizes=[])

    # ---- damaged streams with right CRCs, one per refusal rule
    y = rng.integers(-500, 500, size=(96, 1))

    plain = {"bs_code": None, "sr_code": None, "ss_code": None, "reserved": 0, "tail": b"", "specs": [{}]}

    def damaged(name, **kw):
        """Frame 1 of 3 carries the damage."""
        add(name, y, 16, sizes=[32, 32, 32], **{k: (lambda f, k=k, v=v: v if f == 1 else plain[k]) for k, v in kw.items()})
    damaged("bad_bs_code0", bs_code=0)
    damaged("bad_sr_code15", sr_code=15)
    damaged("bad_ss_code3", ss_code=3)
    damaged("bad_reserved_bit", reserved=1)
    for t in list(range(2, 8)) + list(range(13, 32)):
        damaged("bad_type%d" % t, specs=[{"sub_type": t}])
    damaged("bad_prec15", specs=[{"kind": "lpc", "coefs": [1], "prec": 4, "shift": 0, "prec_code": 15}])
    damaged("bad_shift_neg", specs=[{"kind": "lpc", "coefs": [1], "prec": 4, "shift": -1, "raw": np.zeros(31, int)}])
    damaged("bad_method2", specs=[{"method": 2}])
    damaged("bad_method3", specs=[{"method": 3}])
    add("bad_po_remainder", y[:30], 16, sizes=[20, 10], specs=lambda f: [{"order": 0, "po": 2 if f else 0}])
    damaged("bad_order_psize", specs=[{"order": 4, "po": 4}])
    damaged("bad_pad", specs=[{"pad": 1}])
    add("bad_wasted_eq_sbps", np.r_[y[:32], 0 * y[:32], y[64:]], 16, sizes=[32] * 3,
        specs=lambda f: [{"kind": "constant", "wasted": 16} if f == 1 else {}])
    damaged("bad_run_past", specs=[{"kind": "verbatim"}])
    return out


def build(name, pcm, bps, rate, kw):
    """The stream's bytes.  bad_run_past: frame 1 loses the last 3 bytes of its subframe data, CRC-16
    recomputed, so the data runs past the frame."""
    data, lens = fw.stream(pcm, bps, rate, **kw)
    if name == "bad_run_past":
        f1 = len(data) - sum(lens) + lens[0]
        body = data[f1:f1 + lens[1] - 2][:-3]
        data = data[:f1] + body + fw.crc16(body).to_bytes(2, "big") + data[f1 + lens[1]:]
    return data


def bad_ch_code():
    """A stereo stream whose frame 1 has channel code 11 (reserved), CRC-8 and CRC-16 right."""
    y = np.random.default_rng(11).integers(-500, 500, size=(96, 2))
    data, lens = fw.stream(y, 16, 11025, sizes=[32] * 3)
    f1 = len(data) - sum(lens) + lens[0]
    fr = bytearray(data[f1:f1 + lens[1]])
    fr[3] = (11 << 4) | (fr[3] & 15)
    fr[5] = fw.crc8(fr[:5])
    fr[-2:] = fw.crc16(fr[:-2]).to_bytes(2, "big")
    return data[:f1] + bytes(fr) + data[f1 + lens[1]:]


def streams():
    """[(name, bytes, rate, channels, bps, written samples)]."""
    out = []
    for name, pcm, bps, rate, kw in cases():
        out.append((name, build(name, pcm, bps, rate, kw), rate, pcm.shape[1], bps, pcm.size))
    out.append(("bad_ch_code11", bad_ch_code(), 11025, 2, 16, 192))
    return out


def save(path, arrays):
    """np.savez_compressed with fixed zip timestamps, so that the same arrays give the same bytes."""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            b = io.BytesIO()
            np.lib.format.write_array(b, np.asanyarray(v), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", (1980, 1, 1, 0, 0, 0)), b.getvalue(), zipfile.ZIP_DEFLATED)
    with open(path, "wb") as f:
        f.write(buf.getvalue())


def main():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from make_golden_flac import ff_decode
    out, names = {}, []
    for name, data, rate, nch, bps, written in streams():
        pcm, status = ref.decode(flac.parse(data))
        try:
            got = ff_decode(data, rate, nch)
            nff = len(got)
        except IOError:
            got, nff = None, -1
        if nch in (3, 4):
            # FFmpeg's default 3- and 4-channel layouts are not FLAC's, so its s16 output is a remix:
            # these two store the reference's decode, which the 1-2 and 5-8 channel streams pin to FFmpeg
            got, nff = pcm, -2
        if status == 0:
            if written == 0:       # no frames: FFmpeg finds no audio stream, the reference no samples
                got = pcm
            assert nff in (written, -2) and np.array_equal(got, pcm) or written == 0, name
            out[name + "/pcm"] = got
        out[name + "/flac"] = np.frombuffer(data, np.uint8)
        out[name + "/meta"] = np.array([rate, nch, bps, status, nff, written], np.int64)
        names.append(name)
    out["names"] = np.array(names)
    save(OUT, out)
    print("wrote", OUT, len(names), "streams,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
