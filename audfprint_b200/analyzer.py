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
import wave

import numpy as np

from . import _lib

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


def pcm_frontend(raw, channels, src_rate, dst_rate=None, device=None, to_host=True):
    """Interleaved int16 PCM -> mono float32 at dst_rate, on the device (afp_pcm_frontend:
    channel mean, 1/32768 scaling, polyphase resampling).  Returns a NumPy array, or with
    to_host=False a torch CUDA tensor that Analyzer.fingerprint_packed takes as it is."""
    from math import gcd
    raw = np.ascontiguousarray(raw, dtype=np.int16).reshape(-1)
    nframes = len(raw) // max(1, int(channels))
    up, down = 1, 1
    if dst_rate is not None and int(dst_rate) != int(src_rate):
        g = gcd(int(dst_rate), int(src_rate))
        up, down = int(dst_rate) // g, int(src_rate) // g
    taps = resample_taps(up, down) if (up, down) != (1, 1) else None
    ctx = _lib.context(device)
    nout = -(-nframes * up // down)
    n = C.c_int64(0)
    if to_host:
        out = np.empty(nout, np.float32)
        optr, on_host = out.ctypes.data, 1
    else:
        import torch
        out = torch.empty(nout, dtype=torch.float32, device=torch.device("cuda", ctx.device))
        optr, on_host = out.data_ptr(), 0
    ctx.check(ctx.lib.afp_pcm_frontend(ctx.h, raw.ctypes.data if nframes else None, 1, nframes, int(channels), up, down,
                                       taps.ctypes.data if taps is not None else None,
                                       len(taps) if taps is not None else 0, optr if nout else None, on_host,
                                       C.byref(n)))
    return out


def _wav_reader(filename, sr=None, channels=None, device=None):
    """PCM-WAV reader standing in for audio_read.audio_read (audio_read.py:56-68; ffmpeg decoding
    is out of scope, SURVEY §2 #9).  Returns (float32 samples in [-1,1), sr) like the reference
    reader does (audio_read.py:139-145).  The file is parsed on the host; the arithmetic the
    reference hands to ffmpeg - down-mix to mono, resampling to `sr` - runs on the device
    (afp_pcm_frontend, SURVEY.md 8f-2).  No two resamplers agree bit for bit, so parity statements
    in this repo are made on 11025 Hz PCM."""
    with wave.open(filename, 'rb') as w:
        nch, width, fs, n = w.getnchannels(), w.getsampwidth(), w.getframerate(), w.getnframes()
        if width != 2:
            raise IOError("only 16-bit PCM WAV is supported, got %d-byte samples" % width)
        raw = np.frombuffer(w.readframes(n), dtype='<i2')
    if nch == 1 and (sr is None or fs == sr):
        # nothing to do but the reader's own scaling (exact in float32)
        return raw.astype(np.float32) * np.float32(1.0 / 32768.0), fs
    data = pcm_frontend(raw, nch, fs, sr, device=device)
    return data, (fs if sr is None else sr)


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

    def __init__(self, density=DENSITY, device=None):
        self.density = density
        for attr, default in self._REFERENCE_DEFAULTS.items():
            setattr(self, attr, default)
        # not in the reference: which GPU, the pluggable file reader, and the arithmetic of the
        # spectrogram kernel: 'fp64' (default, results bit-identical to the reference) or 'fp32'
        # (opt-in: K1 at HBM speed, magnitudes within 1e-5, a few files per thousand differ)
        self.device = device
        self.precision = 'fp64'
        self.reader = _wav_reader

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
        if len(signals) == 0:
            return []
        nsh = max(1, int(self.shifts if shifts is None else shifts))
        frames = [nsh * (1 + len(x) // self.n_hop) for x in signals]
        if sum(frames) > self.max_frames_per_call and len(signals) > 1:
            out, start, acc = [], 0, 0
            for i, f in enumerate(frames):
                if acc + f > self.max_frames_per_call and i > start:
                    out += self.fingerprint_batch(signals[start:i], shifts)
                    start, acc = i, 0
                acc += f
            return out + self.fingerprint_batch(signals[start:], shifts)
        packed, starts, lens = self._pack(signals)
        rows, roff = self.fingerprint_packed(packed, starts, shifts, sample_lengths=lens)
        return [rows[roff[i]:roff[i + 1]] for i in range(len(signals))]

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
        counts, start, acc, pending = [], 0, 0, None
        frames = [nsh * (1 + len(x) // self.n_hop) for x in signals]
        for i in range(len(signals) + 1):
            if i == len(signals) or (acc + frames[i] > self.max_frames_per_call and i > start):
                if i > start:
                    packed, starts, lens = self._pack(signals[start:i])
                    self.fingerprint_packed(packed, starts, nsh, fetch=False, sample_lengths=lens)
                    # the host-side RNG replay of the previous call's overflow runs while the GPU
                    # fingerprints this one
                    counts += hashtable.store_batch_finish(pending)
                    pending = hashtable.store_batch_begin(names[start:i])
                start, acc = i, 0
            if i < len(signals):
                acc += frames[i]
        counts += hashtable.store_batch_finish(pending)
        for sig in signals:
            self._account(len(sig) / self.target_sr)
        return counts

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
            d, sr = self.reader(filename, sr=self.target_sr, channels=1)
        except Exception as e:
            message = "wavfile2peaks: Error reading " + filename
            if self.fail_on_error:
                print(e)
                raise IOError(message)
            print(message, "skipping")
            d, sr = [], self.target_sr
        return d, sr

    def _account(self, dur):
        self.soundfiledur = dur
        self.soundfiletotaldur += dur
        self.soundfilecount += 1

    def wavfile2peaks(self, filename, shifts=None):
        """Soundfile -> peaks, or list of peak lists when shifts > 1
        (audfprint_analyze.py:345-383)."""
        ext = os.path.splitext(filename)[1]
        if ext == PRECOMPPKEXT:
            peaks = peaks_load(filename)
            dur = np.max(peaks, axis=0)[0] * self.n_hop / self.target_sr
        else:
            d, sr = self._read(filename)
            dur = len(d) / sr
            if shifts is None or shifts < 2:
                peaks = self.find_peaks(d, sr)
            elif len(d) == 0:
                peaks = [[] for _ in range(shifts)]
            else:
                # NB the reference takes the offsets from self.shifts (:375)
                a, dtype = _as_pcm(d)
                ctx = self._configure(self.shifts)
                off = np.array([0, len(a)], np.int64)
                ctx.check(ctx.lib.afp_fingerprint_batch(ctx.h, a.ctypes.data, dtype, 1, 1,
                                                        off.ctypes.data_as(C.POINTER(C.c_int64)), None, None))
                peaks = [self._fetch_peaks(ctx, s, 1)[0] for s in range(min(shifts, self.shifts))]
        self._account(dur)
        return peaks

    def wavfile2hashes(self, filename):
        """Soundfile -> int32 (U,2) [time, hash] rows (audfprint_analyze.py:385-426)."""
        ext = os.path.splitext(filename)[1]
        if ext == PRECOMPEXT:
            hashes = hashes_load(filename)
            dur = np.max(hashes, axis=0)[0] * self.n_hop / self.target_sr
            self._account(dur)
            return hashes
        if ext == PRECOMPPKEXT:
            peaks = self.wavfile2peaks(filename, self.shifts)
            if len(peaks) == 0:
                return []
            rows = landmarks2hashes(self.peaks2landmarks(peaks))
            key = np.unique((rows[:, 0].astype(np.uint64) << np.uint64(32)) + rows[:, 1].astype(np.uint64))
            return np.stack([key >> np.uint64(32), key & np.uint64(0xFFFFFFFF)], axis=1).astype(np.int32)
        d, sr = self._read(filename)
        self._account(len(d) / sr)
        if len(d) == 0:
            return []
        hashes = self.fingerprint_batch([d], self.shifts)[0]
        if self.shifts < 2 and len(hashes) == 0:
            return []        # the reference returns [] when there are no peaks (:401-402)
        return hashes

    def ingest(self, hashtable, filename):
        """Read a file and add it to the table (audfprint_analyze.py:430-457)."""
        hashes = self.wavfile2hashes(filename)
        hashtable.store(filename, hashes)
        return self.soundfiledur, len(hashes)

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
