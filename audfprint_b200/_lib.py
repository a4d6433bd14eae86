"""ctypes binding of libafp.so (include/afp.h).  There is no CPU fallback: if
the library is missing or no CUDA device is present every call fails loudly."""
from __future__ import annotations

import contextlib
import ctypes as C
import os
import re
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libafp.so")
HEADER = os.path.join(os.path.dirname(_HERE), "include", "afp.h")

PCM_I16, PCM_F32, PCM_S24, PCM_S32 = 0, 1, 2, 3


class AfpError(RuntimeError):
    pass


class RowCapacityError(AfpError):
    """afp_match_batch: a query produced more rows than row_capacity (retry with more)."""


class AnalyzerParams(C.Structure):
    _fields_ = [("a_dec", C.c_double), ("hpf_pole", C.c_double), ("maxpksperframe", C.c_int32),
                ("maxpairsperpeak", C.c_int32), ("targetdf", C.c_int32), ("mindt", C.c_int32),
                ("targetdt", C.c_int32), ("shifts", C.c_int32), ("spectrogram_fp32", C.c_int32)]


class MatcherParams(C.Structure):
    _fields_ = [("window", C.c_int32), ("threshcount", C.c_int32), ("search_depth", C.c_int32),
                ("max_alignments_per_id", C.c_int32), ("publish_candidates", C.c_int32),
                ("row_capacity", C.c_int32), ("force_general", C.c_int32)]


class FlacStream(C.Structure):
    _fields_ = [("byte_offset", C.c_int64), ("nbytes", C.c_int64), ("sample_rate", C.c_int32),
                ("channels", C.c_int32), ("bits_per_sample", C.c_int32), ("max_blocksize", C.c_int32)]


_P = C.c_void_p
_I64P = C.POINTER(C.c_int64)
_SIGS = {
    "afp_abi_version": (C.c_int, []),
    "afp_create": (C.c_int, [C.POINTER(_P), C.c_int]),
    "afp_destroy": (None, [_P]),
    "afp_last_error": (C.c_char_p, [_P]),
    "afp_set_stream": (C.c_int, [_P, _P]),
    "afp_get_stream": (C.c_int, [_P, C.POINTER(_P)]),
    "afp_sync": (C.c_int, [_P]),
    "afp_launch_count": (C.c_int64, [_P]),
    "afp_set_profiling": (C.c_int, [_P, C.c_int]),
    "afp_get_stage_ms": (C.c_int, [_P, C.POINTER(C.c_float)]),
    "afp_pcm_frontend": (C.c_int, [_P, _P, C.c_int, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int32, _P,
                                   C.c_int, _I64P]),
    "afp_pcm_frontend_batch": (C.c_int, [_P, _P, C.c_int, C.c_int64, C.c_int32, _I64P, _I64P, _P, _P, _P, C.c_int32,
                                         _P, _I64P, _P, _P, C.c_int64, _I64P, _I64P]),
    "afp_pcm_frontend_batch_bytes": (C.c_int, [_P, _P, C.c_int, C.c_int64, C.c_int32, _I64P, _P, _I64P, _P, _P, _P,
                                               C.c_int32, _P, _I64P, _P, _P, C.c_int64, _I64P, _I64P]),
    "afp_swr_design": (C.c_int, [C.c_int32, C.c_int32, _P, C.c_int64, _P, _P]),
    "afp_swr_length": (C.c_int, [C.c_int64, C.c_int32, C.c_int32, _I64P]),
    "afp_swr_frontend_batch": (C.c_int, [_P, _P, C.c_int, C.c_int64, C.c_int32, _I64P, _I64P, _P, _P, C.c_int32, _P,
                                         C.c_int64, _I64P, _I64P]),
    "afp_swr_frontend_batch_bytes": (C.c_int, [_P, _P, C.c_int, C.c_int64, C.c_int32, _I64P, _P, _I64P, _P, _P,
                                               C.c_int32, _P, C.c_int64, _I64P, _I64P]),
    "afp_flac_locate_batch": (C.c_int, [_P, _P, C.c_int, C.c_int64, C.c_int32, C.POINTER(FlacStream), _I64P, _P]),
    "afp_flac_decode_batch": (C.c_int, [_P, _P, C.c_int64, _I64P, _P]),
    "afp_flac_decode_batch_bytes": (C.c_int, [_P, _P, C.c_int64, _I64P, C.c_int32, _P]),
    "afp_set_analyzer": (C.c_int, [_P, C.POINTER(AnalyzerParams), _P, _P, C.c_double]),
    "afp_fingerprint_batch": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int32, _I64P, _I64P, _I64P]),
    "afp_fetch_hashes": (C.c_int, [_P, _P, C.c_int, _I64P]),
    "afp_fetch_peaks": (C.c_int, [_P, C.c_int32, _P, C.c_int, _I64P]),
    "afp_landmarks_from_peaks": (C.c_int, [_P, _P, C.c_int64, C.c_int, _I64P]),
    "afp_fetch_landmarks": (C.c_int, [_P, _P, C.c_int]),
    "afp_fingerprint_from_peaks": (C.c_int, [_P, _P, C.c_int, C.c_int32, _I64P, _P, _I64P]),
    "afp_spread_peaks": (C.c_int, [_P, _P, C.c_int32, _P, C.c_double, _P, _P]),
    "afp_stft_mag": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int64, _P, C.c_int]),
    "afp_sgram": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int64, _P, C.c_int]),
    "afp_fingerprint_from_logs": (C.c_int, [_P, _P, C.c_int, C.c_int32, _P, _P, _I64P]),
    "afp_table_upload": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int]),
    "afp_table_create": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_int32]),
    "afp_table_set_hashesperid": (C.c_int, [_P, _P, C.c_int64]),
    "afp_table_store_batch": (C.c_int, [_P, _P, C.c_int, _I64P, C.c_int32, _I64P, _I64P]),
    "afp_table_fetch_overflow": (C.c_int, [_P, _P, _P, _P]),
    "afp_table_apply_patches": (C.c_int, [_P, _P, _P, _P, C.c_int64]),
    "afp_table_fetch_overflow_counts": (C.c_int, [_P, _P]),
    "afp_table_apply_slots": (C.c_int, [_P, _P, C.c_int64]),
    "afp_table_download": (C.c_int, [_P, _P, _P]),
    "afp_mt_randint_replay": (C.c_int, [_P, _P, C.c_int64, _P]),
    "afp_table_restrict_ids": (C.c_int, [_P, C.c_int64, C.c_int64]),
    "afp_table_remove_ids": (C.c_int, [_P, _I64P, C.c_int64, _I64P]),
    "afp_table_retrieve_ids": (C.c_int, [_P, _I64P, C.c_int64, _I64P]),
    "afp_fetch_retrieved": (C.c_int, [_P, _P, C.c_int, _I64P]),
    "afp_table_merge": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, C.c_int64, _P, _I64P, _P]),
    "afp_table_merge_device": (C.c_int, [_P, _P, _P, C.c_int32, C.c_int32, C.c_int64, _P, _I64P, _P]),
    "afp_table_export": (C.c_int, [_P, _P, _P]),
    "afp_np_permutation_replay": (C.c_int, [_P, _P, C.c_int64, C.c_int32, _P]),
    "afp_table_pruning_bound": (C.c_int, [_P, C.POINTER(C.c_uint32)]),
    "afp_get_hits": (C.c_int, [_P, _P, C.c_int64, C.c_int, _I64P]),
    "afp_fetch_hits": (C.c_int, [_P, _P, C.c_int]),
    "afp_match_batch": (C.c_int, [_P, _P, C.c_int, C.c_int32, _I64P, C.POINTER(MatcherParams), _I64P]),
    "afp_fetch_match_rows": (C.c_int, [_P, _P, C.c_int, _I64P]),
    "afp_match_general_count": (C.c_int, [_P, _I64P]),
    "afp_fetch_match_status": (C.c_int, [_P, _P]),
    "afp_shard_record_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "afp_shard_pack": (C.c_int, [_P, C.c_int32, _P]),
    "afp_shard_merge": (C.c_int, [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _I64P]),
    "afp_fetch_match_candidates": (C.c_int, [_P, _P, _P, C.c_int]),
    "afp_match_options_batch": (C.c_int, [_P, _P, C.c_int, C.c_int32, _I64P, C.POINTER(MatcherParams), C.c_int32,
                                          C.c_int32, C.c_double, _I64P, _I64P]),
    "afp_match_options_shard_rank": (C.c_int, [_P, _P, C.c_int, C.c_int32, _I64P, C.POINTER(MatcherParams),
                                               C.c_int32, C.c_int32, C.c_double, _I64P, _P, _I64P]),
    "afp_match_options_shard_finish": (C.c_int, [_P, _P, _I64P]),
}

_lib = None
_lock = threading.Lock()


def header_symbols():
    """Function names declared in include/afp.h."""
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(afp_[a-z0-9_]+)\s*\(", txt)))


def load(check_symbols: bool = False):
    """dlopen the in-tree libafp.so (built by __graft_entry__.build())."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise AfpError("libafp.so is not built (%s); run `python __graft_entry__.py`. "
                               "There is no CPU fallback." % LIB_PATH)
            lib = C.CDLL(LIB_PATH)
            for name, (res, args) in _SIGS.items():
                fn = getattr(lib, name)
                fn.restype = res
                fn.argtypes = args
            _lib = lib
    if check_symbols:
        missing = [s for s in header_symbols() if not hasattr(_lib, s)]
        if missing:
            raise AfpError("libafp.so does not export: " + ", ".join(missing))
        unbound = [s for s in header_symbols() if s not in _SIGS]
        if unbound:
            raise AfpError("no ctypes signature for: " + ", ".join(unbound))
    return _lib


def ptr_of(x):
    """(address, on_host) of a numpy array (host) or a torch CUDA/CPU tensor."""
    if x is None:
        return None, 1
    if isinstance(x, np.ndarray):
        if not x.flags["C_CONTIGUOUS"]:
            raise AfpError("array must be C-contiguous")
        return x.ctypes.data, 1
    if hasattr(x, "data_ptr"):      # torch tensor, used as a raw device/pinned buffer only
        if not x.is_contiguous():
            raise AfpError("tensor must be contiguous")
        return x.data_ptr(), 0 if x.is_cuda else 1
    raise AfpError("unsupported buffer type %r" % type(x))


def pack_rows(arrays):
    """A list of (n_i, 2) int32 arrays -> (rows int32 (sum n_i, 2) contiguous, offsets int64 [len + 1])."""
    arrs = [np.asarray(a, dtype=np.int32).reshape(-1, 2) for a in arrays]
    off = np.zeros(len(arrs) + 1, np.int64)
    off[1:] = np.cumsum([len(a) for a in arrs])
    rows = np.ascontiguousarray(np.concatenate(arrs)) if arrs else np.zeros((0, 2), np.int32)
    return rows, off


class Context:
    """One afp_ctx (one per process per GPU)."""

    def __init__(self, device: int = 0):
        self.lib = load()
        h = _P()
        rc = self.lib.afp_create(C.byref(h), int(device))
        if rc != 0:
            raise AfpError("afp_create(device=%d) failed with status %d: a CUDA device is required "
                           "(no CPU fallback)" % (device, rc))
        self.h = h
        self.device = device
        self.analyzer_key = None
        self.table_key = None
        self.table_owner = None      # weakref to the HashTable whose device copy is newer than its host arrays
        self._ext = None             # torch.cuda.ExternalStream of the context's stream (after_torch)
        self._ready = self._done = None     # after_torch's events: torch's stream ready / calls passed
        self._held = []              # tensors after_torch keeps alive until _done completes

    def check(self, rc):
        if rc != 0:
            msg = self.lib.afp_last_error(self.h)
            msg = msg.decode() if msg else ""
            if rc == -2:
                raise ValueError("libafp: " + msg)
            if rc == -6:
                raise IndexError("libafp: " + msg)
            if rc == -3 and msg.startswith("row capacity exceeded"):
                raise RowCapacityError(msg)
            raise AfpError("libafp status %d: %s" % (rc, msg))

    def set_stream(self, cuda_stream: int | None):
        """Run the context's calls on `cuda_stream` (a cudaStream_t handle; None or 0: the library's
        own stream).  Returns once the work queued on the outgoing stream has finished."""
        self.check(self.lib.afp_set_stream(self.h, _P(cuda_stream) if cuda_stream else None))
        self._release_finished()

    def stream(self) -> int:
        """The cudaStream_t handle the context's calls run on."""
        s = _P()
        self.check(self.lib.afp_get_stream(self.h, C.byref(s)))
        return s.value or 0

    def sync(self):
        self.check(self.lib.afp_sync(self.h))
        self._release_finished()

    @contextlib.contextmanager
    def after_torch(self, *tensors):
        """Order the library calls made inside the block after torch's work on the torch tensors among
        `tensors` (the tensors the calls read or write; other values are ignored):
          - the context's stream first waits, on the device, for everything queued so far on torch's
            current stream of this device (an event: the host does not wait);
          - the tensors are then held until the context's stream has passed the calls, so that
            torch's caching allocator cannot give their memory to new work while a call that returned
            without synchronising (afp_fingerprint_batch with fetch=False) still reads it.
        Nothing is done when no torch tensor is given, or when the context runs on torch's current
        stream: stream order alone then orders both sides."""
        tensors = [t for t in tensors if hasattr(t, "data_ptr") and not isinstance(t, np.ndarray)]
        if not tensors:
            yield
            return
        import torch
        cur = torch.cuda.current_stream(self.device)
        handle = self.stream()
        if handle == cur.cuda_stream:
            yield
            return
        if self._ext is None or self._ext.cuda_stream != handle:
            self._ext = torch.cuda.ExternalStream(handle, device=torch.device("cuda", self.device))
        if self._ready is None:
            self._ready, self._done = torch.cuda.Event(), torch.cuda.Event()
        self._release_finished()
        self._ready.record(cur)
        self._ext.wait_event(self._ready)
        try:
            yield
        finally:
            self._held.append(tensors)
            self._done.record(self._ext)

    def _release_finished(self):
        """Drop the tensors held by after_torch once the context's stream has passed the last call
        that held any (its event covers every earlier one: the holds of a stream that was switched
        away from were synchronised by the switch)."""
        if self._held and self._done.query():
            self._held = []

    def set_profiling(self, on: bool):
        self.check(self.lib.afp_set_profiling(self.h, 1 if on else 0))

    def stage_ms(self):
        out = (C.c_float * 5)()
        self.check(self.lib.afp_get_stage_ms(self.h, out))
        return [float(v) for v in out]

    def launch_count(self) -> int:
        return int(self.lib.afp_launch_count(self.h))

    def close(self):
        if self.h:
            self.lib.afp_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_contexts = {}


def context(device: int | None = None) -> Context:
    """Process-wide context of `device` (default: AFP_DEVICE / LOCAL_RANK / 0)."""
    if device is None:
        device = int(os.environ.get("AFP_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    ctx = _contexts.get(device)
    if ctx is None:
        ctx = _contexts[device] = Context(device)
    return ctx
