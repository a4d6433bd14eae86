"""audfprint_b200 — H100-native (sm_90a) landmark audio-fingerprint engine
behind the Analyzer / HashTable / Matcher API of dpwe/audfprint.

Only the one hot path of SURVEY.md §8 lives here: csrc/ (CUDA kernels + C ABI,
built into libafp.so) and the host-side mirror of the reference classes.
Importing the package does not need a GPU; using it does (no CPU fallback)."""
from .analyzer import (Analyzer, landmarks2hashes, hashes2landmarks, hashes_save, hashes_load,
                       peaks_save, peaks_load, PRECOMPEXT, PRECOMPPKEXT)
from .hash_table import HashTable
from .matcher import Matcher

__all__ = ["Analyzer", "HashTable", "Matcher", "landmarks2hashes", "hashes2landmarks",
           "hashes_save", "hashes_load", "peaks_save", "peaks_load", "PRECOMPEXT", "PRECOMPPKEXT"]
