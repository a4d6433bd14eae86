"""The reference's multi-process ingest (`audfprint.py new / add --ncores N`: multiproc_add,
audfprint.py:199-235, with make_ht_from_list, :130-144) as a plain sequence, the statement that
dist.ingest_sharded and merge_batch of per-rank device tables are held to:

  * file ix goes to worker ix % ncores;
  * worker r stores its files, in order, into a fresh table of the base's geometry, drawing from its
    OWN `random` state (tests/table_reference.py's store with a random.Random per worker);
  * the parent merges the worker tables into the base in worker order 0..N-1, drawing from its
    np.random state (tests/merge_reference.py's merge), after reporting
    "hash_table r has N files H hashes" for each.

The reference's forked workers reseed `random` from OS entropy, so its own --ncores table is only
reproducible once each worker's seed is fixed; oracle/make_golden_ingest_merge.py fixes it to
SEED + r and stores what the reference then builds in tests/golden/ingest_merge.npz.
tests/test_ingest_merge_cpu.py pins this statement to that fixture."""
import random

import numpy as np

from tests import merge_reference as mref
from tests import table_reference as ref

# the fixture's inputs (oracle/make_golden_ingest_merge.py): a 2^10 x 6 table that overflows in the
# workers and in the merge, 24 files of match.npz track hashes, one of them with no hashes
HASHBITS, DEPTH, MAXTIMEBITS = 10, 6, 12
SEED = 1000                 # worker r: random.seed(SEED + r)
NP_SEED = 4242              # the parent's np.random before multiproc_add
BASE_SEED = 77              # `random` while the reference builds the base of the `add` cases
NFILES, EMPTY_AT = 24, 5    # file EMPTY_AT has no hashes
BASE_TRACKS, BASE_REMOVED = range(30, 36), "track32"
CASES = [("new", 1), ("new", 2), ("new", 3), ("new", 5), ("add", 1), ("add", 2), ("add", 3), ("add", 5),
         ("few", 5)]        # "few": `new` of the first 3 files on 5 workers (two workers get none)


def fixture_files(gm, mode="new"):
    """(name, int32 (n, 2) [time, hash] rows) of the fixture's files, in command-line order."""
    n = 3 if mode == "few" else NFILES
    out = []
    for i in range(n):
        if i == EMPTY_AT:
            out.append(("silence", np.zeros((0, 2), np.int32)))
        else:
            out.append(("track%d" % i, np.asarray(gm["track%d/hashes" % i], np.int32)))
    return out


def deal(nfiles, ncores):
    """Indices of the files of every worker (audfprint.py:211-214)."""
    return [list(range(r, nfiles, ncores)) for r in range(ncores)]


def worker_table(files, hashbits, depth, maxtimebits, rng):
    """make_ht_from_list: a fresh table, one store per file, draws from `rng`."""
    st = ref.State(hashbits, depth, maxtimebits)
    for name, rows in files:
        ref.store(st, ref.name_to_id(st, name), rows, rng)
    return st


def multiproc_add(base, files, ncores, seeds, np_rng=np.random):
    """Merge the worker tables of `files` on `ncores` workers into `base` (changed in place); worker
    r draws from random.Random(seeds[r]).  Returns the report lines."""
    lines = []
    for r, idx in enumerate(deal(len(files), ncores)):
        w = worker_table([files[i] for i in idx], base.hashbits, base.depth, base.maxtimebits,
                         random.Random(seeds[r]))
        lines.append("hash_table %d has %d files %d hashes" % (r, len(w.names), int(w.counts.sum())))
        mref.merge(base, w, np_rng)
    return lines


def golden_base(want, mode):
    """The case's base table as the fixture stores it (empty for `new`)."""
    if mode != "add":
        return ref.State(HASHBITS, DEPTH, MAXTIMEBITS)
    names = [None if n == "" else str(n) for n in want["base/names"]]
    return ref.State(HASHBITS, DEPTH, MAXTIMEBITS, want["base/table"], want["base/counts"], names,
                     want["base/hashesperid"])


def golden_names(want, key):
    return [None if n == "" else str(n) for n in want[key + "/names"]]
