"""Timing of HashTable.merge_batch next to the host merge, on two table pairs:

  bench   2^20 buckets x 100 slots, 500,000 ids per table, every slot filled and every count above
          depth (tools/table_edit_timing.py's geometry): every bucket of the merge overflows;
  mirex   2^20 x 100, 4.46 M entries per table spread over the buckets (Poisson counts) and 5,000
          ids: few buckets overflow.

Per pair it reports the median over --reps calls (after one warm-up) of the whole merge_batch,
of the library call afp_table_merge alone (through its final synchronise) and of that call's
stages: the upload of the incoming rows, the classify / fit / compaction kernels, the host replay
of np.random.permutation, the pool-index uploads and the apply kernels (CUDA events), and the wait
after the last replay.  Every call starts from a freshly uploaded table; that upload is not timed.
The host merge runs once per pair.  The stages come from a second library call per repetition,
which synchronises after the upload and after the classify step to time them apart; the library
total is taken from the call without stage timing.

    python tools/table_merge_timing.py [--reps 3]
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import HashTable, _lib  # noqa: E402
from audfprint_b200.synth import synth_table  # noqa: E402
from tools.table_edit_timing import card  # noqa: E402

HASHBITS, DEPTH, MTB = 20, 100, 12
STAGES = ("upload", "classify", "replay", "idx upload", "apply", "tail")


def make(table, counts, hpi, names):
    """A table object over the given arrays (depth=1 at construction: no 419 MB zero table)."""
    ht = HashTable(hashbits=HASHBITS, depth=1, maxtime=1 << MTB)
    ht.table, ht.counts, ht.hashesperid, ht.depth = table, counts, hpi, DEPTH
    ht.names = list(names)
    return ht


def mirex_table(seed, nids, entries=4_460_000):
    rng = np.random.default_rng(seed)
    nb = 1 << HASHBITS
    counts = rng.poisson(entries / nb, nb).astype(np.int32)
    table = np.zeros((nb, DEPTH), np.uint32)
    live = np.arange(DEPTH)[None, :] < np.minimum(counts, DEPTH)[:, None]
    n = int(live.sum())
    table[live] = ((rng.integers(0, nids, n).astype(np.uint32) + 1) << np.uint32(MTB)) | \
        rng.integers(0, 1 << MTB, n).astype(np.uint32)
    hpi = np.bincount((table[live] >> np.uint32(MTB)).astype(np.int64) - 1, minlength=nids).astype(np.uint32)
    return table, counts, hpi


def med(xs):
    return float(np.median(xs))


def run_pair(label, mine, theirs, reps):
    (t1, c1, h1, n1), (t2, c2, h2, n2) = mine, theirs
    other = make(t2, c2, h2, n2)
    tot, lib, stages = [], [], []
    for r in range(reps + 1):
        # the whole method
        ht = make(t1.copy(), c1.copy(), h1.copy(), n1)
        ctx = ht._sync_device()
        ctx.sync()
        np.random.seed(r)
        a = time.perf_counter()
        novf = ht.merge_batch([other])
        ctx.sync()
        b = time.perf_counter()
        # the library call alone, then once more with its stage timings
        for timed in (False, True):
            ht = make(t1, c1, h1, n1)
            ctx = ht._sync_device()
            ctx.sync()
            st = np.random.get_state()
            state = np.empty(625, np.uint32)
            state[:624], state[624] = st[1], st[2]
            ms = np.zeros(6, np.float64)
            c = time.perf_counter()
            ctx.check(ctx.lib.afp_table_merge(ctx.h, t2.ctypes.data, c2.ctypes.data, HASHBITS, DEPTH, len(n1),
                                              state.ctypes.data, None, ms.ctypes.data if timed else None))
            ctx.sync()
            d = time.perf_counter()
            ctx.table_key = None                        # the device copy no longer equals `t1`
            if r and timed:
                stages.append(ms)
            elif r:
                lib.append(d - c)
        if r:
            tot.append(b - a)
    print("%s: %d overflowing buckets" % (label, novf))
    print("  merge_batch %.1f ms, library call %.1f ms" % (1e3 * med(tot), 1e3 * med(lib)))
    s = np.median(np.array(stages), axis=0)
    print("  stages (ms): " + ", ".join("%s %.1f" % (k, v) for k, v in zip(STAGES, s)))
    host = make(t1.copy(), c1.copy(), h1.copy(), n1)
    np.random.seed(0)
    a = time.perf_counter()
    host.merge(other)
    print("  host merge %.1f ms" % (1e3 * (time.perf_counter() - a)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    card()
    nids = 500_000
    t1, c1, h1 = synth_table(HASHBITS, DEPTH, nids, MTB, seed=1)
    t2, c2, h2 = synth_table(HASHBITS, DEPTH, nids, MTB, seed=2)
    run_pair("bench 2^20 x 100, every bucket overflows", (t1, c1, h1, ["a%d" % i for i in range(nids)]),
             (t2, c2, h2, ["b%d" % i for i in range(nids)]), args.reps)
    del t1, t2
    m1, m2 = mirex_table(3, 5000), mirex_table(4, 5000)
    run_pair("mirex 2^20 x 100, 4.46 M entries each", m1 + (["a%d" % i for i in range(5000)],),
             m2 + (["b%d" % i for i in range(5000)],), args.reps)


if __name__ == "__main__":
    main()
