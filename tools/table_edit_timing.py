"""Timing of HashTable.remove_batch / retrieve_batch on the bench table geometry (2^20 buckets x
100 slots, 1 M ids, every bucket full, counts above depth), next to the host remove / retrieve of
one name.

For 1, 100, 1000 and 10,000 names it reports the median over repeated calls (after one warm-up)
of the whole method, of its Python name lookup, and of the library call alone (ctypes call
through its final stream synchronise).  Every remove starts from a freshly uploaded table; the
upload is not timed.

    python tools/table_edit_timing.py [--reps 5]
"""
import argparse
import contextlib
import ctypes as C
import io
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import HashTable, _lib  # noqa: E402
from audfprint_b200.synth import synth_table  # noqa: E402

HASHBITS, DEPTH, MTB, NIDS = 20, 100, 12, 1_000_000
I64P = C.POINTER(C.c_int64)


def card():
    """The card the library context times (AFP_DEVICE / LOCAL_RANK), found by UUID for nvidia-smi."""
    import torch
    dev = _lib.context().device
    props = torch.cuda.get_device_properties(dev)
    uuid = str(props.uuid)
    uuid = uuid if uuid.startswith("GPU-") else "GPU-" + uuid
    print("device %d: %s (%s)" % (dev, props.name, uuid))
    try:
        print(subprocess.run(["nvidia-smi", "-i", uuid, "--query-gpu=power.limit,clocks.max.sm",
                              "--format=csv"], capture_output=True, text=True, timeout=30).stdout.strip())
    except (OSError, subprocess.SubprocessError) as e:
        print("nvidia-smi unavailable:", e)


def fresh(table, counts, hpi, names):
    """A table object over the shared arrays (depth=1 at construction: no 419 MB zero table)."""
    ht = HashTable(hashbits=HASHBITS, depth=1, maxtime=1 << MTB)
    ht.table, ht.counts, ht.hashesperid, ht.depth = table, counts, hpi.copy(), DEPTH
    ht.names = list(names)
    return ht


def med(xs):
    return 1e3 * float(np.median(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    card()
    t0 = time.perf_counter()
    table, counts, hpi = synth_table(HASHBITS, DEPTH, NIDS, MTB, seed=5)
    names = ["t%d" % i for i in range(NIDS)]
    print("table 2^%d x %d, %d ids, built in %.1f s" % (HASHBITS, DEPTH, NIDS, time.perf_counter() - t0))
    rng = np.random.default_rng(1)
    quiet = contextlib.redirect_stdout(io.StringIO())
    print("%-9s %6s %12s %12s %12s" % ("method", "names", "total ms", "lookup ms", "library ms"))
    for n in (1, 100, 1000, 10000):
        pick = [names[i] for i in rng.choice(NIDS, n, replace=False)]
        # remove: a freshly uploaded table per call
        tot, look, dev = [], [], []
        for r in range(args.reps + 1):
            ht = fresh(table, counts, hpi, names)
            ctx = ht._sync_device()
            ctx.sync()
            a = time.perf_counter()
            with quiet:
                ht.remove_batch(pick)
            ctx.sync()
            b = time.perf_counter()
            ht = fresh(table, counts, hpi, names)
            ctx = ht._sync_device()
            ctx.sync()
            c = time.perf_counter()
            ids = ht._ids_of(pick, distinct=True)
            d = time.perf_counter()
            ctx.check(ctx.lib.afp_table_remove_ids(ctx.h, ids.ctypes.data_as(I64P), n, None))
            ctx.sync()
            e = time.perf_counter()
            ctx.table_key = None                        # the device copy no longer equals `table`
            if r:
                tot.append(b - a), look.append(d - c), dev.append(e - d)
        print("%-9s %6d %12.3f %12.3f %12.3f" % ("remove", n, med(tot), med(look), med(dev)))
        # retrieve: the table does not change
        ht = fresh(table, counts, hpi, names)
        ctx = ht._sync_device()
        tot, look, dev = [], [], []
        for r in range(args.reps + 1):
            ctx.sync()
            a = time.perf_counter()
            ht.retrieve_batch(pick)
            ctx.sync()
            b = time.perf_counter()
            ids = ht._ids_of(pick, distinct=False)
            c = time.perf_counter()
            total = C.c_int64(0)
            ctx.check(ctx.lib.afp_table_retrieve_ids(ctx.h, ids.ctypes.data_as(I64P), n, C.byref(total)))
            rows = np.empty((total.value, 2), np.int32)
            off = np.empty(n + 1, np.int64)
            ctx.check(ctx.lib.afp_fetch_retrieved(ctx.h, rows.ctypes.data, 1, off.ctypes.data_as(I64P)))
            ctx.sync()
            d = time.perf_counter()
            if r:
                tot.append(b - a), look.append(c - b), dev.append(d - c)
        print("%-9s %6d %12.3f %12.3f %12.3f" % ("retrieve", n, med(tot), med(look), med(dev)))
    # the host methods, one name, for comparison
    host = fresh(table.copy(), counts.copy(), hpi, names)
    t_rm, t_rt = [], []
    for name in names[:3]:
        a = time.perf_counter()
        host.retrieve(name)
        b = time.perf_counter()
        with quiet:
            host.remove(name)
        t_rm.append(time.perf_counter() - b), t_rt.append(b - a)
    print("host remove, one name: %.1f ms; host retrieve, one name: %.1f ms" % (med(t_rm), med(t_rt)))


if __name__ == "__main__":
    main()
