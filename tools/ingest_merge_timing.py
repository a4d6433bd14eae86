"""Timing of building one table from W per-rank ingest tables (dist.ingest_sharded's merge), on
the BASELINE configs[3] geometry: 2^20 buckets x 100 slots, maxtimebits 14, each per-rank table
filled by one batch of --files x --seconds tracks (Analyzer.fingerprint_packed + store_batch on the
device, random.seed(1000 + r) for table r).  On one GPU the W tables live in one process.

It reports, per stage, the median over --reps runs (milliseconds):
  export        HashTable.export_device of one per-rank table whose device copy is current
                (device to device, afp_table_export)
  counts copy   afp_table_merge_device's copy of the incoming counts to the host for its checks
  classify      classify + compaction kernels
  host replay   the np.random.permutation replay of the overflowing buckets
  apply         pool-index uploads + gather / write-back kernels (CUDA events, overlap the replay)
  merge_batch   the whole merge of the W snapshots into an empty table
next to the host route: each table's `ht.table` / `ht.counts` pulled to the host, then merge_batch
of the host tables (which uploads their rows).  The transfer between GPUs (NCCL send / recv) and
the broadcast of replicate=True need W GPUs and are not timed here.

    python tools/ingest_merge_timing.py [--tables 2] [--files 1024] [--seconds 180] [--reps 3]
"""
import argparse
import multiprocessing as mp
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import Analyzer, HashTable, _lib  # noqa: E402
from audfprint_b200.synth import SR, synth_track  # noqa: E402
from tools.table_edit_timing import card  # noqa: E402

HASHBITS, DEPTH, MTB = 20, 100, 14


def _gen(args):
    return synth_track(*args)


def rank_table(an, dev_pcm, offs, lens, r):
    random.seed(1000 + r)
    ht = HashTable(hashbits=HASHBITS, depth=DEPTH, maxtime=1 << MTB)
    an.fingerprint_packed(dev_pcm, offs, fetch=False, sample_lengths=lens)
    ht.store_batch(["r%d/t%d" % (r, i) for i in range(len(lens))])
    return ht


def med(xs):
    return float(np.median(xs)) if len(xs) else float("nan")


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--tables", type=int, default=2)
    ap.add_argument("--files", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--distinct", type=int, default=128, help="distinct synthetic tracks per table, recycled")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    card()
    nsamp = int(round(a.seconds * SR))
    stride = (nsamp + 7) // 8 * 8
    with mp.get_context("fork").Pool(min(32, os.cpu_count() or 1)) as pool:
        tracks = [pool.map(_gen, [(5000 + 1000 * r + i, a.seconds) for i in range(a.distinct)], chunksize=4)
                  for r in range(a.tables)]
    dev = torch.device("cuda", _lib.context().device)
    lens = np.full(a.files, nsamp, np.int64)
    offs = np.arange(a.files + 1, dtype=np.int64) * stride
    an = Analyzer()
    an.density, an.maxpairsperpeak, an.maxpksperframe = 20.0, 3, 5
    tables = []
    for r in range(a.tables):
        # table r's files: its own distinct tracks, recycled
        buf = np.zeros(a.files * stride + 8, np.int16)
        for i in range(a.files):
            buf[i * stride:i * stride + nsamp] = tracks[r][i % a.distinct]
        dev_pcm = torch.from_numpy(buf).to(dev)
        tables.append(rank_table(an, dev_pcm, offs, lens, r))
        del dev_pcm
    for r, t in enumerate(tables):
        c = t.counts
        print("table %d: %d names, %d entries, %d buckets above depth" % (r, len(t.names), int(c.sum()),
                                                                          int((c > DEPTH).sum())))
    ex, tot, stages, host_pull, host_merge = [], [], [], [], []
    for rep in range(a.reps + 1):
        snaps = []
        for t in tables:
            t._sync_device().sync()                  # (one context holds one table: upload it first)
            a0 = time.perf_counter()
            snaps.append(t.export_device())
            if rep:
                ex.append(time.perf_counter() - a0)
        # the whole merge of the snapshots into an empty table
        np.random.seed(rep)
        ht = HashTable(hashbits=HASHBITS, depth=DEPTH, maxtime=1 << MTB)
        ctx = ht._sync_device()
        ctx.sync()
        a0 = time.perf_counter()
        ht.merge_batch(snaps)
        ctx.sync()
        if rep:
            tot.append(time.perf_counter() - a0)
        # the same merges with the library's stage timing
        ht = HashTable(hashbits=HASHBITS, depth=DEPTH, maxtime=1 << MTB)
        ctx = ht._sync_device()
        st = np.random.get_state()
        state = np.empty(625, np.uint32)
        state[:624], state[624] = st[1], st[2]
        ms_all = np.zeros(6)
        nn = 0
        for s in snaps:
            ms = np.zeros(6)
            ctx.check(ctx.lib.afp_table_merge_device(ctx.h, s.table.data_ptr(), s.counts.data_ptr(), s.hashbits,
                                                     s.depth, nn, state.ctypes.data, None, ms.ctypes.data))
            nn += len(s.names)
            ms_all += ms
        ctx.table_key = None
        if rep:
            stages.append(ms_all)
        del snaps
        # the host route: every table pulled to the host, then merge_batch of the host tables
        if rep:
            for t in tables:
                ctx_t = t._sync_device()
                ctx_t.sync()
                tab = np.empty((1 << HASHBITS, DEPTH), np.uint32)
                cnt = np.empty(1 << HASHBITS, np.int32)
                b0 = time.perf_counter()
                ctx_t.check(ctx_t.lib.afp_table_download(ctx_t.h, tab.ctypes.data, cnt.ctypes.data))
                host_pull.append(time.perf_counter() - b0)
            np.random.seed(rep)
            ht = HashTable(hashbits=HASHBITS, depth=DEPTH, maxtime=1 << MTB)
            ctx = ht._sync_device()
            ctx.sync()
            a0 = time.perf_counter()
            ht.merge_batch(tables)
            ctx.sync()
            host_merge.append(time.perf_counter() - a0)
    s = np.median(np.array(stages), axis=0)
    print("W = %d tables of %d x %.0f s" % (a.tables, a.files, a.seconds))
    print("  export %.1f ms per table" % (1e3 * med(ex)))
    print("  device route: merge_batch of %d snapshots %.1f ms; summed over the merges: counts copy %.1f, "
          "classify %.1f, host replay %.1f, index upload %.1f, apply kernels %.1f, tail %.1f ms"
          % (a.tables, 1e3 * med(tot), *s))
    print("  host route: table pull %.1f ms per table, merge_batch of %d host tables %.1f ms"
          % (1e3 * med(host_pull), a.tables, 1e3 * med(host_merge)))


if __name__ == "__main__":
    main()
