"""Timing of exact_count (-x) and find_time_range (-R) on a table sharded by track-id range, on one
GPU: bench.py's 2^20 x 100 table with 1 M ids split into --shards id ranges, visited in turn as
the ranks of a sharded match would run them.  Per shard: afp_match_options_shard_rank (ranking +
the per-query largest qtime), afp_match_options_shard_finish (with the maxima reduced over the
shards) and afp_shard_pack; then afp_shard_merge of the stacked records.  Next to it, for the same
queries, afp_match_options_batch on the whole table (Matcher.match_batch's device call).  The
all-reduce and the all-gather between the steps are not part of these numbers.

Times are host wall clock around whole calls (each ends in a stream synchronise; queries already
on the device): median of --repeats after one warm-up call.

    python tools/shard_options_timing.py [--queries 1024] [--shards 4] [--row-cap 16]
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from audfprint_b200 import Analyzer, HashTable, Matcher  # noqa: E402
from audfprint_b200 import dist as afd  # noqa: E402
from audfprint_b200.matcher import timebits_breaks  # noqa: E402
from audfprint_b200.synth import synth_query, synth_track  # noqa: E402
from tools.long_query_timing import card  # noqa: E402


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--shards", type=int, default=4)
    ap.add_argument("--row-cap", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    card()
    an = Analyzer()
    tracks = [synth_track(9000 + i, 30.0) for i in range(64)]
    th = an.fingerprint_batch(tracks)
    rows = np.concatenate(th)
    roff = np.concatenate([[0], np.cumsum([len(h) for h in th])]).astype(np.int64)
    table, counts, hashbits, depth, mtb, hpi, _ = bench.build_big_table(rows, roff, 1000000)
    ht = HashTable(hashbits=hashbits, depth=1, maxtime=1 << mtb)
    ht.table, ht.counts, ht.hashesperid, ht.depth = table, counts, hpi, depth
    ht.names = [None] * 1000000
    qan = Analyzer()
    qan.shifts = 4
    qs = qan.fingerprint_batch([synth_query(tracks[j % 64], j, seconds=10.0, noise_sigma=0.02)[0]
                                for j in range(args.queries)])
    qoff = np.concatenate([[0], np.cumsum([len(q) for q in qs])]).astype(np.int64)
    dq = torch.from_numpy(np.ascontiguousarray(np.concatenate(qs))).cuda()
    nq, ns, rcap = len(qs), args.shards, args.row_cap
    qp = qoff.ctypes.data_as(C.POINTER(C.c_int64))
    br = timebits_breaks().ctypes.data_as(C.POINTER(C.c_int64))
    print("bench table 2^20 x 100, 1 M ids, %d shards by id range; %d queries of %.0f rows on average; row_cap %d"
          % (ns, nq, np.mean(np.diff(qoff)), rcap))
    for exact, trange, tag in ((True, False, "-x"), (False, True, "-R"), (True, True, "-x -R")):
        m = Matcher()
        m.window, m.exact_count, m.find_time_range = 2, exact, trange
        p = m._params()
        p.row_capacity = 256
        tot = C.c_int64(0)
        ctx = ht._sync_device()
        t_whole = timed(lambda: ctx.check(ctx.lib.afp_match_options_batch(
            ctx.h, dq.data_ptr(), 0, nq, qp, C.byref(p), int(exact), int(trange), float(m.time_quantile), br,
            C.byref(tot))), args.repeats)
        whole_rows = int(tot.value)
        sd = m.search_depth
        rb = int(ctx.lib.afp_shard_record_bytes(sd, rcap))
        qmax = [torch.empty(nq, dtype=torch.int32, device="cuda") for _ in range(ns)]

        def rank(s):
            ctx.check(ctx.lib.afp_match_options_shard_rank(
                ctx.h, dq.data_ptr(), 0, nq, qp, C.byref(p), int(exact), int(trange), float(m.time_quantile), br,
                C.c_void_p(qmax[s].data_ptr()), C.byref(tot)))
        for s in range(ns):                                   # pass 1: every shard's maxima
            ht.restrict_device_ids(*afd.id_range(1000000, s, ns))
            rank(s)
        red = torch.stack(qmax).amax(dim=0).contiguous()
        torch.cuda.synchronize()
        bufs, t_rank, t_fin, t_pack, shard_rows = [], [], [], [], []
        for s in range(ns):
            ctx = ht.restrict_device_ids(*afd.id_range(1000000, s, ns))
            buf = torch.empty((nq, rb), dtype=torch.uint8, device="cuda")
            t_rank.append(timed(lambda: rank(s), args.repeats))

            def rank_finish():
                rank(s)
                ctx.check(ctx.lib.afp_match_options_shard_finish(ctx.h, C.c_void_p(red.data_ptr()), C.byref(tot)))
            t_fin.append(timed(rank_finish, args.repeats))
            shard_rows.append(int(tot.value))
            t_pack.append(timed(lambda: ctx.check(ctx.lib.afp_shard_pack(ctx.h, rcap, buf.data_ptr())), args.repeats))
            bufs.append(buf)
        gathered = torch.cat(bufs, dim=0).contiguous()
        t_merge = timed(lambda: ctx.check(ctx.lib.afp_shard_merge(ctx.h, gathered.data_ptr(), ns, nq, sd, rcap,
                                                                  C.byref(tot))), args.repeats)
        ht._touch()
        print("  %-6s whole table afp_match_options_batch %8.2f ms (%d rows)" % (tag, 1e3 * t_whole, whole_rows))
        for s in range(ns):
            print("         shard %d/%d: rank %7.2f ms; rank + finish %7.2f ms; pack %6.2f ms; rank + finish + pack "
                  "%7.2f ms (%d rows)" % (s, ns, 1e3 * t_rank[s], 1e3 * t_fin[s], 1e3 * t_pack[s],
                                          1e3 * (t_fin[s] + t_pack[s]), shard_rows[s]))
        print("         merge of %d shards: %6.2f ms (%d rows); slowest shard + merge %7.2f ms"
              % (ns, 1e3 * t_merge, int(tot.value),
                 1e3 * (max(b + c for b, c in zip(t_fin, t_pack)) + t_merge)))


if __name__ == "__main__":
    main()
