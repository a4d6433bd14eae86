"""Timing of K4 on long queries: the long-query path (rows * depth >= 2^24) next to the general
kernel (Matcher.force_general_kernel), on two workloads.

Ad search (the reference's searching_for_ads.md workflow): --ads synthetic 30 s "ads" at density
100, stored with store_batch into a 2^20 x depth table (depth 100, then 500); --shows synthetic
one-hour "shows" at density 100, shifts 1, each with --per-show ads spliced into its PCM at known
sample offsets (multiples of the hop).  Matcher: window 2, max_alignments_per_id default,
threshcount 10.  Per depth: ms per show on the long path (every show) and on the general kernel
(the first --general-shows shows), rows of the two paths identical, every spliced ad found at its
offset (dtime = -offset / hop, +-1 frame).

Broadcast day: one 24-hour recording at density 20 and one at density 100 (24 one-hour synthetic
pieces, fingerprinted and concatenated in time) against the bench table (2^20 x 100, 1 M ids,
every bucket full).  Reports the call time, the device memory the library allocated for it (the
drop of free memory over a first call), hits and candidates; at density 20 also the general
kernel's time.

Times are host wall clock around Matcher.match_batch (query upload, matching, row fetch), which
ends in a stream synchronise.

    python tools/long_query_timing.py [--ads 2000] [--shows 100] [--general-shows 10] [--skip-day]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import Analyzer, HashTable, Matcher, _lib  # noqa: E402
from audfprint_b200.synth import synth_track, synth_table  # noqa: E402

SR, HOP = 11025, 256


def card():
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


def free_bytes():
    import torch
    return torch.cuda.mem_get_info(_lib.context().device)[0]


def fingerprint(density, pcms):
    an = Analyzer(density=density)
    return an.fingerprint_batch(pcms)


def timed_match(m, ht, q, general):
    m.force_general_kernel = general
    t0 = time.perf_counter()
    r = m.match_batch(ht, [q], sort=False)[0]
    dt = time.perf_counter() - t0
    m.force_general_kernel = False
    return r, dt


def ad_search(args):
    rng = np.random.default_rng(7)
    ad_len = int(30 * SR)
    ads = [synth_track(100000 + i, 30.0) for i in range(args.ads)]
    t0 = time.perf_counter()
    ad_h = fingerprint(100.0, ads)
    print("ads: %d x 30 s, density 100: %d hashes (%.0f per ad), fingerprinted in %.1f s"
          % (args.ads, sum(map(len, ad_h)), np.mean([len(h) for h in ad_h]), time.perf_counter() - t0))
    truth, show_h = [], []
    t0 = time.perf_counter()
    for s0 in range(0, args.shows, 4):                      # 4 one-hour shows of PCM at a time
        pcms = []
        for s in range(s0, min(args.shows, s0 + 4)):
            pcm = synth_track(200000 + s, args.show_seconds)
            which = rng.choice(args.ads, args.per_show, replace=False)
            slots = np.sort(rng.choice(int(args.show_seconds // 60) - 1, args.per_show, replace=False))
            spl = []
            for a, k in zip(which, slots):
                off = int(k) * 60 * SR + int(rng.integers(0, 20 * SR)) // HOP * HOP
                pcm[off:off + ad_len] = ads[a]
                spl.append((int(a), off // HOP))
            pcms.append(pcm)
            truth.append(spl)
        show_h += fingerprint(100.0, pcms)
    nrows = np.array([len(h) for h in show_h])
    print("shows: %d x %.0f s, density 100: %.0f rows per hour on average (min %d, max %d), fingerprinted in %.1f s"
          % (args.shows, args.show_seconds, nrows.mean() * 3600 / args.show_seconds, nrows.min(), nrows.max(),
             time.perf_counter() - t0))
    names = ["ad%d" % i for i in range(args.ads)]
    for depth in (100, 500):
        ht = HashTable(hashbits=20, depth=depth, maxtime=1 << 14)
        ht.store_batch(names, ad_h)
        m = Matcher()
        m.window, m.threshcount = 2, 10
        print("depth %d: rows x depth of a show %.2e .. %.2e (long from %.2e)"
              % (depth, nrows.min() * depth, nrows.max() * depth, 2.0 ** 24))
        timed_match(m, ht, show_h[0], False)                       # warm-up of both paths
        if args.general_shows:
            timed_match(m, ht, show_h[0], True)
        t_long, t_gen, found, same = [], [], 0, 0
        for i, q in enumerate(show_h):
            r, dt = timed_match(m, ht, q, False)
            t_long.append(dt)
            assert Matcher.last_status(ht, 1)[0, 0] == 6
            for a, dtf in truth[i]:
                found += int(np.any((r[:, 0] == a) & (np.abs(r[:, 2] + dtf) <= 1)))
            if i < args.general_shows:
                rg, dtg = timed_match(m, ht, q, True)
                t_gen.append(dtg)
                same += int(np.array_equal(r, rg))
        print("  long path     : %.1f ms per show (median of %d; mean %.1f)"
              % (1e3 * np.median(t_long), len(t_long), 1e3 * np.mean(t_long)))
        if t_gen:
            print("  general kernel: %.1f ms per show (median of %d; mean %.1f); rows identical on %d / %d shows"
                  % (1e3 * np.median(t_gen), len(t_gen), 1e3 * np.mean(t_gen), same, len(t_gen)))
        print("  spliced ads found at their offset: %d / %d" % (found, sum(map(len, truth))))
        del ht


def broadcast_day(args):
    t0 = time.perf_counter()
    table, counts, hpi = synth_table(20, 100, 1_000_000, 12, seed=5)
    print("bench table 2^20 x 100, 1 M ids, every bucket full (built in %.1f s)" % (time.perf_counter() - t0))
    for density in (20.0, 100.0):
        parts, t_end = [], 0
        t0 = time.perf_counter()
        for h in range(args.day_hours):
            q = fingerprint(density, [synth_track(300000 + h, 3600.0)])[0].astype(np.int64)
            q[:, 0] += t_end
            t_end += int(3600 * SR / HOP)
            parts.append(q)
        q = np.concatenate(parts).astype(np.int32)
        print("%d h recording, density %g: %d rows (%.0f per hour), fingerprinted in %.1f s"
              % (args.day_hours, density, len(q), len(q) / args.day_hours, time.perf_counter() - t0))
        ht = HashTable(hashbits=20, depth=1, maxtime=1 << 12)
        ht.table, ht.counts, ht.hashesperid, ht.depth = table, counts, hpi, 100
        ht.names = ["t%d" % i for i in range(1_000_000)]
        m = Matcher()
        m.match_batch(ht, [q[:1000]])                  # table upload, short-query scratch
        free0 = free_bytes()
        r, dt = timed_match(m, ht, q, False)
        grew = free0 - free_bytes()
        r2, dt2 = timed_match(m, ht, q, False)
        hits = int(np.minimum(100, counts[q[:, 1].astype(np.int64) & ((1 << 20) - 1)]).sum())
        rows, roff, cand, cnts = m._publish_call(ht, q, np.array([0, len(q)], np.int64))
        print("  long path: %.1f ms (first call %.1f ms), library allocated %.2f GB on the first call; "
              "%d hits, %d ids above threshcount, %d candidates, %d rows; status %d"
              % (1e3 * dt2, 1e3 * dt, grew / 1e9, hits, int(cnts[0, 1]), min(int(cnts[0, 1]), m.search_depth),
                 len(r2), Matcher.last_status(ht, 1)[0, 0]))
        if density == 20.0 and not args.skip_general_day:
            rg, dtg = timed_match(m, ht, q, True)
            print("  general kernel: %.1f ms; rows identical: %s" % (1e3 * dtg, np.array_equal(rg, r2)))
        del ht


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ads", type=int, default=2000)
    ap.add_argument("--shows", type=int, default=100)
    ap.add_argument("--show-seconds", type=float, default=3600.0)
    ap.add_argument("--per-show", type=int, default=4)
    ap.add_argument("--general-shows", type=int, default=10)
    ap.add_argument("--day-hours", type=int, default=24)
    ap.add_argument("--skip-ads", action="store_true")
    ap.add_argument("--skip-day", action="store_true")
    ap.add_argument("--skip-general-day", action="store_true")
    args = ap.parse_args()
    card()
    if not args.skip_ads:
        ad_search(args)
    if not args.skip_day:
        broadcast_day(args)


if __name__ == "__main__":
    main()
