"""Timing of the item statistics and K3 stages of the fingerprint batch on the bench's batch, and where
the rest of a bench step goes.

Input: --files seeded synthetic tracks of --seconds each (bench.py's flagship batch by default: 1024 x
30 s), resident on the device as bench.py packs them.  For shifts 1 and 4 the batch is warmed up, then
--steps calls of afp_fingerprint_batch are timed with the library's stage events, as bench.py times
them: the per-stage means (prep, K1, stats, K2, K3), their sum and the step from CUDA events around
the loop.  The step minus the stage sum is the time the device spends outside the five stages.

With --trace DIR, a separate run records --trace-steps shifts-1 steps under torch.profiler with CUDA
activities and writes the chrome trace to DIR.  It prints each kernel's mean time per step and the
device idle time between consecutive GPU activities, summed by the activity that ends the gap: the
gap before the first copy of a step is the host time between steps.

--root times another checkout of the project (its library must be built).  The card's name and power
limit are printed first, in the same run.

    python tools/k3_stats_timing.py [--files 1024] [--seconds 30] [--steps 20] [--trace DIR]
"""
import argparse
import collections
import json
import multiprocessing as mp
import os
import subprocess
import sys

import numpy as np

STAGES = ("prep", "k1_stft_log", "stats", "k2_peaks", "k3_hashes")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def _gen(args):
    from audfprint_b200.synth import synth_track
    return synth_track(*args)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace", metavar="DIR", default=None)
    ap.add_argument("--trace-steps", type=int, default=5)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.root))
    print("card:", card(), flush=True)
    with mp.get_context("fork").Pool(min(32, os.cpu_count() or 1)) as pool:
        tracks = pool.map(_gen, [(i, a.seconds) for i in range(a.files)], chunksize=8)

    import torch
    from audfprint_b200 import Analyzer, _lib
    nsamp = len(tracks[0])
    stride = (nsamp + 7) // 8 * 8          # every file on a 16-byte boundary, as bench.py packs them
    host = torch.zeros(a.files * stride + 8, dtype=torch.int16)
    hp = host.numpy()
    for i, t in enumerate(tracks):
        hp[i * stride:i * stride + nsamp] = t
    pcm = host.cuda()
    offs = np.arange(a.files + 1, dtype=np.int64) * stride
    lens = np.full(a.files, nsamp, np.int64)
    stream = torch.cuda.current_stream()
    ctx = _lib.context(0)
    ctx.set_stream(stream.cuda_stream)

    def step(an):
        an.fingerprint_packed(pcm, offs, fetch=False, sample_lengths=lens)

    out = {"root": os.path.abspath(a.root), "files": a.files, "seconds": a.seconds, "steps": a.steps}
    for shifts in (1, 4):
        an = Analyzer()
        an.shifts = shifts
        for _ in range(a.warmup):
            step(an)
        torch.cuda.synchronize()
        ctx.set_profiling(True)
        st = np.zeros(len(STAGES))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = ctx.launch_count()
        e0.record(stream)
        for _ in range(a.steps):
            step(an)
            st += np.array(ctx.stage_ms())
        e1.record(stream)
        torch.cuda.synchronize()
        ctx.set_profiling(False)
        st /= a.steps
        ms = e0.elapsed_time(e1) / a.steps
        out["shifts%d" % shifts] = {"ms_per_step": ms, "stages_ms": dict(zip(STAGES, st.tolist())),
                                    "stage_sum_ms": float(st.sum()), "outside_stages_ms": ms - float(st.sum()),
                                    "stats_plus_k3_ms": float(st[2] + st[4]),
                                    "launches_per_step": (ctx.launch_count() - l0) / a.steps}
    print(json.dumps(out, indent=1), flush=True)

    if a.trace:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.trace, exist_ok=True)
        an = Analyzer()
        for _ in range(a.warmup):
            step(an)
        torch.cuda.synchronize()
        ctx.set_profiling(True)                  # bench.py's loop: stage events, read after every step
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(a.trace_steps):
                step(an)
                ctx.stage_ms()
            torch.cuda.synchronize()
        ctx.set_profiling(False)
        path = os.path.join(a.trace, "bench_step_trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            ev = json.load(f)["traceEvents"]
        gpu = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")),
                     key=lambda e: e["ts"])
        busy = collections.defaultdict(float)
        gaps = collections.defaultdict(float)
        for prev, e in zip(gpu, gpu[1:]):
            busy[e["name"]] += e["dur"]
            gaps[e["name"]] += max(0.0, e["ts"] - (prev["ts"] + prev["dur"]))
        if gpu:
            busy[gpu[0]["name"]] += gpu[0]["dur"]
        n = a.trace_steps
        span = (gpu[-1]["ts"] + gpu[-1]["dur"] - gpu[0]["ts"]) if gpu else 0.0
        print(json.dumps({"trace": path, "steps": n, "span_us_per_step": span / n,
                          "busy_us_per_step": {k: v / n for k, v in sorted(busy.items(), key=lambda kv: -kv[1])},
                          "idle_us_per_step_before": {k: v / n for k, v in sorted(gaps.items(), key=lambda kv: -kv[1])
                                                      if v / n >= 0.5}}, indent=1), flush=True)


if __name__ == "__main__":
    main()
