"""Timing of the 'ffmpeg' front-end (afp_swr_frontend_batch) against the default one
(afp_pcm_frontend_batch) on the same batch: --files files of --seconds of seeded random stereo int16
at each --rates rate, already on the device (so no host-to-device copy is timed).

Each call is what _frontend_packed does for a round of files: the host sizing call, the zeroed float32
output, the one launch and its synchronise.  Reported: the median of --reps calls after one warm-up
call, host wall clock around calls that end in a device synchronise, and the kernel alone from CUDA
events around the compute call with a preallocated output.

    python tools/ffmpeg_frontend_timing.py [--files 1024] [--seconds 30] [--rates 44100,48000,32000]
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from audfprint_b200 import _lib  # noqa: E402
from audfprint_b200 import analyzer as an_mod  # noqa: E402
from tools.long_query_timing import card  # noqa: E402


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--rates", default="44100,48000,32000")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    card()
    ctx = _lib.context()
    dev = torch.device("cuda", ctx.device)
    P = C.POINTER(C.c_int64)
    for rate in [int(r) for r in a.rates.split(",")]:
        nfr = int(rate * a.seconds)
        g = torch.Generator(device=dev).manual_seed(rate)
        pcm = torch.randint(-32768, 32768, (a.files * nfr * 2,), dtype=torch.int16, device=dev, generator=g)
        inoff = np.arange(a.files, dtype=np.int64) * (2 * nfr)
        frames, chans, rates = [nfr] * a.files, [2] * a.files, [rate] * a.files
        line = ["%d x %.0f s stereo %d Hz (%.2f GB int16)" % (a.files, a.seconds, rate, pcm.numel() * 2 / 1e9)]
        for mode in ("poly", "ffmpeg"):
            call = lambda: an_mod._frontend_packed(ctx, pcm, inoff, frames, chans, rates, 11025, mode)  # noqa: E731
            out, off, lens = call()
            torch.cuda.synchronize()
            ts = []
            for _ in range(a.reps):
                t = time.perf_counter()
                call()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t)
            line.append("%s: %.2f ms per call, %d outputs" % (mode, 1e3 * float(np.median(ts)), int(lens.sum())))
            if mode == "ffmpeg":
                rt = np.array(rates, np.int32)
                ch = np.array(chans, np.int32)
                nf = np.array(frames, np.int64)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ks = []
                for _ in range(a.reps):
                    e0.record(torch.cuda.current_stream(dev))
                    ctx.check(ctx.lib.afp_swr_frontend_batch(ctx.h, pcm.data_ptr(), 0, pcm.numel(), a.files,
                                                             inoff.ctypes.data_as(P), nf.ctypes.data_as(P),
                                                             ch.ctypes.data, rt.ctypes.data, 11025, out.data_ptr(),
                                                             out.numel(), None, None))
                    e1.record(torch.cuda.current_stream(dev))
                    e1.synchronize()
                    ks.append(e0.elapsed_time(e1))
                line.append("ffmpeg compute call alone: %.2f ms" % float(np.median(ks)))
            del out
        print("; ".join(line), flush=True)
        del pcm
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
