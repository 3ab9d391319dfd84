#!/usr/bin/env python
"""Cost of reduce_noise(use_torch=True) on config 2's geometry (48 kHz, chunk_size 600000, padding 30000, n_fft 1024,
stationary gate, float32 samples from bench.py's generator).

    python scripts/bench_torch_route.py [--channels 64] [--minutes 10] [--runs 3] [--out result.json]

Arms, alternated in one process, each timed by the host clock around work that ends in a device synchronise:
  per_chunk_loop   StreamedTorchGate._get_traces_per_chunk(): the reference's loop, one TorchGate call per padded
                   float64 chunk, copied to the device and back;
  one_call_numpy   reduce_noise(y, use_torch=True) on a pageable numpy array: one library call over the chunk grid;
  one_call_cuda    reduce_noise(y_cuda, use_torch=True) on a resident CUDA tensor, result a CUDA tensor;
  stream_1s        NoiseReduceStream(use_torch=True) fed the CUDA tensor in 1 s blocks (push + finish);
  stream_10s       the same in 10 s blocks.
Per arm: the median of the per-run times and their range.  Also checks, outside the timed calls, that the one call and
the stream equal the loop in every bit, and prints the card, its power limit and maximum SM clock, as one JSON object.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import SR, synth_host  # noqa: E402  (config 2's host workload)
from scripts.bench_stream import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import noisereduce_b200 as nr
    from noisereduce_b200.spectralgate.streamed_torch_gate import StreamedTorchGate

    C, N = args.channels, int(args.minutes * 60 * SR)
    y_np = synth_host(np, C, N)
    x = torch.from_numpy(y_np).cuda()
    kw = dict(sr=SR, stationary=True, use_torch=True)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    def stream(block):
        s = nr.NoiseReduceStream(sr=SR, n_channels=C, stationary=True, use_torch=True)
        outs = [s.push(x[:, i:i + block]) for i in range(0, N, block)]
        outs.append(s.finish())
        return torch.cat(outs, 1)

    arms = {
        "per_chunk_loop": lambda: StreamedTorchGate(y=y_np, sr=SR, stationary=True)._get_traces_per_chunk(),
        "one_call_numpy": lambda: nr.reduce_noise(y_np, **kw),
        "one_call_cuda": lambda: nr.reduce_noise(x, **kw),
        "stream_1s": lambda: stream(SR),
        "stream_10s": lambda: stream(10 * SR),
    }
    nr.reduce_noise(x[:, :1_300_000], **kw)                   # warm-up: kernels loaded, workspace sized
    times = {k: [] for k in arms}
    same = {}
    ref = None
    for run in range(args.runs):
        for k, fn in arms.items():
            t, r = timed(fn)
            times[k].append(t)
            if run == 0:                                      # bit checks against the loop, outside the timings
                r = r.cpu().numpy() if isinstance(r, torch.Tensor) else r
                if ref is None:
                    ref = r
                else:
                    same[k] = bool(r.shape == ref.shape and r.dtype == ref.dtype and
                                   np.array_equal(r.view(np.uint8), ref.view(np.uint8)))
            del r
            torch.cuda.empty_cache()

    def summary(ts):
        ts = sorted(t * 1e3 for t in ts)
        med = float(np.median(ts))
        return {"ms_median": round(med, 1), "ms_min": round(ts[0], 1), "ms_max": round(ts[-1], 1),
                "msamples_per_s": round(C * N / (med * 1e-3) / 1e6, 1)}

    result = {
        "workload": f"{C} ch x {args.minutes:g} min @ {SR} Hz, float32, stationary, use_torch=True, chunk_size 600000, "
                    f"padding 30000; {args.runs} runs, arms alternated",
        "arms": {k: summary(v) for k, v in times.items()},
        "bit_identical_to_per_chunk_loop": same,
        "card": card(),
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
