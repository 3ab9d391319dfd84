#!/usr/bin/env python
"""Streaming throughput: NoiseReduceStream on config 2's data (64 ch x 10 min, 48 kHz, stationary) pushed in 1 s, 10 s
and 60 s blocks, alternated in the same process with reduce_noise() on the same host array.

    python scripts/bench_stream.py [--runs 3] [--minutes 10] [--out result.json]

Per arm: samples/s (median and range over the runs), the per-push wall time of the 1 s arm, and the device memory the
library holds while streaming (cudaMemGetInfo before the stream and at its lowest during it).  Every stream run is
checked bit for bit against reduce_noise()'s result outside the timed pushes.  Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import SR, synth_host  # noqa: E402  (config 2's host workload)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # (reporting only)
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import noisereduce_b200 as nr

    C, N = 64, int(args.minutes * 60 * SR)
    y = synth_host(np, C, N)
    kw = dict(sr=SR, stationary=True)
    nr.reduce_noise(y[:, : 2 * 600000], **kw)                  # warm-up: kernels loaded, pools filled
    ref = None
    arms = {"reduce_noise": []}
    blocks = {"1s": SR, "10s": 10 * SR, "60s": 60 * SR}
    for b in blocks:
        arms["stream_" + b] = []
    push_ms_1s, mem = [], {}

    def stream_run(bs):
        free0 = torch.cuda.mem_get_info()[0]
        lowest = free0
        s = nr.NoiseReduceStream(n_channels=C, **kw)
        outs, times, t_all = [], [], 0.0
        for i in range(0, N, bs):
            blk = y[:, i:i + bs]
            t0 = time.perf_counter()
            out = s.push(blk)
            dt = time.perf_counter() - t0
            t_all += dt
            times.append(dt * 1e3)
            outs.append(out)
            lowest = min(lowest, torch.cuda.mem_get_info()[0])
        t0 = time.perf_counter()
        outs.append(s.finish())
        t_all += time.perf_counter() - t0
        lowest = min(lowest, torch.cuda.mem_get_info()[0])
        pos, equal = 0, True
        for o in outs:
            equal &= bool(np.array_equal(o, ref[:, pos:pos + o.shape[1]]))
            pos += o.shape[1]
        equal &= pos == N
        return t_all, times, (free0 - lowest) / 2**20, equal

    equal_all = True
    for r in range(args.runs):
        t0 = time.perf_counter()
        res = nr.reduce_noise(y, **kw)
        arms["reduce_noise"].append(time.perf_counter() - t0)
        if ref is None:
            ref = res
        del res
        for b, bs in blocks.items():
            t, times, mib, equal = stream_run(bs)
            arms["stream_" + b].append(t)
            equal_all &= equal
            mem["stream_" + b] = max(mem.get("stream_" + b, 0.0), mib)
            if b == "1s":
                push_ms_1s += times

    def summary(ts):
        rates = sorted(C * N / t for t in ts)
        return {"samples_per_s_median": float(np.median(rates)), "samples_per_s_min": rates[0],
                "samples_per_s_max": rates[-1], "wall_s": [round(t, 4) for t in ts]}

    p = np.array(push_ms_1s)
    result = {
        "workload": f"{C} ch x {args.minutes:g} min float32 @ {SR} Hz, stationary, default chunk_size / padding",
        "runs": args.runs,
        "arms": {k: summary(v) for k, v in arms.items()},
        "push_ms_1s_blocks": {"median": float(np.median(p)), "p90": float(np.percentile(p, 90)), "max": float(p.max()),
                              "pushes_returning_a_chunk_median": float(np.median(p[p > 3 * np.median(p)]))
                              if np.any(p > 3 * np.median(p)) else None},
        "device_mib_held_while_streaming": mem,
        "bit_equal_to_reduce_noise": equal_all,
        "card": card(),
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
