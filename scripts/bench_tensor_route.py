#!/usr/bin/env python
"""Cost of reduce_noise() on a CUDA tensor: config 2's data (64 ch x 10 min, 48 kHz, float32) resident on the GPU.

    python scripts/bench_tensor_route.py [--runs 3] [--calls 10] [--minutes 10] [--out result.json]

Arms, alternated in one process, each timed by the host clock around a synchronised call:
  tensor_f32        reduce_noise(y_cuda, sr, stationary=True), end to end (handle, thresholds, gate, output tensor);
  device_gate       DeviceGate.run(x, out) with the library's default workspace limit (thresholds set once, untimed);
  device_gate_64g   the same with bench.py's 64 GB workspace limit;
  thresholds        DeviceGate.noise_stats(x) alone (the threshold computation the tensor route adds);
  numpy_pageable    reduce_noise() on the same samples as a pageable numpy array;
  tensor_f16        reduce_noise() on the samples as a float16 CUDA tensor (promote, gate in float64, cast back);
  tensor_i16        reduce_noise() on the samples as an int16 CUDA tensor (read by the kernels as they are).
Per arm: the median over runs of the median of `calls` calls, and the range of the per-run medians.  tensor_f32's steps
are also timed one by one on SpectralGateStationary (construction with the thresholds, first and second get_traces(),
destruction of the handle): median, min and max over all calls.  Also prints the
largest difference of tensor_f32's output from DeviceGate.run's (0 expected), the card and its power limit, as one
JSON object.
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
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import noisereduce_b200 as nr
    from noisereduce_b200.device import DeviceGate

    C, N = 64, int(args.minutes * 60 * SR)
    y_np = synth_host(np, C, N)
    x = torch.from_numpy(y_np).cuda()
    x16 = x.to(torch.float16)
    xi16 = torch.from_numpy(np.round(y_np * 20000).astype(np.int16)).cuda()
    kw = dict(sr=SR, stationary=True)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    # largest difference from DeviceGate.run (outside the timed calls)
    dg = DeviceGate(**kw)
    dg.noise_stats(x)
    ref = dg.run(x)
    got = nr.reduce_noise(x, **kw)
    max_diff_f32 = float((got - ref).abs().max().item())
    same_nan = bool(torch.equal(torch.isnan(got), torch.isnan(ref)))
    del got, ref, dg
    torch.cuda.empty_cache()

    def gate_arm(limit):
        dg = DeviceGate(**kw, workspace_limit_bytes=limit)
        dg.noise_stats(x)
        out = torch.empty_like(x)
        dg.run(x, out)                                  # workspace sized outside the timed calls
        ts = [timed(lambda: dg.run(x, out))[0] for _ in range(args.calls)]
        th = [timed(lambda: dg.noise_stats(x))[0] for _ in range(args.calls)] if limit == 0 else None
        return ts, th

    def route_arm(y):
        ts = []
        for _ in range(args.calls):
            t, r = timed(lambda: nr.reduce_noise(y, **kw))
            ts.append(t)
            del r
        return ts

    from noisereduce_b200.spectralgate import SpectralGateStationary
    cls_args = dict(sr=SR, y_noise=None, n_std_thresh_stationary=1.5, chunk_size=600000, clip_noise_stationary=True,
                    padding=30000, n_fft=1024, win_length=None, hop_length=None, time_constant_s=2.0,
                    freq_mask_smooth_hz=500, time_mask_smooth_ms=50, tmp_folder=None, prop_decrease=1.0,
                    use_tqdm=False, n_jobs=1)

    def steps_arm():
        """tensor_f32's steps one by one: construction (handle + thresholds), the first get_traces() (which sizes the
        workspace), a second get_traces() on the same object, and the handle's destruction."""
        rows = {"construct": [], "first_get_traces": [], "second_get_traces": [], "destroy": []}
        for _ in range(args.calls):
            t, sg = timed(lambda: SpectralGateStationary(y=x, **cls_args))
            rows["construct"].append(t)
            for k in ("first_get_traces", "second_get_traces"):
                t, r = timed(lambda: sg.get_traces())
                rows[k].append(t)
                del r
            rows["destroy"].append(timed(lambda: sg._gate.close())[0])
            del sg
        return rows

    arms = {k: [] for k in ("tensor_f32", "device_gate", "device_gate_64g", "thresholds", "numpy_pageable",
                            "tensor_f16", "tensor_i16")}
    steps = {k: [] for k in ("construct", "first_get_traces", "second_get_traces", "destroy")}
    nr.reduce_noise(x16[:, :1_300_000], **kw)          # warm-up: kernels loaded
    for _ in range(args.runs):
        arms["tensor_f32"].append(route_arm(x))
        torch.cuda.empty_cache()
        for k, v in steps_arm().items():
            steps[k].append(v)
        torch.cuda.empty_cache()
        ts, th = gate_arm(0.0)
        arms["device_gate"].append(ts)
        arms["thresholds"].append(th)
        torch.cuda.empty_cache()
        arms["device_gate_64g"].append(gate_arm(64e9)[0])
        torch.cuda.empty_cache()
        arms["numpy_pageable"].append(route_arm(y_np))
        arms["tensor_f16"].append(route_arm(x16))
        torch.cuda.empty_cache()
        arms["tensor_i16"].append(route_arm(xi16))
        torch.cuda.empty_cache()

    def summary(runs):
        med = sorted(float(np.median(r)) * 1e3 for r in runs)
        return {"ms_median": float(np.median(med)), "ms_run_medians": [round(m, 2) for m in med],
                "gsamples_per_s": C * N / (float(np.median(med)) * 1e-3) / 1e9}

    result = {
        "workload": f"{C} ch x {args.minutes:g} min @ {SR} Hz, stationary, default chunk_size / padding; "
                    f"{args.runs} runs x {args.calls} calls",
        "arms": {k: summary(v) for k, v in arms.items()},
        "tensor_f32_steps_ms": {k: {"median": float(np.median(v)) * 1e3, "min": float(np.min(v)) * 1e3,
                                    "max": float(np.max(v)) * 1e3} for k, v in steps.items()},
        "tensor_f32_max_abs_diff_from_device_gate": max_diff_f32,
        "tensor_f32_same_nan_as_device_gate": same_nan,
        "card": card(),
    }
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
