"""TorchGate.stream() on an H100: wall time per push, sustained throughput, and one tg(x) call on the same samples.

    python scripts/bench_torchgate_stream.py [--seconds 20] [--runs 3] [--out results/bench_torchgate_stream.json]

For B rows at 16 kHz pushed in blocks of n samples, each push is timed with a host clock around push() plus a device
synchronise (median and p99 over the pushes of a run).  Throughput counts row-samples over the wall time of all pushes
and finish() without per-push synchronisation; the real-time factor is audio seconds over wall seconds.  The stream and
tg(x) arms alternate in one process after a warm-up; every number is the median (min-max) of --runs runs.  The outputs of
the two arms are compared in every bit in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from noisereduce_b200.torchgate import TorchGate  # noqa: E402

SR = 16000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def stream_run(tg, x, n, per_push):
    B, L = x.shape
    s = tg.stream(B)
    times, outs = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, L, n):
        if per_push:
            a = time.perf_counter()
            outs.append(s.push(x[:, i:i + n]))
            torch.cuda.synchronize()
            times.append(time.perf_counter() - a)
        else:
            outs.append(s.push(x[:, i:i + n]))
    outs.append(s.finish())
    torch.cuda.synchronize()
    return time.perf_counter() - t0, times, outs


def forward_run(tg, x):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    y = tg(x)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, y


def med(v):
    return f"{np.median(v):.4g} ({min(v):.4g}-{max(v):.4g})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--rows", type=int, nargs="+", default=[1, 64, 256])
    ap.add_argument("--blocks", type=int, nargs="+", default=[320, 1024, 4096])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    print(f"card: {card()}")
    tg = TorchGate(sr=SR, nonstationary=True).to("cuda")
    L = int(a.seconds * SR)
    results = []
    for B in a.rows:
        g = torch.Generator(device="cuda").manual_seed(B)
        x = (0.1 * torch.randn(B, L, device="cuda", generator=g) +
             torch.sin(torch.arange(L, device="cuda") * 0.05)[None]).contiguous()
        _, ref = forward_run(tg, x)                                  # warm-up
        for n in a.blocks:
            stream_run(tg, x[:, :SR], n, False)                      # warm-up
            wall, push_p50, push_p99, fwd = [], [], [], []
            equal = True
            for _ in range(a.runs):
                w, _, outs = stream_run(tg, x, n, False)
                equal &= torch.equal(torch.cat(outs, 1), ref)
                wall.append(w)
                _, times, outs = stream_run(tg, x, n, True)
                equal &= torch.equal(torch.cat(outs, 1), ref)
                push_p50.append(1e3 * float(np.median(times)))
                push_p99.append(1e3 * float(np.percentile(times, 99)))
                f, y = forward_run(tg, x)
                equal &= torch.equal(y, ref)
                fwd.append(f)
            r = dict(rows=B, block=n, seconds=a.seconds, push_ms_p50=push_p50, push_ms_p99=push_p99, stream_wall_s=wall,
                     row_samples_per_s=[B * L / w for w in wall], realtime_factor=[a.seconds / w for w in wall],
                     forward_s=fwd, forward_row_samples_per_s=[B * L / f for f in fwd], bit_identical=bool(equal))
            results.append(r)
            print(f"B={B:4d} block={n:5d}: push {med(push_p50)} ms (p99 {med(push_p99)} ms)  "
                  f"stream {med(r['row_samples_per_s'])} row-samples/s, real-time x{med(r['realtime_factor'])}  "
                  f"tg(x) {med(r['forward_row_samples_per_s'])} row-samples/s  bit-identical={equal}", flush=True)
        del x, ref
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
