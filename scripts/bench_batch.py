"""Many short clips of different lengths: a loop of reduce_noise() against one reduce_noise_batch() call.

    python scripts/bench_batch.py [--clips 4096] [--runs 3] [--seed 0]

Workload, generated from the seed: mono float32 clips with lengths uniform in 2-30 s at 48 kHz, once as resident CUDA
tensors and once as pageable numpy arrays.  For each gate (non-stationary; stationary with a 2 s noise clip) the two arms
alternate in one process, each run ends in a device synchronise, every arm is warmed up once, and the line gives the
median (min-max) of the runs.  Both arms' outputs on the timed data must be equal in every bit.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SR = 48000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=4096)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_batch.py needs a CUDA device")
    import noisereduce_b200 as nr
    from noisereduce_b200 import _cabi

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}")
    rng = np.random.default_rng(args.seed)
    lens = rng.integers(2 * SR, 30 * SR + 1, args.clips)
    samples = int(lens.sum())
    gen = torch.Generator(device="cuda").manual_seed(args.seed)
    dev = []
    for n in lens.tolist():
        t = torch.arange(n, device="cuda", dtype=torch.float32) / SR
        dev.append(0.05 * torch.randn(n, device="cuda", generator=gen) + 0.3 * ((t % 1.0) < 0.4) * torch.sin(2764.6 * t))
    host = [y.cpu().numpy() for y in dev]
    noise = dev[0][: 2 * SR].clone()
    print(f"{args.clips} clips, {samples / 1e6:.1f} M samples ({samples * 4 / 2**30:.2f} GiB), seed {args.seed}")

    # workspace of the batch call: what b200gate_run_rows carves per unit at the pitch of the longest unit, against
    # the frames the units really have (b200gate_get_stats)
    real_close, seen = _cabi.Gate.close, []

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            seen.append((self.params.stationary, self.stats()))
        real_close(self)

    _cabi.Gate.close = close

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    results = []
    for where, ys in (("cuda tensors", dev), ("pageable numpy", host)):
        for gate, kw in (("non-stationary", {}), ("stationary + y_noise", dict(stationary=True, y_noise=noise if ys is dev else noise.cpu().numpy()))):
            arms = {"loop of reduce_noise": lambda: [nr.reduce_noise(y, SR, **kw) for y in ys],
                    "reduce_noise_batch": lambda: nr.reduce_noise_batch(ys, SR, **kw)}
            times = {k: [] for k in arms}
            for k, fn in arms.items():
                timed(fn)                                   # warm-up
            outs = {}
            for _ in range(args.runs):
                for k, fn in arms.items():                 # alternate the arms
                    dt, outs[k] = timed(fn)
                    times[k].append(dt)
            a, b = outs["loop of reduce_noise"], outs["reduce_noise_batch"]
            same = all(torch.equal(x, y) if isinstance(x, torch.Tensor) else np.array_equal(x, y) for x, y in zip(a, b))
            assert same, f"{where} / {gate}: the batch differs from the loop"
            del outs, a, b
            st = [s for stat, s in seen if stat == (1 if kw else 0)][-1]     # the last batch handle of this gate
            for k in arms:
                med = statistics.median(times[k])
                results.append(dict(inputs=where, gate=gate, arm=k, median_s=med, min_s=min(times[k]), max_s=max(times[k]),
                                    clips_per_s=args.clips / med, gsamples_per_s=samples / med / 1e9))
                print(f"{where:15s} {gate:21s} {k:21s} {med:8.3f} s ({min(times[k]):.3f}-{max(times[k]):.3f})  "
                      f"{args.clips / med:9.1f} clips/s  {samples / med / 1e9:7.3f} Gsamples/s")
            t_max = int(max((min(n, 600000) + 60000) // 256 + 1 for n in lens.tolist()))     # reduce_noise()'s chunk grid
            print(f"{'':15s} {gate:21s} batch: {st['units']} units, {st['frames']} frames; pitch {t_max} frames -> "
                  f"{100.0 * (1 - st['frames'] / (st['units'] * t_max)):.1f} % of the per-unit workspace is padding; bit-equal: {same}")
    print(json.dumps(dict(card=card, clips=args.clips, samples=samples, runs=args.runs, results=results)))


if __name__ == "__main__":
    main()
