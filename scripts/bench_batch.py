"""Many short clips of different lengths: a loop of reduce_noise() against one reduce_noise_batch() call.

    python scripts/bench_batch.py [--clips 4096] [--runs 3] [--seed 0]

Workload, generated from the seed: mono float32 clips with lengths uniform in 2-30 s at 48 kHz, once as resident CUDA
tensors and once as pageable numpy arrays.  For each gate (non-stationary; stationary with a 2 s noise clip) the two arms
alternate in one process, each run ends in a device synchronise, every arm is warmed up once, and the line gives the
median (min-max) of the runs.  Both arms' outputs on the timed data must be equal in every bit.  Needs a GPU.

    python scripts/bench_batch.py --per-item [--clips 512]

runs the stationary gate with every clip its own noise clip instead: a loop of reduce_noise(y, sr, stationary=True)
against reduce_noise_batch(ys, sr, stationary=True, y_noise_per_item=[None] * clips), with the same protocol, and breaks
out the batched statistics pass (CUDA events around b200gate_noise_stats_rows), the analysis kernel time of the batch
against the shared-threshold batch on the same clips (b200gate_get_stats k1_ms), and how many workspace batches ran
the row-maximum re-analysis (kernel durations from torch.profiler, in a separate untimed call).
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
    ap.add_argument("--per-item", action="store_true", help="the stationary gate with per-item thresholds")
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

    if args.per_item:
        return per_item(args, card, lens, samples, dev, host, noise, seen, timed)
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


def per_item(args, card, lens, samples, dev, host, noise, seen, timed):
    """The stationary gate with per-item thresholds (every item its own noise clip)."""
    import torch
    import noisereduce_b200 as nr
    from noisereduce_b200 import _cabi
    stats_ms = []
    real_rows = _cabi.Gate.noise_stats_rows

    def noise_stats_rows(self, *a, **k):                   # CUDA events around the batched statistics pass
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = real_rows(self, *a, **k)
        e1.record()
        e1.synchronize()
        stats_ms.append(e0.elapsed_time(e1))
        return out

    _cabi.Gate.noise_stats_rows = noise_stats_rows
    results = []
    for where, ys in (("cuda tensors", dev), ("pageable numpy", host)):
        none = [None] * len(ys)
        arms = {"loop of reduce_noise": lambda: [nr.reduce_noise(y, SR, stationary=True) for y in ys],
                "reduce_noise_batch": lambda: nr.reduce_noise_batch(ys, SR, stationary=True, y_noise_per_item=none)}
        times = {k: [] for k in arms}
        for fn in arms.values():
            timed(fn)                                       # warm-up
        outs = {}
        for _ in range(args.runs):
            for k, fn in arms.items():                     # alternate the arms
                stats_ms.clear()
                dt, outs[k] = timed(fn)
                times[k].append(dt)
        same = all(torch.equal(x, y) if isinstance(x, torch.Tensor) else np.array_equal(x, y)
                   for x, y in zip(outs["loop of reduce_noise"], outs["reduce_noise_batch"]))
        assert same, f"{where}: the per-item batch differs from the loop"
        del outs
        st_rec = [s for stat, s in seen if stat == 1][-1]  # the last batch handle
        stat_pass = sum(stats_ms)
        seen.clear()
        y_noise = noise if ys is dev else noise.cpu().numpy()
        timed(lambda: nr.reduce_noise_batch(ys, SR, stationary=True, y_noise=y_noise))
        st_shared = [s for stat, s in seen if stat == 1][-1]
        for k in arms:
            med = statistics.median(times[k])
            results.append(dict(inputs=where, gate="stationary, per item", arm=k, median_s=med, min_s=min(times[k]),
                                max_s=max(times[k]), clips_per_s=args.clips / med, gsamples_per_s=samples / med / 1e9))
            print(f"{where:15s} {'stationary, per item':21s} {k:21s} {med:8.3f} s ({min(times[k]):.3f}-{max(times[k]):.3f})  "
                  f"{args.clips / med:9.1f} clips/s  {samples / med / 1e9:7.3f} Gsamples/s")
        ran = "not measured"
        try:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                nr.reduce_noise_batch(ys, SR, stationary=True, y_noise_per_item=none)
                torch.cuda.synchronize()
            fb = [e.device_time for e in prof.events() if "k1_analyze<8" in e.name and ", true, true, true>" in e.name]
            ran = f"{sum(t > 50.0 for t in fb)} of {len(fb)} workspace batches"
        except Exception as e:                              # (the profiler's event API differs between torch versions)
            ran = f"not measured ({type(e).__name__})"
        print(f"{'':15s} statistics pass {stat_pass:.1f} ms (last batch run); k1 {st_rec['k1_ms']:.1f} ms per-item "
              f"thresholds vs {st_shared['k1_ms']:.1f} ms shared thresholds; row-maximum re-analysis ran in {ran}; "
              f"bit-equal: {same}")
        results.append(dict(inputs=where, stats_pass_ms=stat_pass, k1_ms_per_item=st_rec["k1_ms"],
                            k1_ms_shared=st_shared["k1_ms"], rowmax_fallback=ran))
    print(json.dumps(dict(card=card, clips=args.clips, samples=samples, runs=args.runs, results=results)))


if __name__ == "__main__":
    main()
