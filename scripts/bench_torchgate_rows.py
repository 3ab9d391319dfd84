"""A padded TorchGate batch of rows of different lengths: a loop of per-row forward() against forward(x, lengths=...).

    python scripts/bench_torchgate_rows.py [--rows 256] [--runs 3] [--seed 7]

Workload, generated from the seed: `rows` float32 rows zero-padded to 10 s at 16 kHz, lengths uniform in 1-10 s (the
batch of BASELINE config 4 with lengths), resident on the GPU.  For each gate three arms are timed: (a) a loop of
forward(x[b:b+1, :lengths[b]]), (b) forward(x, lengths=lengths), (c) forward(x) on the padded batch, the cost floor
(it gates the padding too and is not the same result).  (a) and (b) are also timed with backward() of sum(y * g).
The arms alternate in one process, every arm is warmed up once, each run ends in a device synchronise, and the line
gives the median (min-max) of the runs.  (a) and (b) must agree in every bit on the timed data.  Needs a GPU.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SR, HOP = 16000, 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_torchgate_rows.py needs a CUDA device")
    from noisereduce_b200.torchgate import TorchGate

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}")
    B, Lmax = args.rows, 10 * SR
    lengths = torch.randint(SR, Lmax + 1, (B,), generator=torch.Generator().manual_seed(args.seed)).tolist()
    gen = torch.Generator(device="cuda").manual_seed(args.seed)
    t = torch.arange(Lmax, device="cuda", dtype=torch.float32) / SR
    x = 0.05 * torch.randn((B, Lmax), device="cuda", generator=gen) + 0.3 * ((t % 1.0) < 0.4) * torch.sin(2764.6 * t)
    x[torch.arange(Lmax, device="cuda")[None, :] >= torch.tensor(lengths, device="cuda")[:, None]] = 0.0
    g = torch.randn((B, (Lmax // HOP) * HOP), device="cuda", generator=gen)
    samples = sum(lengths)
    print(f"{B} rows padded to {Lmax} samples, {samples / 1e6:.1f} M real samples, seed {args.seed}")

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    results = []
    for gate, kw in (("stationary", {}), ("non-stationary", dict(nonstationary=True))):
        tg = TorchGate(sr=SR, **kw)

        def loop_fwd():
            with torch.no_grad():
                return [tg(x[b:b + 1, :n])[0] for b, n in enumerate(lengths)]

        def rows_fwd():
            with torch.no_grad():
                return tg(x, lengths=lengths)

        def padded_fwd():
            with torch.no_grad():
                return tg(x)

        def loop_bwd():
            grads = []
            for b, n in enumerate(lengths):
                xb = x[b:b + 1, :n].clone().requires_grad_(True)
                yb = tg(xb)
                (yb * g[b:b + 1, :yb.shape[1]]).sum().backward()
                grads.append(xb.grad[0])
            return grads

        def rows_bwd():
            xg = x.clone().requires_grad_(True)
            (tg(xg, lengths=lengths) * g).sum().backward()
            return xg.grad

        arms = {"(a) loop of forward": loop_fwd, "(b) forward(lengths=)": rows_fwd, "(c) forward(padded)": padded_fwd,
                "(a) loop fwd+bwd": loop_bwd, "(b) lengths= fwd+bwd": rows_bwd}
        times = {k: [] for k in arms}
        for fn in arms.values():
            timed(fn)                                           # warm-up
        outs = {}
        for _ in range(args.runs):
            for k, fn in arms.items():                         # alternate the arms
                dt, outs[k] = timed(fn)
                times[k].append(dt)
        a, b = outs["(a) loop of forward"], outs["(b) forward(lengths=)"]
        same_fwd = all(torch.equal(b[i, :(n // HOP) * HOP], a[i]) and not bool(b[i, (n // HOP) * HOP:].any())
                       for i, n in enumerate(lengths))
        ga, gb = outs["(a) loop fwd+bwd"], outs["(b) lengths= fwd+bwd"]
        same_bwd = all(torch.equal(gb[i, :n], ga[i]) for i, n in enumerate(lengths))
        worst_bwd = max(float((gb[i, :n] - ga[i]).abs().max() / ga[i].abs().max().clamp_min(1e-30))
                        for i, n in enumerate(lengths))
        assert same_fwd, f"{gate}: forward(lengths=) differs from the loop"
        del outs, a, b, ga, gb
        for k in arms:
            med = statistics.median(times[k])
            results.append(dict(gate=gate, arm=k, median_s=med, min_s=min(times[k]), max_s=max(times[k])))
            print(f"{gate:15s} {k:22s} {med * 1e3:9.2f} ms ({min(times[k]) * 1e3:.2f}-{max(times[k]) * 1e3:.2f})")
        print(f"{gate:15s} forward bit-equal: {same_fwd}; backward bit-equal: {same_bwd} "
              f"(largest relative difference {worst_bwd:.2e})")
        results.append(dict(gate=gate, forward_bit_equal=same_fwd, backward_bit_equal=same_bwd, backward_max_rel=worst_bwd))
    print(json.dumps(dict(card=card, rows=B, samples=samples, runs=args.runs, results=results)))


if __name__ == "__main__":
    main()
