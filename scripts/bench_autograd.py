"""Time reduce_noise() forward alone against forward + backward on device tensors (b200gate_adjoint).

Config 2 (64 ch x 10 min @ 48 kHz, stationary, float32) and config 3 (the same samples, non-stationary, n_fft 2048).
Arms alternate within each run; each run reports the median of `--calls` calls, and the script prints the median and
min-max over `--runs` runs, the kept-mask store size, and the card's name, power limit and max SM clock read in the same
process.  One JSON line per config on stdout."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import noisereduce_b200 as nr  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as e:                                                  # (no nvidia-smi: report what torch knows)
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--minutes", type=float, default=10.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--calls", type=int, default=3)
    a = ap.parse_args()
    sr = 48000
    n = int(a.minutes * 60 * sr)
    gen = torch.Generator(device="cuda").manual_seed(0)
    y = (torch.randn(a.channels, n, device="cuda", generator=gen) * 0.1).float()
    g = torch.randn(a.channels, n, device="cuda", generator=gen)
    info = card()
    for name, kw in (("config2", dict(stationary=True)), ("config3", dict(stationary=False, n_fft=2048))):
        res = dict(config=name, channels=a.channels, samples=n, card=info)
        try:
            yg = y.detach().requires_grad_(True)
            out = nr.reduce_noise(yg, sr=sr, **kw)
            del out
        except Exception as e:                                             # a geometry without an adjoint
            res["error"] = str(e).splitlines()[0]
            print(json.dumps(res), flush=True)
            continue
        fwd_runs, bwd_runs = [], []
        for _ in range(a.runs):
            f, b = [], []
            for _ in range(a.calls):
                f.append(timed(lambda: nr.reduce_noise(y, sr=sr, **kw)))

                def fb():
                    yg = y.detach().requires_grad_(True)
                    out = nr.reduce_noise(yg, sr=sr, **kw)
                    out.backward(g)
                b.append(timed(fb))
            fwd_runs.append(statistics.median(f))
            bwd_runs.append(statistics.median(b))
        from noisereduce_b200 import _cabi
        gate = _cabi.Gate(surface=_cabi.SURFACE_NUMPY, stationary=1 if kw.get("stationary") else 0,
                          n_fft=kw.get("n_fft", 1024), win_length=kw.get("n_fft", 1024),
                          hop_length=kw.get("n_fft", 1024) // 4, n_grad_freq=1, n_grad_time=1, chunk_size=600000,
                          padding=30000, sr=float(sr), prop_decrease=1.0, top_db=80.0)
        res.update(forward_ms=dict(median=statistics.median(fwd_runs), min=min(fwd_runs), max=max(fwd_runs)),
                   forward_backward_ms=dict(median=statistics.median(bwd_runs), min=min(bwd_runs), max=max(bwd_runs)),
                   store_bytes=gate.mask_store_bytes(a.channels, n),
                   store_bytes_per_sample=gate.mask_store_bytes(a.channels, n) / (a.channels * n))
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
