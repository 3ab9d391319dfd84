"""TorchGate.sessions() on an H100: many live sessions that start and end at their own ticks, against one TorchGateStream
per session and against a lockstep TorchGate.stream().

    python scripts/bench_torchgate_sessions.py [--rows 64 256] [--ticks 500] [--runs 3] [--out results/x.json]

The workload is a server tick loop at 16 kHz with nominal 20 ms ticks: every tick, each live row receives a number of
samples drawn uniformly from 0-640, and seeded sessions of 5-60 s start after an idle gap of 0-50 ticks and end when
their length is reached.  The arms, alternated in one process after a warm-up:
  (a) sessions()          one push(block, lengths) per tick, plus one end(rows) on ticks where sessions end;
  (b) a stream per session one TorchGateStream per live session, one push per session and tick, finish() at its end
                           (the exact result without sessions(); each stream opens its own library handle);
  (c) lockstep stream()   one push of equal 320-sample blocks per tick for all rows: the cost floor.
Tick wall time is a host clock around one tick's calls plus a device synchronise (median and p99 over the ticks of a
run).  Throughput is row-samples over the wall time of all ticks without per-tick synchronisation; the real-time factor
is the ticks' audio time over that wall time.  Every number is the median (min-max) of --runs runs.  The sessions of arms
(a) and (b) are compared in every bit, and arm (c) against tg(x)."""
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

SR, TICK = 16000, 320


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def schedule(B, ticks, seed):
    """Per tick: lengths n[B] and the rows whose session ends after it; per row: its samples, one contiguous tensor."""
    rng = np.random.default_rng(seed)
    idle = rng.integers(0, 50, size=B)
    left = np.zeros(B, dtype=np.int64)                  # samples the live session still receives (0: idle)
    total = np.zeros(B, dtype=np.int64)
    lens, ends = [], []
    for _ in range(ticks):
        start = (left == 0) & (idle == 0)
        left[start] = rng.integers(5 * SR, 60 * SR + 1, size=int(start.sum()))
        idle[(left == 0) & (idle > 0)] -= 1
        n = np.where(left > 0, np.minimum(rng.integers(0, 641, size=B), left), 0)
        left -= n
        total += n
        e = np.nonzero((n > 0) & (left == 0))[0]
        idle[e] = rng.integers(0, 51, size=e.size)
        lens.append(n)
        ends.append(e.tolist())
    g = torch.Generator(device="cuda").manual_seed(seed)
    src = [(0.1 * torch.randn(int(t), device="cuda", generator=g) +
            torch.sin(torch.arange(int(t), device="cuda") * 0.05)).contiguous() for t in total]
    return lens, ends, src


def blocks(lens, src):
    """Arm (a)'s [B, max n] block of every tick, gathered ahead of the timed loop."""
    B = len(src)
    pos = np.zeros(B, dtype=np.int64)
    out = []
    for n in lens:
        blk = torch.zeros((B, int(n.max())), device="cuda")
        for b in np.nonzero(n)[0]:
            blk[b, :n[b]] = src[b][pos[b]:pos[b] + n[b]]
        pos += n
        out.append(blk)
    return out


def arm_sessions(tg, lens, ends, blks, per_tick):
    B = len(lens[0])
    ss = tg.sessions(B)
    times, outs = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for n, e, blk in zip(lens, ends, blks):
        a = time.perf_counter()
        outs.append(ss.push(blk, n))
        if e:
            outs.append((e, ss.end(e)))
        if per_tick:
            torch.cuda.synchronize()
            times.append(time.perf_counter() - a)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ss.close()
    return wall, times, outs


def arm_streams(tg, lens, ends, src, per_tick):
    B = len(src)
    streams, pos = [None] * B, np.zeros(B, dtype=np.int64)
    times, outs = [], [[] for _ in range(B)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for n, e in zip(lens, ends):
        a = time.perf_counter()
        for b in np.nonzero(n)[0]:
            if streams[b] is None:
                streams[b] = tg.stream(1)
            outs[b].append(streams[b].push(src[b][pos[b]:pos[b] + n[b]][None]))
        for b in e:
            outs[b].append(streams[b].finish())
            outs[b].append(None)                        # (session boundary)
            streams[b] = None
        if per_tick:
            torch.cuda.synchronize()
            times.append(time.perf_counter() - a)
        pos += n
    torch.cuda.synchronize()
    return time.perf_counter() - t0, times, outs


def arm_lockstep(tg, x, per_tick):
    s = tg.stream(x.shape[0])
    times, outs = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, x.shape[1], TICK):
        a = time.perf_counter()
        outs.append(s.push(x[:, i:i + TICK]))
        if per_tick:
            torch.cuda.synchronize()
            times.append(time.perf_counter() - a)
    outs.append(s.finish())
    torch.cuda.synchronize()
    return time.perf_counter() - t0, times, outs


def sessions_of_a(outs, B):
    """Per row, the ended sessions' outputs (arm a)."""
    cur, done = [[] for _ in range(B)], [[] for _ in range(B)]
    for o in outs:
        if isinstance(o[0], list):
            rows, (y, m) = o
            for i, b in enumerate(rows):
                done[b].append(torch.cat(cur[b] + [y[i, :m[i]]]))
                cur[b] = []
        else:
            y, m = o
            for b in np.nonzero(m)[0]:
                cur[b].append(y[b, :m[b]])
    return done


def sessions_of_b(outs):
    done = []
    for row in outs:
        d, cur = [], []
        for o in row:
            if o is None:
                d.append(torch.cat(cur, 1)[0])
                cur = []
            else:
                cur.append(o)
        done.append(d)
    return done


def med(v):
    return f"{np.median(v):.4g} ({min(v):.4g}-{max(v):.4g})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--ticks", type=int, default=500)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    print(f"card: {card()}")
    tg = TorchGate(sr=SR, nonstationary=True).to("cuda")
    results = []
    for B in a.rows:
        lens, ends, src = schedule(B, a.ticks, seed=B)
        blks = blocks(lens, src)
        row_samples = int(sum(int(n.sum()) for n in lens))
        x = (0.1 * torch.randn(B, a.ticks * TICK, device="cuda") +
             torch.sin(torch.arange(a.ticks * TICK, device="cuda") * 0.05)[None]).contiguous()
        ref_c = tg(x)
        w = 50                                                        # warm-up
        arm_sessions(tg, lens[:w], [[]] * w, blks[:w], True)
        arm_streams(tg, lens[:w], [[]] * w, src, True)
        arm_lockstep(tg, x[:, :w * TICK * 4], True)
        r = {k: [] for k in ("a_tick_ms_p50", "a_tick_ms_p99", "a_wall_s", "b_tick_ms_p50", "b_tick_ms_p99", "b_wall_s",
                             "c_tick_ms_p50", "c_tick_ms_p99", "c_wall_s")}
        equal_ab = equal_c = True
        for _ in range(a.runs):
            wall, _, outs_a = arm_sessions(tg, lens, ends, blks, False)
            r["a_wall_s"].append(wall)
            wall, _, outs_b = arm_streams(tg, lens, ends, src, False)
            r["b_wall_s"].append(wall)
            sa, sb = sessions_of_a(outs_a, B), sessions_of_b(outs_b)
            equal_ab &= all(len(p) == len(q) and all(torch.equal(u, v) for u, v in zip(p, q)) for p, q in zip(sa, sb))
            del outs_a, outs_b, sa, sb
            wall, _, outs_c = arm_lockstep(tg, x, False)
            r["c_wall_s"].append(wall)
            equal_c &= torch.equal(torch.cat(outs_c, 1), ref_c)
            del outs_c
            for arm, fn in (("a", lambda: arm_sessions(tg, lens, ends, blks, True)),
                            ("b", lambda: arm_streams(tg, lens, ends, src, True)),
                            ("c", lambda: arm_lockstep(tg, x, True))):
                _, times, _ = fn()
                r[f"{arm}_tick_ms_p50"].append(1e3 * float(np.median(times)))
                r[f"{arm}_tick_ms_p99"].append(1e3 * float(np.percentile(times, 99)))
        n_sessions = sum(len(e) for e in ends)
        audio_s = a.ticks * TICK / SR
        res = dict(rows=B, ticks=a.ticks, sessions_ended=n_sessions, row_samples=row_samples, **r,
                   a_row_samples_per_s=[row_samples / w for w in r["a_wall_s"]],
                   b_row_samples_per_s=[row_samples / w for w in r["b_wall_s"]],
                   c_row_samples_per_s=[B * a.ticks * TICK / w for w in r["c_wall_s"]],
                   a_realtime_factor=[audio_s / w for w in r["a_wall_s"]],
                   b_realtime_factor=[audio_s / w for w in r["b_wall_s"]],
                   c_realtime_factor=[audio_s / w for w in r["c_wall_s"]],
                   bit_identical_a_b=bool(equal_ab), bit_identical_c_forward=bool(equal_c))
        results.append(res)
        print(f"B={B:4d} ticks={a.ticks} sessions ended={n_sessions}  bit-identical a=b: {equal_ab}, c=tg(x): {equal_c}")
        for arm, name in (("a", "sessions()"), ("b", "stream per session"), ("c", "lockstep stream()")):
            print(f"  ({arm}) {name:20s} tick {med(res[f'{arm}_tick_ms_p50'])} ms (p99 {med(res[f'{arm}_tick_ms_p99'])} ms)  "
                  f"{med(res[f'{arm}_row_samples_per_s'])} row-samples/s  real-time x{med(res[f'{arm}_realtime_factor'])}",
                  flush=True)
        del x, ref_c, blks, src
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
