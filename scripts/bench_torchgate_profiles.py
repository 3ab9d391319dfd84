"""TorchGate.sessions(profiles=...) on an H100: rows at 8, 16 and 48 kHz in one sessions object, against one
single-profile object per sample rate.

    python scripts/bench_torchgate_profiles.py [--rows 64 256] [--ticks 500] [--runs 3] [--out results/x.json]

The workload is the tick loop of scripts/bench_torchgate_sessions.py at three sample rates: row b is on profile b % 3
(8 kHz; 16 kHz; 48 kHz with prop_decrease 0.7) and, every 20 ms tick, each live row receives a number of samples drawn
uniformly from 0 to twice its rate's 20 ms; seeded sessions of 5-60 s start after an idle gap of 0-50 ticks and end when
their length is reached.  The arms, alternated in one process after a warm-up:
  (a) profiles            one sessions() object with the 3 profiles: one push(block, lengths) per tick, plus one
                          end(rows) on ticks where sessions end;
  (b) one per profile     three single-profile sessions() objects, each holding the rows of one profile: three pushes
                          per tick and up to three end() calls (the exact result without profiles);
  (c) one profile         one single-profile (16 kHz) object taking the same blocks: the cost floor of a tick.
Tick wall time is a host clock around one tick's calls plus a device synchronise (median and p99 over the ticks of a
run).  Throughput is row-samples over the wall time of all ticks without per-tick synchronisation; the real-time factor
is the ticks' audio time over that wall time.  Every number is the median (min-max) of --runs runs.  The sessions of arms
(a) and (b) are compared in every bit."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_torchgate_sessions import card, med  # noqa: E402
from noisereduce_b200.torchgate import TorchGate  # noqa: E402

PROFILES = [dict(sr=8000), dict(sr=16000), dict(sr=48000, prop_decrease=0.7)]
RATES = np.array([8000, 16000, 48000])


def schedule(B, ticks, seed):
    """Per tick: lengths n[B] and the rows whose session ends after it; per row: its samples, one contiguous tensor."""
    rng = np.random.default_rng(seed)
    rate = RATES[np.arange(B) % 3]
    idle = rng.integers(0, 50, size=B)
    left = np.zeros(B, dtype=np.int64)                  # samples the live session still receives (0: idle)
    total = np.zeros(B, dtype=np.int64)
    lens, ends = [], []
    for _ in range(ticks):
        start = (left == 0) & (idle == 0)
        left[start] = (rng.uniform(5, 60, size=int(start.sum())) * rate[start]).astype(np.int64)
        idle[(left == 0) & (idle > 0)] -= 1
        n = np.where(left > 0, np.minimum((rng.uniform(0, 1, size=B) * rate * 0.04).astype(np.int64), left), 0)
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


def blocks(lens, src, rows):
    """The [len(rows), max n] block of the listed rows for every tick, gathered ahead of the timed loop."""
    pos = np.zeros(len(src), dtype=np.int64)
    out = []
    for n in lens:
        nr = n[rows]
        blk = torch.zeros((len(rows), int(nr.max()) if nr.size else 0), device="cuda")
        for i, b in enumerate(rows):
            if n[b]:
                blk[i, :n[b]] = src[b][pos[b]:pos[b] + n[b]]
        pos += n
        out.append(blk)
    return out


def arm(objs, groups, lens, ends, blks, per_tick):
    """objs[j] holds rows groups[j]; blks[j][tick] is its block.  Returns wall, tick times and, per row, its outputs."""
    B = len(lens[0])
    local = np.zeros(B, dtype=np.int64)
    owner = np.zeros(B, dtype=np.int64)
    for j, g in enumerate(groups):
        local[g] = np.arange(len(g))
        owner[g] = j
    times, outs = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k, (n, e) in enumerate(zip(lens, ends)):
        a = time.perf_counter()
        for j, (ss, g) in enumerate(zip(objs, groups)):
            outs.append((j, ss.push(blks[j][k], n[g])))
        for j, ss in enumerate(objs):
            rows = [int(local[b]) for b in e if owner[b] == j]
            if rows:
                outs.append((j, rows, ss.end(rows)))
        if per_tick:
            torch.cuda.synchronize()
            times.append(time.perf_counter() - a)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, times, outs


def sessions_of(outs, groups, B):
    """Per global row, the ended sessions' outputs."""
    cur, done = [[] for _ in range(B)], [[] for _ in range(B)]
    for o in outs:
        if len(o) == 3:
            j, rows, (y, m) = o
            for i, r in enumerate(rows):
                b = groups[j][r]
                done[b].append(torch.cat(cur[b] + [y[i, :m[i]]]))
                cur[b] = []
        else:
            j, (y, m) = o
            for r in np.nonzero(m)[0]:
                cur[groups[j][r]].append(y[r, :m[r]])
    return done


def run_arm(name, tg, B, lens, ends, blk_all, blk_per, per_tick):
    everyone = np.arange(B)
    if name == "a":
        ss = tg.sessions(B, profiles=PROFILES)
        for k in range(3):
            ss.assign(everyone[everyone % 3 == k].tolist(), k)
        objs, groups, blks = [ss], [everyone], [blk_all]
    elif name == "b":
        groups = [everyone[everyone % 3 == k] for k in range(3)]
        objs = [tg.sessions(len(g), profiles=[p]) for g, p in zip(groups, PROFILES)]
        blks = blk_per
    else:
        objs, groups, blks = [tg.sessions(B)], [everyone], [blk_all]
    res = arm(objs, groups, lens, ends, blks, per_tick)
    for ss in objs:
        ss.close()
    return res, groups


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
    tg = TorchGate(sr=16000, nonstationary=True).to("cuda")
    results = []
    for B in a.rows:
        lens, ends, src = schedule(B, a.ticks, seed=B)
        everyone = np.arange(B)
        blk_all = blocks(lens, src, everyone)
        blk_per = [blocks(lens, src, everyone[everyone % 3 == k]) for k in range(3)]
        row_samples = int(sum(int(n.sum()) for n in lens))
        w = 50                                                        # warm-up
        for name in "abc":
            run_arm(name, tg, B, lens[:w], [[]] * w, blk_all[:w], [b[:w] for b in blk_per], True)
        r = {f"{x}_{k}": [] for x in "abc" for k in ("tick_ms_p50", "tick_ms_p99", "wall_s")}
        equal_ab = True
        for _ in range(a.runs):
            done = {}
            for name in "abc":
                (wall, _, outs), groups = run_arm(name, tg, B, lens, ends, blk_all, blk_per, False)
                r[f"{name}_wall_s"].append(wall)
                if name != "c":
                    done[name] = sessions_of(outs, groups, B)
                del outs
            equal_ab &= all(len(p) == len(q) and all(torch.equal(u, v) for u, v in zip(p, q))
                            for p, q in zip(done["a"], done["b"]))
            del done
            for name in "abc":
                (_, times, _), _ = run_arm(name, tg, B, lens, ends, blk_all, blk_per, True)
                r[f"{name}_tick_ms_p50"].append(1e3 * float(np.median(times)))
                r[f"{name}_tick_ms_p99"].append(1e3 * float(np.percentile(times, 99)))
        n_sessions = sum(len(e) for e in ends)
        audio_s = a.ticks * 0.02
        res = dict(rows=B, ticks=a.ticks, sessions_ended=n_sessions, row_samples=row_samples, **r,
                   **{f"{x}_row_samples_per_s": [row_samples / t for t in r[f"{x}_wall_s"]] for x in "abc"},
                   **{f"{x}_realtime_factor": [audio_s / t for t in r[f"{x}_wall_s"]] for x in "abc"},
                   bit_identical_a_b=bool(equal_ab))
        results.append(res)
        print(f"B={B:4d} ticks={a.ticks} sessions ended={n_sessions}  bit-identical a=b: {equal_ab}")
        for x, name in (("a", "3 profiles, 1 object"), ("b", "1 object per profile"), ("c", "1 profile (floor)")):
            print(f"  ({x}) {name:22s} tick {med(res[f'{x}_tick_ms_p50'])} ms (p99 {med(res[f'{x}_tick_ms_p99'])} ms)  "
                  f"{med(res[f'{x}_row_samples_per_s'])} row-samples/s  real-time x{med(res[f'{x}_realtime_factor'])}",
                  flush=True)
        del blk_all, blk_per, src
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
