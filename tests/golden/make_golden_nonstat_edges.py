"""Generate tests/golden/nonstat_edges*.npz by running the UNMODIFIED reference on the inputs defined below: TorchGate
(moving-mean follower) and reduce_noise(use_torch=True) on rows with runs of digital silence, the numpy surface on a
silent padded chunk and on a single NaN sample, and two quiet-then-loud inputs of the IIR follower.  Needs an
unmodified checkout of the reference:   python tests/golden/make_golden_nonstat_edges.py /path/to/noisereduce

NaN-heavy outputs are stored as their NaN pattern (np.packbits of np.isnan); the finite samples are compared with
oracle/ in the tests.  The arrays are split over files of less than 1 MB (tests/parity_cases.load_golden)."""
import os
import sys
import warnings

import numpy as np

SR = 16000
HOP = 256
TG_L = 64 * HOP
SILENCE_FRAMES = (19, 20, 21, 22, 23)         # n_movemean - 1 .. n_movemean + 3 (default n_movemean 20)
TG_SMOOTHING = {"f500_t50": dict(), "fNone_t50": dict(freq_mask_smooth_hz=None),
                "f500_tNone": dict(time_mask_smooth_ms=None),
                "fNone_tNone": dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None)}


def silence_rows(start_frame, scale_left=1.0, scale_right=1.0, seed=0):
    """[5, TG_L] float64: row i has exact zeros on every sample that reaches frames start_frame ..
    start_frame + SILENCE_FRAMES[i] - 1 of the centred 1024-point STFT, noise elsewhere (scale_left before
    the silence, scale_right after it)."""
    rng = np.random.default_rng(seed)
    x = 0.05 * rng.standard_normal((len(SILENCE_FRAMES), TG_L))
    for i, k in enumerate(SILENCE_FRAMES):
        z0, z1 = start_frame * HOP - 512, (start_frame + k - 1) * HOP + 512
        x[i, :z0] *= scale_left
        x[i, z1:] *= scale_right
        x[i, z0:z1] = 0.0
    return x


def torchgate_inputs():
    """name -> [5, TG_L] float64 rows (cast to float32 for the float32 cases)."""
    return {
        "even": silence_rows(20, seed=1),
        "odd": silence_rows(21, seed=2),
        # content on the two sides 1e9 apart in amplitude (more than 2^29): the follower's running sum must
        # still return exactly zero on all-zero windows
        "loud_quiet": silence_rows(21, scale_left=2e4, scale_right=2e-5, seed=3),
        "quiet_loud": silence_rows(20, scale_left=2e-5, scale_right=2e4, seed=4),
    }


def torch_route_inputs():
    """name -> (y [C, n] float32, reduce_noise kwargs) for reduce_noise(use_torch=True, stationary=False)."""
    rng = np.random.default_rng(7)
    n, cs, pad = 12000, 3000, 1100
    y = (0.05 * rng.standard_normal((3, n))).astype(np.float32)
    y[0, 4000:9000] = 0.0                             # a run of silence crossing a chunk border
    y[1, 3000 - pad: 6000 + pad] = 0.0                # the second padded chunk entirely silent
    y[2, 7000:7000 + 21 * HOP] = 0.0
    return {"silences": (y, dict(chunk_size=cs, padding=pad, stationary=False, time_constant_s=0.2))}


def numpy_nan_inputs():
    """name -> (y, y_noise or None, reduce_noise kwargs) for the numpy surface."""
    rng = np.random.default_rng(11)
    n, cs, pad = 30000, 6000, 1000
    loud = (0.3 * rng.standard_normal((2, n))).astype(np.float32)
    silent_chunk = loud.copy()
    silent_chunk[:, 2 * cs - pad: 3 * cs + pad] = 0.0   # padded chunk 2 made entirely of silence
    nan_even = loud.copy()
    nan_even[0, 13900] = np.nan                          # chunk 2, padded-chunk sample 2900: frames 10..13
    nan_odd = loud.copy()
    nan_odd[1, 14100] = np.nan                           # padded-chunk sample 3100: frames 11..14
    noise = (0.3 * rng.standard_normal((2, 8000))).astype(np.float32)
    base = dict(chunk_size=cs, padding=pad, time_constant_s=0.25)
    return {
        "silent_chunk_nonstat": (silent_chunk, None, dict(base, stationary=False)),
        "silent_chunk_stat": (silent_chunk, noise, dict(base, stationary=True)),
        "nan_even_nonstat": (nan_even, None, dict(base, stationary=False)),
        "nan_odd_nonstat": (nan_odd, None, dict(base, stationary=False)),
        "nan_even_stat": (nan_even, noise, dict(base, stationary=True)),
        "nan_odd_stat": (nan_odd, noise, dict(base, stationary=True)),
    }


def quiet_then_loud(n, split, n_clicks=60, seed=5, scale=0.3, dtype=np.float32):
    """Exact zeros before `split` with log-spaced clicks (1e-6 .. 1e-2, shuffled) every 1100 samples from
    sample 1000, scale * N(0, 1) from `split` on."""
    rng = np.random.default_rng(seed)
    y = np.zeros(n)
    y[split:] = scale * rng.standard_normal(n - split)
    amps = rng.permutation(np.logspace(-6, -2, n_clicks))
    pos = 1000 + 1100 * np.arange(n_clicks)
    keep = pos < split
    y[pos[keep]] += amps[keep]
    return y.astype(dtype)


def iir_inputs():
    """name -> (y [n] float32, reduce_noise kwargs): quiet-then-loud columns for the IIR follower (sim-sized)."""
    return {
        "qtl_1024": (quiet_then_loud(48000, 30000, n_clicks=26),
                     dict(stationary=False, chunk_size=None, padding=1000, time_constant_s=0.15)),
        "qtl_2048": (quiet_then_loud(80000, 50000, n_clicks=44),
                     dict(stationary=False, chunk_size=None, padding=1000, time_constant_s=0.3, n_fft=2048)),
    }


def nan_bits(a):
    return np.packbits(np.isnan(np.asarray(a)).ravel())


if __name__ == "__main__":
    REF = sys.argv[1]
    HERE = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, REF)
    warnings.filterwarnings("ignore")
    import torch
    import noisereduce as nr  # noqa: E402  (the reference)
    from noisereduce.torchgate import TorchGate  # noqa: E402

    parts = [{"versions": np.array([f"reference=51c8534 v3.0.3 numpy={np.__version__} torch={torch.__version__}"])}]
    for name, x in torchgate_inputs().items():
        for sm, kw in TG_SMOOTHING.items():
            for dt in (torch.float32, torch.float64):
                tg = TorchGate(sr=SR, nonstationary=True, **kw)
                with torch.no_grad():
                    out = tg(torch.from_numpy(x).to(dt)).numpy()
                key = f"tg_{name}_{sm}_{'f32' if dt == torch.float32 else 'f64'}"
                parts[0][key + "_nan"] = nan_bits(out)
                print(f"{key:40s} NaN samples {int(np.isnan(out).sum())}")
    arrays = {}
    for name, (y, kw) in torch_route_inputs().items():
        arrays[f"route_{name}"] = nr.reduce_noise(y=y, sr=SR, use_torch=True, device="cpu", **kw)
    for name, (y, y_noise, kw) in numpy_nan_inputs().items():
        arrays[f"np_{name}"] = nr.reduce_noise(y=y, sr=SR, y_noise=y_noise, **kw)
    for name, (y, kw) in iir_inputs().items():
        arrays[f"iir_{name}"] = nr.reduce_noise(y=y, sr=SR, **kw)
    for key, r in arrays.items():
        print(f"{key:40s} {r.dtype} {r.shape} NaN samples {int(np.isnan(r).sum())}")
        if sum(v.nbytes for v in parts[-1].values()) + r.nbytes > 900_000:
            parts.append({})
        parts[-1][key] = r
    for i, p in enumerate(parts):
        fn = os.path.join(HERE, "nonstat_edges.npz" if i == 0 else f"nonstat_edges_{i + 1}.npz")
        np.savez_compressed(fn, **p)
        print(fn, os.path.getsize(fn))
