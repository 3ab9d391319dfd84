"""Generate tests/golden/torch_route.npz by running the UNMODIFIED reference's torch route,
reduce_noise(use_torch=True, device="cpu"), on the inputs of torch_route_cases() below.
Needs an unmodified checkout of the reference:   python tests/golden/make_golden_torch_route.py /path/to/noisereduce"""
import os
import sys
import warnings

import numpy as np

SR = 16000


def torch_route_cases():
    """name -> (y, y_noise or None, reduce_noise keyword arguments).  Deterministic (seeded) inputs."""
    rng = np.random.default_rng(20261016)
    n = 9000
    t = np.arange(n) / SR
    tone = np.stack([np.sin(2 * np.pi * 440 * t) * (t > 0.15), np.sin(2 * np.pi * 1250 * t) * (t < 0.4)])
    y = (0.4 * tone + 0.05 * rng.standard_normal((2, n))).astype(np.float32)
    noise = (0.05 * rng.standard_normal((2, 5000))).astype(np.float32)
    base = dict(chunk_size=3000, padding=1100, time_constant_s=0.2)
    return {
        "stationary": (y, None, dict(base, stationary=True)),
        "nonstationary": (y, None, dict(base, stationary=False, thresh_n_mult_nonstationary=1.5)),
        "stationary_y_noise": (y, noise, dict(base, stationary=True)),
        "nonstationary_512_400_100": (y, None, dict(base, stationary=False, n_fft=512, win_length=400,
                                                    hop_length=100, prop_decrease=0.8)),
        "stationary_single_chunk": (y[:, :2500], None, dict(base, stationary=True)),
    }


if __name__ == "__main__":
    REF = sys.argv[1]
    HERE = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, REF)
    warnings.filterwarnings("ignore")
    import torch
    import noisereduce as nr  # noqa: E402  (the reference)

    out = {"versions": np.array([f"reference=51c8534 v3.0.3 numpy={np.__version__} torch={torch.__version__}"])}
    for name, (y, y_noise, kw) in torch_route_cases().items():
        out[name] = nr.reduce_noise(y=y, sr=SR, y_noise=y_noise, use_torch=True, device="cpu", **kw)
        print(f"{name:32s} {out[name].dtype} {out[name].shape}")
    np.savez_compressed(os.path.join(HERE, "torch_route.npz"), **out)
