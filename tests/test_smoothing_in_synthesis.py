"""Stationary mask smoothing inside the synthesis kernel (k2c_synthesize kMaskBits*) against the separate smoothing kernel
(path_flags bit 8: k_smooth_packed writes uint16 numerators, k2c_synthesize kMaskU16* reads them back).

Both compute the same integer numerators and share everything downstream, so the outputs and the tapped masks must be
EQUAL, not merely close.  The simulator cases run the .cu sources on the CPU; the gpu-marked ones the nvcc build."""
import numpy as np
import pytest

from noisereduce_b200 import _cabi
from oracle import spectral_gate_oracle as O
from tests import parity_cases as P
from tests.cusim_util import cusim_library
from tests.synth_host import synth_small, synth_torchgate

SEPARATE = 256          # path_flags bit 8: separate smoothing kernel


def _run(lib, y, cfg, tap_unit, path_flags, y_noise=None):
    gate = _cabi.Gate(lib=lib, **P.gate_params(cfg, path_flags=path_flags))
    gate.noise_stats_host(y if y_noise is None else y_noise)
    gate.debug_select_unit(*tap_unit)
    out = gate.run_host(y)
    d = gate.debug_read()
    stats = gate.stats()
    gate.close()
    return out, d["mask"], stats


def _assert_same(lib, y, cfg, units, y_noise=None):
    for unit in units:
        out_a, mask_a, st_a = _run(lib, y, cfg, unit, 0, y_noise)
        out_b, mask_b, st_b = _run(lib, y, cfg, unit, SEPARATE, y_noise)
        assert out_a.dtype == y.dtype and np.array_equal(out_a, out_b), unit
        assert mask_a.any() and np.array_equal(mask_a, mask_b), unit
        assert st_a["rowfloor_flags"] == st_b["rowfloor_flags"]
    return st_a


def _torchgate_same(lib, x, to_dev, from_dev, **kw):
    """TorchGate surface (one unit per row, no chunking): forward, then the reuse_masks adjoint on another signal."""
    import torch
    B, L = x.shape
    Lo = (L // 256) * 256
    outs = []
    for fl in (0, SEPARATE):
        nf, nt = 16, 3                                   # TorchGate(sr=16000) defaults: 33 x 7 filter
        gate = _cabi.Gate(lib=lib, surface=_cabi.SURFACE_TORCH, stationary=1, n_fft=1024, win_length=1024, hop_length=256,
                          n_grad_freq=nf, n_grad_time=nt, std_ddof=1, chunk_size=0, padding=0, sr=16000.0,
                          prop_decrease=kw.get("prop_decrease", 1.0), n_std_thresh=1.5, top_db=40.0, n_movemean=20,
                          thresh_n_mult=1.0, sigmoid_slope=10.0, path_flags=fl)
        gate.set_window(torch.hann_window(1024).numpy())
        xi, y = to_dev(x), to_dev(np.zeros((B, Lo), np.float32))
        gate.torch_set_noise(None, 0, 0, 0, True, None)
        gate.run_device(_ptr(xi), _ptr(y), np.float32, B, L, L, Lo, None)
        g = np.sin(np.arange(B * L, dtype=np.float32).reshape(B, L) * np.float32(0.01))
        gi, gy = to_dev(g), to_dev(np.zeros((B, Lo), np.float32))
        gate.torch_apply_masks_device(_ptr(gi), _ptr(gy), np.float32, B, L, L, Lo, None)
        outs.append((from_dev(y), from_dev(gy)))
        gate.close()
    (ya, ga), (yb, gb) = outs
    assert np.abs(ya).max() > 0 and np.array_equal(ya, yb)
    assert np.abs(ga).max() > 0 and np.array_equal(ga, gb)


def _ptr(a):
    return a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr()


def _cases():
    """(name, y, cfg, tap units, y_noise) -- small enough for the simulator."""
    y2 = synth_small(C=2, n=12000)
    y48 = synth_small(C=3, n=13000)
    n = 6000
    t = np.arange(n) / 16000
    rng = np.random.default_rng(5)
    tone = (1e-5 * rng.standard_normal(n) + 0.9 * np.sin(2 * np.pi * 1000 * t)).astype(np.float32)[None, :]
    quiet = (1e-5 * rng.standard_normal(4000)).astype(np.float32)[None, :]
    return [
        # 48 kHz: nf = 5, nt = 9 (config 2's 11 x 19 filter); first / interior / last chunk
        ("48k_chunks", y48, O.GateConfig(sr=48000, stationary=True, chunk_size=4000, padding=2000), [(0, 0), (1, 2), (3, 1)], None),
        # 48 kHz, T = 17 frames per chunk: fewer than 2 nt + 2 and odd
        ("48k_short_odd_T", y48[:, :9000], O.GateConfig(sr=48000, stationary=True, chunk_size=3000, padding=600),
         [(0, 0), (1, 1), (2, 2)], None),
        # 16 kHz defaults: 33 frequency taps, nt = 3; blend
        ("16k_blend", y2, O.GateConfig(sr=16000, stationary=True, chunk_size=5000, padding=600, prop_decrease=0.8),
         [(1, 1), (2, 0)], None),
        # other tap-word counts: nf = 9 (7 words), nf = 17 (10 words), nt = 13 (the byte-lane limit); no smoothing
        ("nf9", y2, O.GateConfig(sr=16000, stationary=True, chunk_size=5000, padding=600, freq_mask_smooth_hz=300), [(1, 0)], None),
        ("nf17_nt13", y2, O.GateConfig(sr=16000, stationary=True, chunk_size=5000, padding=600, freq_mask_smooth_hz=540,
                                       time_mask_smooth_ms=210, prop_decrease=0.9), [(1, 1)], None),
        ("no_smoothing", y2[:1], O.GateConfig(sr=16000, stationary=True, chunk_size=2500, padding=100, freq_mask_smooth_hz=None,
                                              time_mask_smooth_ms=None), [(1, 0)], None),
        # int16 samples in and out
        ("int16", (y2 * 20000).astype(np.int16), O.GateConfig(sr=16000, stationary=True, chunk_size=2500, padding=400), [(1, 1)], None),
        # top_db row floor: the tone's row is lifted (row flags set)
        ("rowfloor", tone, O.GateConfig(sr=16000, stationary=True, chunk_size=None, padding=300), [(0, 0)], quiet),
    ]


CASES = _cases()


@pytest.fixture(scope="module")
def simlib():
    return cusim_library()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_smoothing_in_synthesis_equals_separate_kernel_on_simulator(simlib, case):
    name, y, cfg, units, y_noise = case
    st = _assert_same(simlib, y, cfg, units, y_noise)
    if name == "rowfloor":
        assert st["rowfloor_flags"] > 0


def test_torchgate_forward_and_backward_on_simulator(simlib):
    x = synth_torchgate(B=2, n=24 * 256)
    _torchgate_same(simlib, x, lambda a: np.ascontiguousarray(a, np.float32), lambda a: a)


@pytest.mark.gpu
def test_smoothing_in_synthesis_equals_separate_kernel_on_gpu():
    lib = _cabi.library()
    for name, y, cfg, units, y_noise in CASES:
        st = _assert_same(lib, y, cfg, units, y_noise)
        if name == "rowfloor":
            assert st["rowfloor_flags"] > 0
    # config 2's geometry at full chunk size: 48 kHz, default chunk_size / padding (T = 2579), 3 channels x 1.3 M samples
    rng = np.random.default_rng(1000)
    n = 1_300_000
    t = np.arange(n) / 48000
    y = 0.05 * rng.standard_normal((3, n))
    for c in range(3):
        y[c] += 0.25 * ((t % 2.0) < 0.5) * np.sin(2 * np.pi * 440 * 2 ** (c / 12) * t)
    _assert_same(lib, y.astype(np.float32), O.GateConfig(sr=48000, stationary=True), [(0, 0), (1, 2), (2, 1)])


@pytest.mark.gpu
def test_torchgate_forward_and_backward_on_gpu():
    import torch
    lib = _cabi.library()
    x = synth_torchgate(B=8, n=160000)
    _torchgate_same(lib, x, lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda(),
                    lambda a: (torch.cuda.synchronize(), a.cpu().numpy())[1])
