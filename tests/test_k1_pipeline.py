"""Stationary analysis: the default k1_analyze (sample windows prefetched by bulk copy, top_db row maxima left to a
guarded fallback kernel that runs only when a frame could reach the floor) against the row-maximum kernel doing the
whole analysis with direct loads (path_flags bit 9).

Both run the same FP32 arithmetic, guard band and FP64 re-decision, so outputs, tapped spectra and masks and the
exactness counters must be EQUAL.  The simulator cases run the .cu sources on the CPU; the gpu-marked ones the nvcc
build."""
import numpy as np
import pytest

from noisereduce_b200 import _cabi
from oracle import spectral_gate_oracle as O
from tests import parity_cases as P
from tests.cusim_util import cusim_library
from tests.synth_host import synth_small

ROWMAX_K1 = 512         # path_flags bit 9: the row-maximum analysis kernel alone
COUNTERS = ("bins_rechecked_fp64", "bins_unresolved", "rowfloor_flags", "rowfloor_ambiguous")


def _run(lib, y, cfg, tap_unit, path_flags, y_noise=None, **extra):
    gate = _cabi.Gate(lib=lib, **P.gate_params(cfg, path_flags=path_flags, **extra))
    gate.noise_stats_host(y if y_noise is None else y_noise)
    gate.debug_select_unit(*tap_unit)
    out = gate.run_host(y)
    d = gate.debug_read()
    stats = gate.stats()
    gate.close()
    return out, d, stats


def _assert_same(lib, y, cfg, units, y_noise=None, **extra):
    for unit in units:
        out_a, d_a, st_a = _run(lib, y, cfg, unit, 0, y_noise, **extra)
        out_b, d_b, st_b = _run(lib, y, cfg, unit, ROWMAX_K1, y_noise, **extra)
        assert out_a.dtype == y.dtype and np.array_equal(out_a, out_b), unit
        assert np.abs(d_a["X"]).max() > 0 and np.array_equal(d_a["X"], d_b["X"]), unit
        assert np.array_equal(d_a["mask0"], d_b["mask0"]), unit
        assert d_a["mask"].any() and np.array_equal(d_a["mask"], d_b["mask"]), unit
        assert {k: st_a[k] for k in COUNTERS} == {k: st_b[k] for k in COUNTERS}, unit
    return st_a


def _cases():
    """(name, y, cfg, tap units, y_noise, extra gate params) -- small enough for the simulator."""
    y2 = synth_small(C=2, n=12000)
    y48 = synth_small(C=3, n=13000)
    n = 6000
    t = np.arange(n) / 16000
    rng = np.random.default_rng(5)
    tone = (1e-5 * rng.standard_normal(n) + 0.9 * np.sin(2 * np.pi * 1000 * t)).astype(np.float32)[None, :]
    quiet = (1e-5 * rng.standard_normal(4000)).astype(np.float32)[None, :]
    cfg600 = O.GateConfig(sr=16000, stationary=True, chunk_size=5000, padding=600)
    return [
        # 48 kHz (config 2's filter); first / interior / last chunk
        ("48k_chunks", y48, O.GateConfig(sr=48000, stationary=True, chunk_size=4000, padding=2000), [(0, 0), (1, 2), (3, 1)],
         None, {}),
        # T = 17 frames per chunk: short and odd
        ("48k_short_odd_T", y48[:, :9000], O.GateConfig(sr=48000, stationary=True, chunk_size=3000, padding=600),
         [(0, 0), (1, 1), (2, 2)], None, {}),
        # padding 600: 16-byte-aligned windows; 601: every window starts off a 16-byte boundary
        ("pad600", y2, cfg600, [(0, 0), (1, 1), (2, 0)], None, {}),
        ("pad601", y2, O.GateConfig(sr=16000, stationary=True, chunk_size=5000, padding=601), [(0, 1), (1, 0), (2, 1)],
         None, {}),
        # many bins through the FP64 re-decision (counters must agree)
        ("wide_guard_band", y2[:1, :5000], O.GateConfig(sr=16000, stationary=True, chunk_size=None, padding=300), [(0, 0)],
         None, dict(debug_guard_scale=100000)),
        ("int16", np.round(y2 * 20000).astype(np.int16), O.GateConfig(sr=16000, stationary=True, chunk_size=5000, padding=601),
         [(0, 0), (1, 1), (2, 1)], None, {}),
        ("float64", y2.astype(np.float64), cfg600, [(0, 1), (1, 0)], None, {}),
        # top_db row floor reachable: the flag is raised and the row-maximum fallback runs
        ("rowfloor", tone, O.GateConfig(sr=16000, stationary=True, chunk_size=None, padding=300), [(0, 0)], quiet, {}),
    ]


CASES = _cases()


@pytest.fixture(scope="module")
def simlib():
    return cusim_library()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_k1_default_equals_rowmax_kernel_on_simulator(simlib, case):
    name, y, cfg, units, y_noise, extra = case
    st = _assert_same(simlib, y, cfg, units, y_noise, **extra)
    if name == "rowfloor":
        assert st["rowfloor_flags"] > 0
    if name == "wide_guard_band":
        assert st["bins_rechecked_fp64"] > 100


@pytest.mark.gpu
def test_k1_default_equals_rowmax_kernel_on_gpu():
    lib = _cabi.library()
    for name, y, cfg, units, y_noise, extra in CASES:
        st = _assert_same(lib, y, cfg, units, y_noise, **extra)
        if name == "rowfloor":
            assert st["rowfloor_flags"] > 0
    # config 2's geometry at full chunk size: 48 kHz, default chunk_size / padding (T = 2579), 3 channels x 1.3 M samples
    rng = np.random.default_rng(1000)
    n = 1_300_000
    t = np.arange(n) / 48000
    y = 0.05 * rng.standard_normal((3, n))
    for c in range(3):
        y[c] += 0.25 * ((t % 2.0) < 0.5) * np.sin(2 * np.pi * 440 * 2 ** (c / 12) * t)
    y = y.astype(np.float32)
    cfg = O.GateConfig(sr=48000, stationary=True)
    _assert_same(lib, y, cfg, [(0, 0), (1, 2), (2, 1)])
    _assert_same(lib, y[:, 1:], cfg, [(1, 1)])            # rows starting off a 16-byte boundary
