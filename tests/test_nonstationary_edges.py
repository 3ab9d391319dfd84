"""The non-stationary gates at their numeric edges, against float64 references.

  * the IIR noise-floor follower (numpy surface, k_iir_sigmoid) on columns with a large dynamic range: quiet-then-loud
    with log-spaced clicks, loud-then-quiet, exact zeros at the start, an int16 recording whose quiet part is +-1 LSB;
    at T ln(1/(1-b)) from config 3's 6.9 to past 20, on both sides of the switch between the regenerated and the stored
    forward sweep, and at b >= 0.5; the default path and the stored sweep (path_flags 64) each against the oracle;
  * the moving-mean follower (TorchGate, k_tgate_movmean) on runs of digital silence of n_movemean - 1 .. n_movemean + 3
    frames, where the reference's mask is NaN: the NaN pattern must be the reference's (a NaN mask row must not reach the
    frame that shares its complex FFT in k2c_synthesize), the finite samples within the TorchGate tolerances;
  * NaN spans of the numpy surface: a padded chunk made entirely of silence, a single NaN sample.

Every case runs on the CPU simulator build (tests/cusim) and, marked gpu, on the product library.  Expected values come
from oracle/ (float64) and, for NaN patterns and the reference's own outputs, from tests/golden/nonstat_edges*.npz
(tests/golden/make_golden_nonstat_edges.py, the unmodified reference)."""
import math

import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from noisereduce_b200.torchgate import TorchGate
from oracle import spectral_gate_oracle as O
from oracle import torchgate_oracle as TO
from tests import parity_cases as P
from tests.golden import make_golden_nonstat_edges as G

TG_TOL = {np.float32: 5e-6, np.float64: 5e-7}      # TorchGate forward vs the float64 oracle (tests/test_cusim_torchgate.py)
OUT_TOL_NONSTAT = P.OUT_TOL_TIGHT * 5               # non-stationary waveform (tests/test_cusim_parity.py)


@pytest.fixture(scope="module", params=["sim", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    if request.param == "gpu":
        return _cabi.library()
    from tests.cusim import build_cusim
    lib = _cabi.GateLibrary(build_cusim.build())
    lib.simulated_device = True                     # CPU tensors take the device route of reduce_noise(use_torch=True)
    return lib


def _on_gpu(lib):
    return not getattr(lib, "simulated_device", False)


# ---- the IIR follower -------------------------------------------------------------------------------------------
def regen_selected(b, T):
    """gate_host.cu iir_regen_ok: the forward sweep is rebuilt by the inverse recurrence only where the bound
    2.5 u (1-b)^(-2T) / b on the relative error of S stays within 2^-24."""
    return b < 0.5 and 2.0 * T * -math.log1p(-b) - math.log(b) <= 29.0 * math.log(2.0) - math.log(2.5)


def _switch_T(b):
    """The largest T that still regenerates."""
    return int(math.floor((29.0 * math.log(2.0) - math.log(2.5) + math.log(b)) / (2.0 * -math.log1p(-b))))


PAD = 1000


def _geometry(sr, n_fft, tc, where):
    """(cfg, n, T, b): a single padded chunk of T frames, T from `where` = a value of T ln(1/(1-b)), or
    'switch' / 'switch+1' (the last regenerating T and the first storing one)."""
    H = n_fft // 4
    b = O.iir_coefficient(tc, sr, H)
    if where == "switch":
        T = _switch_T(b)
    elif where == "switch+1":
        T = _switch_T(b) + 1
    else:
        T = int(round(where / -math.log1p(-b)))
    n = (T - 1) * H - 2 * PAD
    cfg = O.GateConfig(sr=sr, stationary=False, n_fft=n_fft, chunk_size=None, padding=PAD, time_constant_s=tc)
    return cfg, n, T, b


def _column(kind, n, sr):
    rng = np.random.default_rng(17)
    if kind == "quiet_then_loud":
        return G.quiet_then_loud(n, int(0.6 * n), n_clicks=min(60, (int(0.6 * n) - 1000) // 1100))
    if kind == "loud_then_quiet":
        return G.quiet_then_loud(n, int(0.6 * n), n_clicks=min(60, (int(0.6 * n) - 1000) // 1100))[::-1].copy()
    t = np.arange(n) / sr
    y = 0.05 * rng.standard_normal(n) + 0.3 * np.sin(2 * np.pi * 440 * t) * ((t % 1.0) < 0.4)
    if kind == "zeros_at_start":
        y[: n // 3] = 0.0
        return y.astype(np.float32)
    assert kind == "int16_lsb"                      # loud half, then a quiet half of -1 / 0 / +1 LSB
    q = np.round(y * 8000.0)
    q[n // 2:] = rng.integers(-1, 2, n - n // 2)
    return q.astype(np.int16)


def _check_iir(lib, y, cfg, path_flags):
    y2d = y[None, :]
    taps = {(0, 0): O.Taps()}
    ref = O.reduce_noise(y2d, cfg.sr, cfg=cfg, unit_taps=taps, return_float64=True)
    gate = _cabi.Gate(lib=lib, **P.gate_params(cfg, path_flags=path_flags))
    gate.debug_select_unit(0, 0)
    out = gate.run_host(y2d)
    d = gate.debug_read()
    gate.close()
    tp = taps[(0, 0)]
    assert out.dtype == y2d.dtype
    touched = d["mask"].any(axis=0)                 # the frames the synthesis needed (tests/parity_cases.py)
    mask_err = float(np.abs(d["mask"] - tp.mask)[:, touched].max())
    if np.issubdtype(y2d.dtype, np.integer):
        lsb = int(np.abs(out.astype(np.int64) - O.cast_like_reference(ref, y2d.dtype).astype(np.int64)).max())
        return mask_err, lsb, out
    return mask_err, P.relinf(out, ref), out


# (sr, n_fft, time_constant_s, T ln(1/(1-b)) or the switch point): both row pitches (544 and 1056)
IIR_GEOMETRIES = [
    (16000, 1024, 2.0, 7.0), (16000, 1024, 2.0, 14.0), (16000, 1024, 2.0, 19.9), (16000, 1024, 2.0, 20.5),
    (16000, 1024, 2.0, "switch"), (16000, 1024, 2.0, "switch+1"), (16000, 1024, 0.012, 400.0),
    (48000, 2048, 2.0, 6.88), (48000, 2048, 0.5, 14.0), (48000, 2048, 0.5, 19.9), (48000, 2048, 0.5, 20.5),
    (48000, 2048, 0.5, "switch"), (48000, 2048, 0.5, "switch+1"), (48000, 2048, 0.008, 400.0),
]                                                   # (time constants 0.012 / 0.008 s: b = 0.66 / 0.71)


@pytest.mark.parametrize("geo", IIR_GEOMETRIES, ids=lambda g: f"{g[0] // 1000}k-nfft{g[1]}-tc{g[2]}-TL{g[3]}")
def test_iir_follower_quiet_then_loud(lib, geo):
    """The 35 s single chunk at 16 kHz (TL = 19.4) put mask errors of 3e-3 on such columns when the forward sweep
    was rebuilt by the inverse recurrence up to TL < 20."""
    sr, n_fft, tc, where = geo
    cfg, n, T, b = _geometry(sr, n_fft, tc, where)
    if where == "switch":
        assert regen_selected(b, T) and not regen_selected(b, T + 1)
    if sr == 48000 and tc == 2.0:
        assert T == 1290 and regen_selected(b, T)   # config 3 keeps the regenerated sweep
    if tc < 0.1:
        assert b >= 0.5
    y = _column("quiet_then_loud", n, sr)
    for fl in (0, 64):
        mask_err, out_err, _ = _check_iir(lib, y, cfg, fl)
        assert mask_err < P.MASK_TOL_NONSTAT and out_err < OUT_TOL_NONSTAT, (geo, T, b, fl, mask_err, out_err)


@pytest.mark.parametrize("kind", ["loud_then_quiet", "zeros_at_start", "int16_lsb"])
@pytest.mark.parametrize("geo", [g for g in IIR_GEOMETRIES if g[3] in (14.0, "switch", "switch+1")],
                         ids=lambda g: f"{g[0] // 1000}k-nfft{g[1]}-TL{g[3]}")
def test_iir_follower_other_columns(lib, geo, kind):
    sr, n_fft, tc, where = geo
    cfg, n, T, b = _geometry(sr, n_fft, tc, where)
    y = _column(kind, n, sr)
    for fl in (0, 64):
        mask_err, out_err, _ = _check_iir(lib, y, cfg, fl)
        tol = 1 if kind == "int16_lsb" else OUT_TOL_NONSTAT
        assert mask_err < P.MASK_TOL_NONSTAT and out_err <= tol, (geo, kind, T, fl, mask_err, out_err)


def test_iir_follower_35s_at_16k(lib):
    """The geometry the defect was found on: one 560000-sample recording at 16 kHz, default settings (T = 2422,
    T ln(1/(1-b)) = 19.4), zeros up to 60 % with clicks of 1e-6 .. 1e-2, then noise."""
    y = G.quiet_then_loud(560000, 336000)
    cfg = O.GateConfig(sr=16000, stationary=False)
    for fl in (0, 64):
        mask_err, out_err, _ = _check_iir(lib, y, cfg, fl)
        assert mask_err < P.MASK_TOL_NONSTAT and out_err < OUT_TOL_NONSTAT, (fl, mask_err, out_err)


def test_iir_follower_config3_quiet_first_half(lib):
    """Config 3's geometry (48 kHz, n_fft 2048, default chunking): two chunks of a recording whose first half is exact
    zeros with clicks; the first chunk's (regenerated) follower and the output against the oracle."""
    n = 1_000_000 if _on_gpu(lib) else 700_000
    y = G.quiet_then_loud(n, n // 2)
    cfg = O.GateConfig(sr=48000, stationary=False, n_fft=2048)
    taps = {(0, 0): O.Taps()}
    ref = O.reduce_noise(y[None], 48000, cfg=cfg, unit_taps=taps, return_float64=True)
    for fl in (0, 64):
        gate = _cabi.Gate(lib=lib, **P.gate_params(cfg, path_flags=fl))
        gate.debug_select_unit(0, 0)
        out = gate.run_host(y[None])
        d = gate.debug_read()
        gate.close()
        touched = d["mask"].any(axis=0)
        assert float(np.abs(d["mask"] - taps[(0, 0)].mask)[:, touched].max()) < P.MASK_TOL_NONSTAT
        assert P.relinf(out, ref) < OUT_TOL_NONSTAT


def test_iir_quiet_then_loud_against_the_reference(lib, golden_dir):
    """Two of the quiet-then-loud inputs, against the unmodified reference's own outputs (and the oracle against them)."""
    g = P.load_golden(golden_dir, "nonstat_edges")
    for name, (y, kw) in G.iir_inputs().items():
        cfg = O.GateConfig(sr=G.SR, **kw)
        gate = _cabi.Gate(lib=lib, **P.gate_params(cfg))
        out = gate.run_host(y[None])[0]
        gate.close()
        want = g[f"iir_{name}"]
        assert out.dtype == want.dtype and out.shape == want.shape
        assert P.relinf(O.reduce_noise(y, G.SR, cfg=cfg, return_float64=True), want) < P.OUT_TOL, name
        assert P.relinf(out, want) < P.OUT_TOL, name


# ---- the moving-mean follower and NaN regions (TorchGate) ---------------------------------------------------------
def _nan_pattern(g, key, shape):
    return np.unpackbits(g[key + "_nan"])[: int(np.prod(shape))].reshape(shape).astype(bool)


def _check_nan_and_finite(got, want_nan, ref, tol, what):
    got = np.asarray(got, dtype=np.float64)
    assert np.array_equal(np.isnan(got), want_nan), (what, np.flatnonzero(np.isnan(got) != want_nan)[:8])
    fin = ~want_nan
    assert np.abs(got[fin] - ref[fin]).max() <= tol * np.abs(ref[fin]).max(), what


@pytest.mark.parametrize("name", list(G.torchgate_inputs()))
def test_torchgate_nan_regions(lib, golden_dir, name):
    g = P.load_golden(golden_dir, "nonstat_edges")
    x = G.torchgate_inputs()[name]
    w = torch.hann_window(1024).numpy()
    dev = "cuda" if _on_gpu(lib) else "cpu"
    for sm, kw in G.TG_SMOOTHING.items():
        ref = TO.torchgate_forward(x, G.SR, nonstationary=True, window=w, **kw)
        want_nan = _nan_pattern(g, f"tg_{name}_{sm}_f32", ref.shape)
        assert np.array_equal(np.isnan(ref), want_nan), (name, sm)           # the oracle agrees with the reference
        assert np.array_equal(_nan_pattern(g, f"tg_{name}_{sm}_f64", ref.shape), want_nan)
        # rows 1.. have n_movemean or more silent frames: NaN there; row 0 (n_movemean - 1) has none
        assert not want_nan[0].any() and all(want_nan[i].any() for i in range(1, x.shape[0]))
        tg = TorchGate(sr=G.SR, nonstationary=True, **kw)
        for dt in (np.float32, np.float64):
            for xn in (None, x[0, :4096]):
                xt = torch.from_numpy(x.astype(dt)).to(dev)
                xnt = None if xn is None else torch.from_numpy(xn.astype(dt)).to(dev)
                y = tg(xt, xnt, _lib=None if dev == "cuda" else lib)
                assert y.dtype == xt.dtype and tuple(y.shape) == ref.shape
                _check_nan_and_finite(y.cpu().numpy(), want_nan, ref, TG_TOL[dt], (name, sm, dt.__name__, xn is None))


def test_torchgate_config4_batch_with_silences(lib):
    """A config-4-shaped batch (TorchGate(sr=16000), 10 s rows at 16 kHz; 255 rows on the GPU) with silences of
    19 .. 23 frames starting on even and odd frames, content around them 1e9 apart in amplitude."""
    B, L = (255, 160000) if _on_gpu(lib) else (15, 48000)
    rng = np.random.default_rng(23)
    x = 0.05 * rng.standard_normal((B, L))
    for i in range(B):
        k, t0 = G.SILENCE_FRAMES[i % 5], 40 + (i % 7) * 17 + (i // 5) % 2
        z0, z1 = t0 * G.HOP - 512, (t0 + k - 1) * G.HOP + 512
        if i % 3 == 1:
            x[i, :z0] *= 2e4
            x[i, z1:] *= 2e-5
        elif i % 3 == 2:
            x[i, :z0] *= 2e-5
            x[i, z1:] *= 2e4
        x[i, z0:z1] = 0.0
    x = x.astype(np.float32)
    ref = TO.torchgate_forward(x.astype(np.float64), G.SR, nonstationary=True, window=torch.hann_window(1024).numpy())
    want_nan = np.isnan(ref)
    assert want_nan[1].any() and not want_nan[0].any()
    dev = "cuda" if _on_gpu(lib) else "cpu"
    y = TorchGate(sr=G.SR, nonstationary=True)(torch.from_numpy(x).to(dev), _lib=None if dev == "cuda" else lib)
    _check_nan_and_finite(y.cpu().numpy(), want_nan, ref, TG_TOL[np.float32], "config4")


def _nr(lib, monkeypatch):
    if not _on_gpu(lib):
        monkeypatch.setattr(_cabi, "_LIB", lib)
    import noisereduce_b200 as nr
    return nr


def test_torch_route_nonstationary_silences(lib, golden_dir, monkeypatch):
    """reduce_noise(use_torch=True, stationary=False) on rows with silences, one padded chunk entirely silent."""
    nr = _nr(lib, monkeypatch)
    g = P.load_golden(golden_dir, "nonstat_edges")
    for name, (y, kw) in G.torch_route_inputs().items():
        want = g[f"route_{name}"]
        got = nr.reduce_noise(y=y, sr=G.SR, use_torch=True, **kw)
        assert got.dtype == want.dtype and got.shape == want.shape
        assert np.isnan(want).any()
        assert np.array_equal(np.isnan(got), np.isnan(want)), name
        fin = ~np.isnan(want)
        assert P.relinf(got[fin], want[fin]) < P.OUT_TOL, name


# ---- NaN spans of the numpy surface -------------------------------------------------------------------------------
STATIONARY_NAN_GAP = (
    "stationary gate, known difference: a NaN bin does not turn its row's top_db floor NaN (the reference's row max is "
    "NaN, so every decision of that row is False), and a NaN sample reaches the frame sharing its packed FFT")


@pytest.mark.parametrize("name", [n if "_stat" not in n or "silent" in n else
                                  pytest.param(n, marks=pytest.mark.xfail(strict=True, reason=STATIONARY_NAN_GAP))
                                  for n in G.numpy_nan_inputs()])
def test_numpy_surface_nan_spans(lib, golden_dir, monkeypatch, name):
    nr = _nr(lib, monkeypatch)
    g = P.load_golden(golden_dir, "nonstat_edges")
    y, y_noise, kw = G.numpy_nan_inputs()[name]
    want = g[f"np_{name}"]
    got = nr.reduce_noise(y=y, sr=G.SR, y_noise=y_noise, **kw)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want)), (name, int(np.isnan(got).sum()), int(np.isnan(want).sum()))
    ref = O.reduce_noise(y, G.SR, y_noise=y_noise, cfg=O.GateConfig(sr=G.SR, **kw), return_float64=True)
    assert np.array_equal(np.isnan(ref), np.isnan(want)), name
    fin = ~np.isnan(want)
    assert P.relinf(got[fin], ref[fin]) < P.OUT_TOL, name
