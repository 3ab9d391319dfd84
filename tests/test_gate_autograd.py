"""Backpropagation through reduce_noise() / SpectralGate*.get_traces() on device tensors (b200gate_adjoint).

The gradient convention is TorchGate's: every unit's final mask is a constant, and the gradient flows through
STFT -> mask -> iSTFT and the chunk assembly.  The reference here is a float64 restatement in torch of the oracle's own
read_chunk / stft / istft / chunk_table, with each unit's final mask taken from the oracle's unit taps, differentiated by
torch autograd.  On the CPU simulator (tests/cusim) CPU tensors take the device route, so every kernel of the forward
and the adjoint runs here; the GPU tests repeat the checks at config 2's scale on an H100."""
import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from oracle import spectral_gate_oracle as orc
from tests.synth_host import synth_small

SR = 16000


@pytest.fixture(scope="module")
def simlib():
    from tests.cusim import build_cusim
    lib = _cabi.GateLibrary(build_cusim.build())
    lib.simulated_device = True
    return lib


@pytest.fixture
def sim(simlib, monkeypatch):
    monkeypatch.setattr(_cabi, "_LIB", simlib)
    import noisereduce_b200 as nr
    return nr


# ---- the float64 restatement -------------------------------------------------------------------------------------
def _t_stft(x, N, W, H):
    w = torch.from_numpy(orc.hann_periodic(W))
    xe = torch.nn.functional.pad(x, (W // 2, W // 2))
    T = (xe.shape[0] - W) // H + 1
    idx = (torch.arange(T) * H)[:, None] + torch.arange(W)[None, :]
    return (torch.fft.rfft(w * xe[idx], n=N) / w.sum()).T                   # [F, T]


def _t_istft(X, N, W, H):
    T = X.shape[1]
    w = torch.from_numpy(orc.hann_periodic(W))
    seg = torch.fft.irfft(X.T, n=N)[:, :W] * w.sum()
    L = W + (T - 1) * H
    idx = ((torch.arange(T) * H)[:, None] + torch.arange(W)[None, :]).reshape(-1)
    out = torch.zeros(L, dtype=torch.float64).index_add(0, idx, (seg * w).reshape(-1))
    norm = np.zeros(L)
    for t in range(T):
        norm[t * H: t * H + W] += orc.hann_periodic(W) ** 2
    norm = torch.from_numpy(np.where(norm > 1e-10, norm, 1.0))
    return (out / norm)[W // 2: L - W // 2]


def restatement(y64, cfg, start_frame=None, end_frame=None, y_noise=None):
    """(A as a torch function of a float64 [C, n] tensor, its output on y64's values): the gate with the oracle's final
    masks of y64 held fixed."""
    y2d = y64.detach().numpy()
    C, n = y2d.shape
    tab = orc.chunk_table(n, cfg.chunk_size, cfg.padding, start_frame, end_frame)
    taps = {(i, c): orc.Taps() for i in range(len(tab)) for c in range(C)}
    orc.reduce_noise(y2d, cfg.sr, y_noise=y_noise, cfg=cfg, return_float64=True, unit_taps=taps,
                     start_frame=start_frame, end_frame=end_frame)
    N, W, H = cfg.resolve()
    s0, s1 = orc.traces_span(n, cfg.chunk_size, start_frame, end_frame)

    def A(y):
        out = [torch.zeros(n, dtype=torch.float64) for _ in range(C)]
        for ich, (i1, i2, lo, hi) in enumerate(tab):
            for c in range(C):
                x = torch.nn.functional.pad(y[c, max(i1, 0): min(i2, n)], (max(0, -i1), max(0, i2 - n)))
                m = torch.from_numpy(taps[(ich, c)].mask)
                sig = _t_istft(_t_stft(x, N, W, H) * m, N, W, H)
                yu = torch.cat([sig, torch.zeros(x.shape[0] - sig.shape[0], dtype=torch.float64)])[: x.shape[0]]
                out[c] = torch.cat([out[c][:lo], yu[lo - i1: hi - i1], out[c][hi:]])
        return torch.stack(out)[:, s0:s1]

    return A


def _cfg(**kw):
    base = dict(sr=SR, stationary=True, chunk_size=6000, padding=1500, freq_mask_smooth_hz=500, time_mask_smooth_ms=50)
    base.update(kw)
    return orc.GateConfig(**base)


def _kwargs(cfg):
    return dict(sr=SR, stationary=cfg.stationary, chunk_size=cfg.chunk_size, padding=cfg.padding, n_fft=cfg.n_fft,
                win_length=cfg.win_length, hop_length=cfg.hop_length, prop_decrease=cfg.prop_decrease,
                freq_mask_smooth_hz=cfg.freq_mask_smooth_hz, time_mask_smooth_ms=cfg.time_mask_smooth_ms)


def _grad_case(nr, y_np, cfg, dtype=torch.float32, flat=False, seed=0, y_noise=None):
    """(library gradient, restatement gradient, forward with and without requires_grad) for a random upstream g."""
    y = torch.from_numpy(y_np).to(dtype)
    if flat:
        y = y[0]
    yg = y.clone().requires_grad_(True)
    out = nr.reduce_noise(yg, y_noise=y_noise, **_kwargs(cfg))
    with torch.no_grad():
        plain = nr.reduce_noise(y.clone(), y_noise=y_noise, **_kwargs(cfg))
    g = torch.from_numpy(np.random.default_rng(seed).standard_normal(tuple(out.shape))).to(out.dtype)
    (gl,) = torch.autograd.grad(out, yg, g)
    y64 = y.to(torch.float64).reshape(-1, y.shape[-1]).detach().requires_grad_(True)
    A = restatement(y64, cfg, y_noise=y_noise)
    (gr,) = torch.autograd.grad(A(y64), y64, g.to(torch.float64).reshape(y64.shape[0], -1))
    return gl, gr.reshape(gl.shape), out, plain


def _close(gl, gr, rtol):
    err = (gl.to(torch.float64) - gr).abs().max().item()
    assert err <= rtol * gr.abs().max().item(), (err, gr.abs().max().item())


CASES = {
    # name: (gate options, signal length, channels)
    "stationary": (dict(), 20000, 2),
    "nonstationary": (dict(stationary=False), 20000, 2),
    "pad0": (dict(padding=0), 15000, 1),
    "pad_below_hop": (dict(padding=100), 15000, 1),
    "pad_ge_chunk": (dict(chunk_size=4000, padding=5000), 15000, 1),
    "single_chunk": (dict(chunk_size=30000), 12000, 2),
    "prop_0.6": (dict(prop_decrease=0.6), 15000, 1),
    "no_smoothing": (dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None), 15000, 1),
    "nonstationary_prop_0.6": (dict(stationary=False, prop_decrease=0.6), 15000, 1),
    # the n_fft 2048 non-stationary kernels (config 3's geometry), ragged last chunk
    "nonstationary_2048": (dict(stationary=False, n_fft=2048, chunk_size=8000, padding=2000), 21000, 2),
    "nonstationary_2048_pad_below_hop": (dict(stationary=False, n_fft=2048, chunk_size=8000, padding=300), 17000, 1),
}
GENERIC = {
    "512_400_100": (dict(n_fft=512, win_length=400, hop_length=100, chunk_size=5000, padding=700), 12000, 2),
    "bluestein_441": (dict(n_fft=441, chunk_size=5000, padding=700), 12000, 1),
    "generic_nonstationary": (dict(stationary=False, n_fft=512, chunk_size=5000, padding=700), 12000, 1),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_gradient_tuned_family(sim, name):
    kw, n, C = CASES[name]
    cfg = _cfg(**kw)
    gl, gr, out, plain = _grad_case(sim, synth_small(C=C, n=n), cfg)
    assert torch.equal(out.detach(), plain)                       # the forward is unchanged by requires_grad
    _close(gl, gr, 2e-5)


@pytest.mark.parametrize("name", sorted(GENERIC))
def test_gradient_general_family(sim, name):
    kw, n, C = GENERIC[name]
    cfg = _cfg(**kw)
    gl, gr, out, plain = _grad_case(sim, synth_small(C=C, n=n), cfg, dtype=torch.float64)
    assert torch.equal(out.detach(), plain)
    _close(gl, gr, 1e-9)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16])
def test_gradient_dtypes(sim, dtype):
    cfg = _cfg()
    gl, gr, out, plain = _grad_case(sim, synth_small(C=1, n=14000), cfg, dtype=dtype)
    assert gl.dtype == dtype and out.dtype == dtype
    assert torch.equal(out.detach(), plain)
    if dtype == torch.float16:
        _close(gl, gr.to(torch.float16).to(torch.float64), 2e-3)  # the gradient is cast to float16 as Tensor.to does
    else:
        _close(gl, gr, 2e-5)


@pytest.mark.parametrize("stationary", [True, False])
def test_gradient_with_noise_clip(sim, stationary):
    """y_noise given: the stationary thresholds come from the clip (the clip-threshold path of the kept decisions)."""
    y_noise = synth_small(C=1, n=9000, seed=3)[0]
    gl, gr, out, plain = _grad_case(sim, synth_small(C=2, n=15000), _cfg(stationary=stationary), y_noise=y_noise)
    assert torch.equal(out.detach(), plain)
    _close(gl, gr, 2e-5)


def test_gradient_2048_float64(sim):
    """float64 samples on the n_fft 2048 kernels, which read float32 rows: the gradient is converted at the edge."""
    cfg = _cfg(stationary=False, n_fft=2048, chunk_size=8000, padding=2000)
    gl, gr, out, plain = _grad_case(sim, synth_small(C=1, n=17000), cfg, dtype=torch.float64)
    assert gl.dtype == torch.float64 and torch.equal(out.detach(), plain)
    _close(gl, gr, 2e-5)


def test_gradient_flat_input(sim):
    gl, gr, out, plain = _grad_case(sim, synth_small(C=1, n=15000), _cfg(), flat=True)
    assert gl.shape == (15000,) and out.shape == (15000,)
    _close(gl, gr, 2e-5)


@pytest.mark.parametrize("rng", [(3000, 14000), (None, 5000)])
def test_gradient_sub_ranges(sim, rng):
    """get_traces(start, end): mode 1 (chunks of the grid) and mode 2 (one padded chunk reading its padding from the
    recording past end_frame)."""
    cfg = _cfg()
    y_np = synth_small(C=2, n=20000)
    yg = torch.from_numpy(y_np).float().requires_grad_(True)
    from noisereduce_b200.spectralgate.stationary import SpectralGateStationary
    sg = SpectralGateStationary(y=yg, sr=SR, y_noise=None, prop_decrease=1.0, n_std_thresh_stationary=1.5,
                                chunk_size=cfg.chunk_size, clip_noise_stationary=True, padding=cfg.padding, n_fft=1024,
                                win_length=None, hop_length=None, time_constant_s=2.0, freq_mask_smooth_hz=500,
                                time_mask_smooth_ms=50, tmp_folder=None, use_tqdm=False, n_jobs=1)
    out = sg.get_traces(*rng)
    g = torch.from_numpy(np.random.default_rng(1).standard_normal(tuple(out.shape))).float()
    (gl,) = torch.autograd.grad(out, yg, g)
    y64 = yg.detach().double().requires_grad_(True)
    (gr,) = torch.autograd.grad(restatement(y64, cfg, *rng)(y64), y64, g.double())
    _close(gl, gr, 2e-5)


def test_y_noise_gets_no_gradient(sim):
    cfg = _cfg()
    y = torch.from_numpy(synth_small(C=1, n=15000)).float().requires_grad_(True)
    yn = torch.from_numpy(synth_small(C=1, n=8000, seed=3)).float().requires_grad_(True)
    out = sim.reduce_noise(y, y_noise=yn, **_kwargs(cfg))
    out.sum().backward()
    assert y.grad is not None and yn.grad is None


def test_adjoint_identity(sim):
    """<A v, g> = <v, A^T g> with A the restatement's map and A^T the library's."""
    cfg = _cfg(stationary=False)
    y_np = synth_small(C=1, n=15000)
    yg = torch.from_numpy(y_np).double().requires_grad_(True)
    out = sim.reduce_noise(yg, **_kwargs(cfg))
    rng = np.random.default_rng(5)
    g = torch.from_numpy(rng.standard_normal(tuple(out.shape)))
    (atg,) = torch.autograd.grad(out, yg, g)
    A = restatement(yg.detach(), cfg)
    v = torch.from_numpy(rng.standard_normal(tuple(yg.shape)))
    lhs = (A(v) * g).sum().item()
    rhs = (v * atg).sum().item()
    assert abs(lhs - rhs) <= 1e-5 * abs(lhs)


def test_finite_differences_stationary(sim, monkeypatch):
    """Stationary gate, float64: central differences of <f(y), g> along v agree with <grad, v>.

    The thresholds come from a fixed noise clip.  The tuned kernels' exactness counters show that no decision of this
    input lies inside the FP32 guard band (|margin| <= kappa eps32 ||frame||, about 1e-6 of the frame's norm), so a step
    of 1e-8 of the signal's norm moves none of them.  The differences are taken in float64 arithmetic (path_flags bit 2:
    the general family on the same geometry, whose decisions are the same float64 decisions)."""
    from noisereduce_b200.spectralgate import base
    from noisereduce_b200.spectralgate.stationary import SpectralGateStationary
    cfg = _cfg()
    y_noise = synth_small(C=1, n=9000, seed=3)[0]
    y = torch.from_numpy(synth_small(C=1, n=15000)).double()
    sg = SpectralGateStationary(y=y.clone(), sr=SR, y_noise=y_noise, prop_decrease=1.0, n_std_thresh_stationary=1.5,
                                chunk_size=cfg.chunk_size, clip_noise_stationary=True, padding=cfg.padding, n_fft=1024,
                                win_length=None, hop_length=None, time_constant_s=2.0, freq_mask_smooth_hz=500,
                                time_mask_smooth_ms=50, tmp_folder=None, use_tqdm=False, n_jobs=1)
    sg.get_traces()
    st = sg._gate.stats()
    assert st["units"] > 0 and st["bins_rechecked_fp64"] == 0 and st["bins_unresolved"] == 0
    assert st["rowfloor_ambiguous"] == 0

    orig = base.SpectralGate._gate_params

    def params(self):
        d = orig(self)
        d["path_flags"] = 4
        return d
    monkeypatch.setattr(base.SpectralGate, "_gate_params", params)
    kw = dict(_kwargs(cfg), y_noise=y_noise)
    yg = y.clone().requires_grad_(True)
    out = sim.reduce_noise(yg, **kw)
    rng = np.random.default_rng(7)
    g = torch.from_numpy(rng.standard_normal(tuple(out.shape)))
    v = torch.from_numpy(rng.standard_normal(tuple(y.shape)))
    v *= y.norm() / v.norm()
    (grad,) = torch.autograd.grad(out, yg, g)
    eps = 1e-8
    with torch.no_grad():
        fp = (sim.reduce_noise(y + eps * v, **kw) * g).sum().item()
        fm = (sim.reduce_noise(y - eps * v, **kw) * g).sum().item()
    fd, an = (fp - fm) / (2 * eps), (grad * v).sum().item()
    assert abs(fd - an) <= 1e-5 * abs(an), (fd, an)


def test_batching_and_reruns_bit_equal(sim, monkeypatch):
    """One workspace batch against several, and two backward passes: the same gradient in every bit."""
    from noisereduce_b200.spectralgate import base
    cfg = _cfg(chunk_size=4000, padding=5000)                    # several overlapping units per sample
    y = torch.from_numpy(synth_small(C=3, n=20000)).float()
    g = torch.from_numpy(np.random.default_rng(2).standard_normal((3, 20000))).float()

    def grad_with(limit):
        orig = base.SpectralGate._gate_params

        def params(self):
            d = orig(self)
            d["workspace_limit_bytes"] = float(limit)
            return d
        monkeypatch.setattr(base.SpectralGate, "_gate_params", params)
        yg = y.clone().requires_grad_(True)
        out = sim.reduce_noise(yg, **_kwargs(cfg))
        return torch.autograd.grad(out, yg, g)[0]

    big, small = grad_with(1 << 34), grad_with(1 << 20)
    again = grad_with(1 << 20)
    assert torch.equal(big, small) and torch.equal(small, again)


def test_routes_without_grad_carry_no_graph(sim):
    cfg = _cfg()
    y = torch.from_numpy(synth_small(C=1, n=15000)).float().requires_grad_(True)
    with torch.no_grad():
        assert sim.reduce_noise(y, **_kwargs(cfg)).grad_fn is None
    assert sim.reduce_noise(y.detach(), **_kwargs(cfg)).grad_fn is None
    assert sim.reduce_noise(y, use_torch=True, **_kwargs(cfg)).grad_fn is None
    st = sim.NoiseReduceStream(SR, 1, **{k: v for k, v in _kwargs(cfg).items() if k != "sr"})
    parts = [st.push(y[:, :8000]), st.push(y[:, 8000:]), st.finish()]
    assert all(getattr(p, "grad_fn", None) is None for p in parts)


def test_double_backward_raises(sim):
    y = torch.from_numpy(synth_small(C=1, n=15000)).float().requires_grad_(True)
    out = sim.reduce_noise(y, **_kwargs(_cfg()))
    (gr,) = torch.autograd.grad(out.sum(), y, create_graph=True)
    with pytest.raises(RuntimeError):
        gr.sum().backward()


# ---- the C ABI's refusals ---------------------------------------------------------------------------------------
def test_cabi_refusals(simlib):
    import ctypes
    d = simlib.dll
    y = np.ascontiguousarray(synth_small(C=1, n=15000).astype(np.float32))
    out = np.empty_like(y)
    g = _cabi.Gate(simlib, surface=_cabi.SURFACE_NUMPY, stationary=0, n_fft=1024, win_length=1024, hop_length=256,
                   chunk_size=6000, padding=1500, sr=SR, prop_decrease=1.0, top_db=80.0, time_constant_s=2.0,
                   thresh_n_mult=2.0, sigmoid_slope=10.0)
    need = g.mask_store_bytes(1, 15000)
    short = np.zeros(need - 4, np.uint8)
    g.set_mask_store(short.ctypes.data, short.nbytes)
    with pytest.raises(_cabi.GateError):                          # a store too short for the run
        g.run_device(y.ctypes.data, out.ctypes.data, np.float32, 1, 15000, 15000, 15000)
    store = np.zeros(need, np.uint8)
    g.set_mask_store(store.ctypes.data, store.nbytes)
    g.run_device(y.ctypes.data, out.ctypes.data, np.float32, 1, 15000, 15000, 15000)
    g.set_mask_store(None)
    grad = np.empty_like(y)
    g.adjoint_device(store.ctypes.data, y.ctypes.data, grad.ctypes.data, np.float32, 1, 15000, 15000, 15000)
    with pytest.raises(_cabi.GateError):                          # a store from another geometry
        g.adjoint_device(store.ctypes.data, y.ctypes.data, grad.ctypes.data, np.float32, 1, 14000, 15000, 15000)
    with pytest.raises(_cabi.GateError):                          # a store no run filled
        g.adjoint_device(short.ctypes.data, y.ctypes.data, grad.ctypes.data, np.float32, 1, 15000, 15000, 15000)
    t = _cabi.Gate(simlib, surface=_cabi.SURFACE_TORCH, stationary=0, n_fft=1024, win_length=1024, hop_length=256,
                   sr=SR, prop_decrease=1.0, top_db=40.0, n_movemean=20, thresh_n_mult=1.0, sigmoid_slope=10.0,
                   std_ddof=1)
    assert d.b200gate_set_mask_store(t._h, ctypes.c_void_p(store.ctypes.data), need) == _cabi.ERR_STATE
    assert d.b200gate_adjoint(t._h, ctypes.c_void_p(store.ctypes.data), ctypes.c_void_p(y.ctypes.data),
                              ctypes.c_void_p(grad.ctypes.data), _cabi.F32, 1, 15000, 15000, 15000, 1, None) == \
        _cabi.ERR_STATE


# ---- on one H100 --------------------------------------------------------------------------------------------------
def _gpu_case(C, seconds, sr, cfg, dtype=torch.float32, offset=0, check=(0,)):
    import noisereduce_b200 as nr
    rng = np.random.default_rng(11)
    n = int(seconds * sr)
    base = synth_small(C=C, n=n + offset, sr=sr)
    y_noise = synth_small(C=1, n=sr, sr=sr, seed=4)[0]
    y = torch.from_numpy(base).to(dtype).cuda()[:, offset:]
    yg = y.detach().requires_grad_(True)                          # (keeps the view's storage offset)
    kw = dict(_kwargs(cfg), sr=sr)
    out = nr.reduce_noise(yg, y_noise=y_noise, **kw)
    g = torch.from_numpy(rng.standard_normal(tuple(out.shape))).to(dtype).cuda()
    (gl,) = torch.autograd.grad(out, yg, g, retain_graph=True)
    (gl2,) = torch.autograd.grad(out, yg, g)
    assert torch.equal(gl, gl2)                                   # run-to-run bit equality
    rows = list(check)
    y64 = yg.detach()[rows].double().cpu().requires_grad_(True)
    A = restatement(y64, cfg, y_noise=y_noise)
    (gr,) = torch.autograd.grad(A(y64), y64, g[rows].double().cpu())
    return gl[rows].cpu(), gr


@pytest.mark.gpu
def test_gpu_config2_slice():
    """8 ch x 2 min at 48 kHz, stationary, float32 (config 2's geometry), against the restatement on two channels."""
    cfg = orc.GateConfig(sr=48000, stationary=True)
    gl, gr = _gpu_case(8, 120, 48000, cfg, check=(0, 5))
    _close(gl, gr, 2e-5)


@pytest.mark.gpu
def test_gpu_nonstationary_2048_slice():
    """Config 3's geometry (non-stationary, n_fft 2048, 48 kHz, default chunks): 4 ch x 40 s, one channel checked."""
    cfg = orc.GateConfig(sr=48000, stationary=False, n_fft=2048)
    gl, gr = _gpu_case(4, 40, 48000, cfg, check=(2,))
    _close(gl, gr, 2e-5)


@pytest.mark.gpu
def test_gpu_general_family_float64():
    cfg = orc.GateConfig(sr=16000, stationary=True, n_fft=512, win_length=400, hop_length=100, chunk_size=40000,
                         padding=5000)
    gl, gr = _gpu_case(2, 6, 16000, cfg, dtype=torch.float64, check=(1,))
    _close(gl, gr, 1e-9)


@pytest.mark.gpu
def test_gpu_nonstationary_offset_rows():
    """Rows that start 3 samples past a 16-byte boundary, non-stationary n_fft 1024."""
    cfg = orc.GateConfig(sr=16000, stationary=False, chunk_size=60000, padding=8000)
    gl, gr = _gpu_case(3, 10, 16000, cfg, offset=3, check=(2,))
    _close(gl, gr, 2e-5)


@pytest.mark.gpu
def test_gpu_float64_and_memory_returns_to_baseline():
    import gc
    import noisereduce_b200 as nr
    y = torch.from_numpy(synth_small(C=2, n=16000 * 20)).double().cuda()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    yg = y.clone().requires_grad_(True)
    out = nr.reduce_noise(yg, sr=16000, stationary=True, chunk_size=100000, padding=10000)
    out.square().sum().backward()
    assert yg.grad.dtype == torch.float64 and torch.isfinite(yg.grad).all()
    del out, yg
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == base
