"""TorchGate.forward(x, lengths=...): a zero-padded batch of rows of different lengths, each row gated as if alone.

The contract is bit-identity with a loop of per-row calls: row b's first (lengths[b] // hop) * hop output samples equal
forward(x[b:b+1, :lengths[b]], xn_b)[0] in every bit, the rest of the row is zero, and samples of x past lengths[b] are
never read.  On the CPU simulator (tests/cusim) the .cu sources run on the host with CPU tensors; the gpu-marked tests
repeat the comparison on the nvcc build at the size of a training batch."""
import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from noisereduce_b200.torchgate import TorchGate
from oracle import torchgate_oracle as TO
from tests.cusim_util import cusim_library
from tests.synth_host import synth_torchgate

TOL = 5e-6     # FP32 pipeline vs the float64 oracle, as in test_cusim_torchgate.py
SR, HOP, L = 16000, 256, 6000
LENGTHS = [L - 1, 2048, L, 4999]       # 2 win_length, off the hop grid, L - 1 and L, shuffled


@pytest.fixture(scope="module")
def lib():
    return cusim_library()


def batch(B=4, fill=0.0, seed=11):
    """[B, L] rows with row b's samples past LENGTHS[b] set to `fill`, and the unpadded rows."""
    x = torch.from_numpy(synth_torchgate(B=B, n=L, seed=seed))
    xp = x.clone()
    for b, n in enumerate(LENGTHS[:B]):
        xp[b, n:] = fill
    return xp, x


def row_xn(xn, b):
    return None if xn is None else (xn[b:b + 1] if xn.ndim == 2 and xn.shape[0] > 1 else xn)


def loop(tg, x, lengths, xn=None, lib=None):
    return [tg(x[b:b + 1, :n].contiguous(), row_xn(xn, b), _lib=lib)[0] for b, n in enumerate(lengths)]


def assert_rows_equal(y, refs, lengths):
    assert tuple(y.shape) == (len(lengths), (y.shape[1] // HOP) * HOP)
    for b, (r, n) in enumerate(zip(refs, lengths)):
        k = (n // HOP) * HOP
        assert r.shape[0] == k and r.dtype == y.dtype, b
        assert torch.equal(y[b, :k], r), b
        assert bool((y[b, k:] == 0).all()), b


def make_xn(kind):
    src = torch.from_numpy(synth_torchgate(B=4, n=3000, seed=5))
    return {"none": None, "1d": src[0], "1row": src[:1], "Brows": src}[kind]


NO_SMOOTHING = dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None)
GATES = {"stationary": dict(), "nonstationary": dict(nonstationary=True), "prop0.7": dict(prop_decrease=0.7),
         "no-smoothing": NO_SMOOTHING, "nonstationary-prop0.7": dict(nonstationary=True, prop_decrease=0.7),
         "nonstationary-no-smoothing": dict(nonstationary=True, **NO_SMOOTHING)}


# (the non-stationary gate ignores xn: one xn form suffices there)
@pytest.mark.parametrize("gate,xn_kind", [(gate, xn) for gate in GATES for xn in ("none", "1d", "1row", "Brows")
                                          if not (gate.startswith("nonstationary") and xn in ("1row", "Brows"))])
def test_rows_equal_the_per_row_loop(lib, gate, xn_kind):
    kw = GATES[gate]
    xn = make_xn(xn_kind)
    tg = TorchGate(sr=SR, **kw)
    _, x = batch()
    refs = loop(tg, x, LENGTHS, xn, lib)
    for fill in (float("nan"), 1e30):                  # the padding is never read
        xp, _ = batch(fill=fill)
        y = tg(xp, xn, lengths=LENGTHS, _lib=lib)
        assert y.dtype == torch.float32
        assert_rows_equal(y, refs, LENGTHS)
    # lengths as a tensor, in the same call form
    y = tg(batch(fill=float("nan"))[0], xn, lengths=torch.tensor(LENGTHS), _lib=lib)
    assert_rows_equal(y, refs, LENGTHS)


@pytest.mark.parametrize("kw", [dict(), dict(nonstationary=True, prop_decrease=0.8)], ids=["stationary", "nonstationary"])
def test_rows_match_the_oracle(lib, kw):
    """An independent check: each row against the float64 oracle of the reference on the truncated row."""
    w = torch.hann_window(1024).numpy()
    xp, x = batch(fill=float("nan"))
    y = TorchGate(sr=SR, **kw)(xp, lengths=LENGTHS, _lib=lib).numpy()
    for b, n in enumerate(LENGTHS):
        ref = TO.torchgate_forward(x[b:b + 1, :n].numpy().astype(np.float64), SR, window=w, **kw)[0]
        got = y[b, :ref.shape[0]]
        assert float(np.abs(got - ref).max() / np.abs(ref).max()) < TOL, b


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_precision_rows(lib, dtype):
    tg = TorchGate(sr=SR)
    xp, x = batch(fill=float("nan"))
    y = tg(xp.to(dtype), lengths=LENGTHS, _lib=lib)
    assert y.dtype == dtype
    assert_rows_equal(y, loop(tg, x.to(dtype), LENGTHS, lib=lib), LENGTHS)


@pytest.mark.parametrize("kw", [dict(), dict(prop_decrease=0.7)], ids=["stationary", "prop0.7"])
def test_smoothing_beyond_the_in_synthesis_lanes(lib, kw):
    """sr 8000: the default 500 Hz filter has nf = 32, beyond the byte lanes of the synthesis kernel, so the numerators
    come from k_smooth_generic<ROWS>."""
    tg = TorchGate(sr=8000, **kw)
    assert tg._extents[0] == 32
    xp, x = batch(fill=float("nan"))
    assert_rows_equal(tg(xp, lengths=LENGTHS, _lib=lib), loop(tg, x, LENGTHS, lib=lib), LENGTHS)


@pytest.mark.parametrize("kw", [dict(sr=SR), dict(sr=SR, nonstationary=True, prop_decrease=0.8), dict(sr=8000, prop_decrease=0.7)],
                         ids=["stationary", "nonstationary", "stationary-8k"])
def test_backward_equals_the_per_row_backward(lib, kw):
    gen = torch.Generator().manual_seed(3)
    xp, x = batch(fill=float("nan"))
    xp = xp.requires_grad_(True)
    tg = TorchGate(**kw)
    y = tg(xp, lengths=LENGTHS, _lib=lib)
    g = torch.randn(y.shape, generator=gen)
    (y * g).sum().backward()
    grad = xp.grad.clone()
    for b, n in enumerate(LENGTHS):
        k = (n // HOP) * HOP
        xb = x[b:b + 1, :n].clone().requires_grad_(True)
        yb = TorchGate(**kw)(xb, _lib=lib)
        (yb * g[b:b + 1, :k]).sum().backward()
        assert torch.equal(grad[b, :n], xb.grad[0]), b
        assert bool((grad[b, n:] == 0).all()), b
    # <A v, g> == <v, A^T g> for the linear map A = the rows gate with these masks (b200gate_torch_apply_masks_rows)
    tg2 = TorchGate(**kw)
    xg = batch()[1].requires_grad_(True)
    y2 = tg2(xg, lengths=LENGTHS, _lib=lib)
    (y2 * g).sum().backward()
    gate = next(iter(tg2._gate.values()))
    v = torch.randn(xg.shape, generator=gen) * 0.05
    for b, n in enumerate(LENGTHS):
        v[b, (n // HOP) * HOP:] = 0.0             # (A^T is taken with zeros past the output length, as _adjoint does)
    Av = torch.zeros(y2.shape)
    gate.torch_apply_masks_rows([(v.data_ptr() + b * L * 4, Av.data_ptr() + b * y2.shape[1] * 4, n, 1)
                                 for b, n in enumerate(LENGTHS)], np.float32, True)
    lhs, rhs = float((Av.double() * g.double()).sum()), float((v.double() * xg.grad.double()).sum())
    assert abs(lhs - rhs) <= 2e-5 * max(abs(lhs), abs(rhs), 1e-3)
    # a second forward overwrites the masks: backward of the first must refuse
    ya = tg2(xg, lengths=LENGTHS, _lib=lib)
    tg2(xg.detach() * 0.5, lengths=LENGTHS, _lib=lib)
    with pytest.raises(RuntimeError, match="another forward ran"):
        ya.sum().backward()


def test_refusals_before_any_handle(lib, monkeypatch):
    def no_handle(**kw):
        raise AssertionError("a handle was created")

    monkeypatch.setattr(_cabi, "Gate", no_handle)
    xp, _ = batch()
    with pytest.raises(NotImplementedError, match="n_fft"):
        TorchGate(sr=SR, n_fft=512)(xp, lengths=LENGTHS, _lib=lib)
    with pytest.raises(NotImplementedError, match="float64"):
        TorchGate(sr=SR)(xp.double(), lengths=LENGTHS, _lib=lib)
    with pytest.raises(NotImplementedError, match="time_mask_smooth_ms"):
        TorchGate(sr=SR, nonstationary=True, time_mask_smooth_ms=1000)(xp, lengths=LENGTHS, _lib=lib)
    # smoothing filters beyond the 16-bit numerators of the n_fft 1024 family (their handles are general-family ones),
    # for each gate; the largest time smoothing that fits, and a small-nf one up to the ring limit, are not refused
    for kw in (dict(time_mask_smooth_ms=240), dict(nonstationary=True, time_mask_smooth_ms=240),
               dict(freq_mask_smooth_hz=2200), dict(nonstationary=True, freq_mask_smooth_hz=2200),
               dict(nonstationary=True, freq_mask_smooth_hz=40, time_mask_smooth_ms=47 * 16)):
        with pytest.raises(NotImplementedError, match="freq_mask_smooth_hz"):
            TorchGate(sr=SR, **kw)(xp, lengths=LENGTHS, _lib=lib)
    monkeypatch.undo()
    for kw in (dict(time_mask_smooth_ms=224), dict(nonstationary=True, time_mask_smooth_ms=224),
               dict(nonstationary=True, freq_mask_smooth_hz=40, time_mask_smooth_ms=46 * 16)):
        tg = TorchGate(sr=SR, **kw)
        assert tg(xp, lengths=LENGTHS, _lib=lib).shape == (4, (L // HOP) * HOP)
    monkeypatch.setattr(_cabi, "Gate", no_handle)
    tg = TorchGate(sr=SR)
    with pytest.raises(Exception, match="x must be bigger than 2048"):
        tg(xp, lengths=[L, 2047, L, L], _lib=lib)
    for bad in ([L, L, L], [L, L, L, L + 1], torch.tensor([LENGTHS]), torch.tensor(LENGTHS, dtype=torch.float32),
                [L, L, L, 5000.0]):
        with pytest.raises(ValueError):
            tg(xp, lengths=bad, _lib=lib)


def test_full_length_rows_agree_with_the_batch_call(lib):
    """forward(x, lengths=[L] * B) is forward(x) up to the last bit at synthesis work-item seams."""
    x = torch.from_numpy(synth_torchgate(B=4, n=40 * HOP))
    for kw in (dict(), dict(nonstationary=True)):
        tg = TorchGate(sr=SR, **kw)
        y0 = tg(x, _lib=lib)
        y1 = tg(x, lengths=[x.shape[1]] * 4, _lib=lib)
        d = float((y1 - y0).abs().max())
        print(f"[full-length rows] {kw or 'stationary'}: largest difference {d:.3e} (max |y| {float(y0.abs().max()):.3e})")
        assert d <= 4 * float(torch.finfo(torch.float32).eps) * float(y0.abs().max())


def test_cabi_rows_on_the_torch_surface(lib):
    kw = dict(surface=_cabi.SURFACE_TORCH, stationary=0, n_fft=1024, win_length=1024, hop_length=256, n_grad_freq=16,
              n_grad_time=3, std_ddof=1, chunk_size=0, padding=0, sr=float(SR), prop_decrease=1.0, n_std_thresh=1.5,
              top_db=40.0, n_movemean=20, thresh_n_mult=1.3, sigmoid_slope=10.0)
    window = torch.hann_window(1024).numpy()
    _, x = batch()
    xs = x.numpy()
    for stationary in (0, 1):
        g = _cabi.Gate(lib=lib, **dict(kw, stationary=stationary))
        g.set_window(window)
        with pytest.raises(_cabi.GateError) as e:                    # nothing to apply yet
            g.torch_apply_masks_rows([(xs.ctypes.data, xs.ctypes.data, L, 1)], np.float32, False)
        assert e.value.code == _cabi.ERR_STATE
        # host rows packed in one buffer each way
        buf = np.concatenate([xs[b, :n] for b, n in enumerate(LENGTHS)])
        out = np.full(buf.size, 7.0, np.float32)
        offs = [int(o) for o in np.concatenate([[0], np.cumsum(LENGTHS)[:-1]])]
        g.run_rows([(buf.ctypes.data + 4 * o, out.ctypes.data + 4 * o, n, 1) for o, n in zip(offs, LENGTHS)],
                   np.float32, False)
        st = g.stats()
        assert st["units"] == len(LENGTHS) and st["frames"] == sum(n // HOP + 1 for n in LENGTHS)
        for o, n in zip(offs, LENGTHS):
            k = (n // HOP) * HOP
            ref = g.run_host(np.ascontiguousarray(buf[o:o + n])[None, :])[0, :k]
            assert np.array_equal(out[o:o + k], ref)
        # the masks of the rows run are kept for the same lengths only
        g.run_rows([(buf.ctypes.data + 4 * o, out.ctypes.data + 4 * o, n, 1) for o, n in zip(offs, LENGTHS)],
                   np.float32, False)
        with pytest.raises(_cabi.GateError) as e:
            g.torch_apply_masks_rows([(buf.ctypes.data + 4 * o, out.ctypes.data + 4 * o, n - 1, 1)
                                      for o, n in zip(offs, LENGTHS)], np.float32, False)
        assert e.value.code == _cabi.ERR_STATE
        for rows, dtype in (([(buf.ctypes.data, out.ctypes.data, 2047, 1)], np.float32),
                            ([(buf.ctypes.data, out.ctypes.data, 4096, 1)], np.float64)):
            with pytest.raises(_cabi.GateError) as e:
                g.run_rows(rows, dtype, False)
            assert e.value.code == _cabi.ERR_ARG
        g.close()
    g = _cabi.Gate(lib=lib, **dict(kw, surface=_cabi.SURFACE_TORCH_CHUNKED))
    with pytest.raises(_cabi.GateError) as e:
        g.run_rows([(xs.ctypes.data, xs.ctypes.data + 4 * L, L, 1)], np.float32, False)
    assert e.value.code == _cabi.ERR_STATE
    g.close()


# ---- on the GPU ------------------------------------------------------------------------------------------------------
def _config4_batch(B=256, sr=16000, seed=7):
    """B rows padded to 10 s at 16 kHz with seeded lengths uniform in 1-10 s (the size of BASELINE config 4's batch)."""
    Lmax = 10 * sr
    lengths = torch.randint(sr, Lmax + 1, (B,), generator=torch.Generator().manual_seed(seed))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.arange(Lmax, device="cuda", dtype=torch.float32) / sr
    x = 0.05 * torch.randn((B, Lmax), device="cuda", generator=gen)
    x += 0.3 * ((t % 1.0) < 0.4) * torch.sin(2 * np.pi * 440.0 * t)
    x[torch.arange(Lmax, device="cuda")[None, :] >= lengths.cuda()[:, None]] = 0.0
    return x, lengths


def _envelope_on_the_host(monkeypatch):
    """TorchGate._ola_envelope sums the squared window with index_add_, whose float atomics on CUDA add a sample's
    overlapping frames in no fixed order; computed on the CPU and copied over, the same divisor comes out on every call."""
    env = TorchGate._ola_envelope
    monkeypatch.setattr(TorchGate, "_ola_envelope", lambda self, L, device: env(self, L, torch.device("cpu")).to(device))


@pytest.mark.gpu
@pytest.mark.parametrize("envelope", ["cuda", "host"])
@pytest.mark.parametrize("nonstationary", [False, True], ids=["stationary", "nonstationary"])
def test_gpu_config4_batch_equals_the_per_row_calls(nonstationary, envelope, monkeypatch):
    """Forward: bit-identical.  Backward: bit-identical when the overlap-add envelope is the same on both sides (host);
    with the envelope as TorchGate computes it on the device, within float32 rounding (DESIGN §4)."""
    if envelope == "host":
        _envelope_on_the_host(monkeypatch)
    x, lengths = _config4_batch()
    B, Lmax = x.shape
    tg = TorchGate(sr=16000, nonstationary=nonstationary)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    side = torch.cuda.Stream()
    xg = x.clone().requires_grad_(True)
    g = torch.randn((B, (Lmax // HOP) * HOP), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        y = tg(xg, lengths=lengths.cuda(), _lib=None)
        (y * g).sum().backward()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    order = sorted(range(B), key=lambda i: int(lengths[i]))
    subset = [order[round(k * (B - 1) / 31)] for k in range(32)]
    worst = 0.0
    exact = True
    for i in subset:
        n = int(lengths[i])
        k = (n // HOP) * HOP
        xb = x[i:i + 1, :n].clone().requires_grad_(True)
        yb = TorchGate(sr=16000, nonstationary=nonstationary)(xb)
        assert torch.equal(y[i, :k].detach(), yb[0].detach()), i
        assert bool((y[i, k:] == 0).all()), i
        (yb * g[i:i + 1, :k]).sum().backward()
        gb, gr = xg.grad[i, :n], xb.grad[0]
        exact &= bool(torch.equal(gb, gr))
        worst = max(worst, float((gb - gr).abs().max() / gr.abs().max().clamp_min(1e-30)))
        assert bool((xg.grad[i, n:] == 0).all()), i
        del xb, yb, gb, gr
    print(f"[gpu rows backward] {'nonstationary' if nonstationary else 'stationary'}, envelope on the {envelope}: "
          f"bit-identical to the per-row backward on all 32 rows: {exact}; largest relative difference {worst:.3e}")
    assert exact if envelope == "host" else worst <= 4 * float(torch.finfo(torch.float32).eps)
    assert float(y.detach().abs().max()) > 0
    del y, g, xg, x
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= base - B * Lmax * 4      # inputs, outputs and graph are gone


@pytest.mark.gpu
def test_gpu_unaligned_float16_rows():
    """Row pointers off 16-byte alignment: a float16 view with a storage offset and a row stride longer than the row, and
    rows of 40001 samples, so that the float32 rows the kernels read start 4 bytes apart from 16-byte alignment."""
    B, Lmax, pitch = 8, 40_001, 40_003
    store = torch.randn(B * pitch + 5, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)) * 0.1
    x = store.to(torch.float16).as_strided((B, Lmax), (pitch, 1), storage_offset=3)
    lengths = [Lmax, 2048, 39_999, 12_345, 30_000, 2049, 20_480, 40_000]
    for nonstationary in (False, True):
        tg = TorchGate(sr=16000, nonstationary=nonstationary)
        y = tg(x, lengths=lengths)
        assert y.dtype == torch.float16
        assert_rows_equal(y, [tg(x[b:b + 1, :n])[0] for b, n in enumerate(lengths)], lengths)
