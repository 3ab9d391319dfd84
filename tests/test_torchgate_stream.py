"""TorchGate.stream(): the non-stationary TorchGate on rows that arrive block by block.

The contract is bit-identity: torch.cat of every push() output and finish() equals tg(x) for the concatenated x, however
x is cut into blocks.  On the CPU simulator (tests/cusim) the .cu sources run on the host with CPU tensors; the
gpu-marked tests repeat the comparison on the nvcc build at the size of a live multi-row front end."""
import ctypes

import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from noisereduce_b200.torchgate import TorchGate, TorchGateStream
from tests.cusim_util import cusim_library
from tests.synth_host import synth_torchgate

SR, HOP = 16000, 256


@pytest.fixture(scope="module")
def lib():
    return cusim_library()


def signal(B, L, seed=7):
    return torch.from_numpy(synth_torchgate(B=B, n=L, seed=seed))


def run_stream(tg, x, sizes, lib=None):
    """Push x in blocks of the given sizes (cycled), check the documented counts after every push, return the output."""
    s = tg.stream(x.shape[0], _lib=lib)
    assert isinstance(s, TorchGateStream)
    outs, i, k = [], 0, 0
    while i < x.shape[1]:
        n = sizes[k % len(sizes)]
        k += 1
        y = s.push(x[:, i:i + n])
        i = min(i + n, x.shape[1])
        assert s.samples_received == i
        assert s.samples_returned == s.returned_after(i) == sum(o.shape[1] for o in outs) + y.shape[1]
        assert 0 <= s.samples_received - s.samples_returned <= s.latency_samples
        assert y.dtype == x.dtype and y.shape[0] == x.shape[0]
        outs.append(y)
    outs.append(s.finish())
    return torch.cat(outs, 1)


NO_SMOOTHING = dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None)


@pytest.mark.parametrize("sizes", [[1], [100], [255], [256], [257], [4096], [10 ** 9], "random"])
def test_block_sizes_equal_forward(lib, sizes):
    tg = TorchGate(sr=SR, nonstationary=True)
    L = 6000 if sizes != [1] else 3100                   # (one-sample pushes are slow on the simulator)
    x = signal(3, L)
    if sizes == "random":
        sizes = list(np.random.default_rng(3).integers(1, 1500, size=50))
    assert torch.equal(run_stream(tg, x, sizes, lib), tg(x, _lib=lib))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_partitions_one_row(lib, seed):
    tg = TorchGate(sr=SR, nonstationary=True)
    rng = np.random.default_rng(seed)
    L = int(rng.integers(2048, 9000))
    x = signal(1, L, seed=seed)
    sizes = list(rng.integers(0, 2000, size=40))        # (empty blocks included)
    assert torch.equal(run_stream(tg, x, sizes, lib), tg(x, _lib=lib))


@pytest.mark.parametrize("L", [2048, 2048 + 100, 7 * 256, 20000])
def test_lengths(lib, L):
    tg = TorchGate(sr=SR, nonstationary=True)
    if L < 2048:
        s = tg.stream(1, _lib=lib)
        s.push(signal(1, L))
        with pytest.raises(Exception, match="x must be bigger than 2048"):
            s.finish()
        return
    x = signal(1, L, seed=L)
    y = run_stream(tg, x, [333], lib)
    assert y.shape[1] == (L // HOP) * HOP
    assert torch.equal(y, tg(x, _lib=lib))


@pytest.mark.parametrize("kw", [dict(n_movemean_nonstationary=7), dict(n_movemean_nonstationary=1), NO_SMOOTHING,
                                dict(time_mask_smooth_ms=239), dict(prop_decrease=0.6),
                                dict(n_movemean_nonstationary=8, time_mask_smooth_ms=32)],
                         ids=["movemean7", "movemean1", "no-smoothing", "largest-nt", "prop0.6", "even-right+nt"])
def test_gate_parameters(lib, kw):
    tg = TorchGate(sr=SR, nonstationary=True, **kw)
    x = signal(3, 9000, seed=5)
    for sizes in ([320], [4000, 17]):
        assert torch.equal(run_stream(tg, x, sizes, lib), tg(x, _lib=lib)), sizes


def test_largest_time_extent_is_the_rows_limit():
    """time_mask_smooth_ms=239 (nt = 14 frames) is the largest the rows kernels take at 16 kHz with the default
    frequency extent (nf = 16 bins)."""
    from noisereduce_b200.torchgate.torchgate import _rows_smoothing_refusal
    tg = TorchGate(sr=SR, nonstationary=True, time_mask_smooth_ms=239)
    nf, nt = tg._extents
    assert (nf, nt) == (16, 14)
    assert _rows_smoothing_refusal(nf, nt, True) is None
    assert _rows_smoothing_refusal(nf, nt + 1, True) is not None


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_precision(lib, dtype):
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(2, 7000, seed=9).to(dtype)
    y = run_stream(tg, x, [320, 1000], lib)
    assert y.dtype == dtype
    assert torch.equal(y, tg(x, _lib=lib))


def test_latency_closed_form():
    tg = TorchGate(sr=SR, nonstationary=True)
    s = tg.stream(1)
    assert (s._right, s._nt) == (10, 3)
    assert s.latency_samples == 512 + 256 * 17 - 1 == 4863
    # the bound is reached: the largest held-back count over R equals latency_samples
    assert max(R - s.returned_after(R) for R in range(0, 20000)) == s.latency_samples
    for kw in (dict(n_movemean_nonstationary=8, time_mask_smooth_ms=32), NO_SMOOTHING, dict(n_movemean_nonstationary=1)):
        s = TorchGate(sr=SR, nonstationary=True, **kw).stream(1)
        assert max(R - s.returned_after(R) for R in range(0, 20000)) == s.latency_samples, kw


def _heap_bytes():
    class MallInfo2(ctypes.Structure):
        _fields_ = [(n, ctypes.c_size_t) for n in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                                   "uordblks", "fordblks", "keepcost")]
    libc = ctypes.CDLL(None)
    libc.mallinfo2.restype = MallInfo2
    m = libc.mallinfo2()
    return m.hblkhd, m.hblks


def test_state_does_not_grow(lib):
    """The simulator's device buffers are host allocations; the stream's large ones are mmapped blocks.  Their count and
    size are the same after 10 pushes and after 1000."""
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(2, 320 * 1000, seed=1)
    s = tg.stream(2, _lib=lib)
    for k in range(1000):
        s.push(x[:, 320 * k:320 * (k + 1)])
        if k == 9:
            after_10 = _heap_bytes()
    assert _heap_bytes() == after_10
    s.finish()


# ---- refusals and misuse ------------------------------------------------------------------------------------------------
@pytest.fixture
def no_handles(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a library handle was made")
    monkeypatch.setattr(_cabi, "Gate", boom)


@pytest.mark.parametrize("kw,arg", [(dict(), "nonstationary"), (dict(nonstationary=True, n_fft=512), "n_fft"),
                                    (dict(nonstationary=True, hop_length=128), "hop_length"),
                                    (dict(nonstationary=True, time_mask_smooth_ms=400), "time_mask_smooth_ms")])
def test_refusals_before_any_handle(no_handles, kw, arg):
    tg = TorchGate(sr=SR, **kw)
    with pytest.raises(NotImplementedError, match=arg):
        tg.stream(1)


@pytest.mark.parametrize("block,exc,match", [(torch.zeros(2, 10, dtype=torch.float64), NotImplementedError, "float64"),
                                             (torch.zeros(2, 10, requires_grad=True), NotImplementedError, "grad"),
                                             (torch.zeros(3, 10), ValueError, "2, n"),
                                             (torch.zeros(10), ValueError, "2, n"),
                                             (torch.zeros(2, 10, dtype=torch.int16), ValueError, "float32")])
def test_bad_blocks_before_any_handle(no_handles, block, exc, match):
    s = TorchGate(sr=SR, nonstationary=True).stream(2, _lib=object())
    with pytest.raises(exc, match=match):
        s.push(block)


def test_cuda_only_without_lib():
    s = TorchGate(sr=SR, nonstationary=True).stream(1)
    with pytest.raises(ValueError, match="CUDA"):
        s.push(torch.zeros(1, 10))


def test_misuse(lib):
    tg = TorchGate(sr=SR, nonstationary=True)
    s = tg.stream(2, _lib=lib)
    s.push(signal(2, 1000))
    with pytest.raises(ValueError, match="float32"):
        s.push(torch.zeros(2, 10, dtype=torch.float16))
    with pytest.raises(Exception, match="x must be bigger than 2048"):
        s.finish()
    s.push(signal(2, 2000))
    s.finish()
    with pytest.raises(ValueError, match="after finish"):
        s.push(torch.zeros(2, 10))
    with pytest.raises(ValueError, match="twice"):
        s.finish()
    with pytest.raises(ValueError, match="n_rows"):
        tg.stream(0)


# ---- C ABI ----------------------------------------------------------------------------------------------------------------
def torch_gate(lib, **kw):
    p = dict(lib=lib, surface=_cabi.SURFACE_TORCH, stationary=0, n_fft=1024, win_length=1024, hop_length=256, n_grad_freq=16,
             n_grad_time=3, std_ddof=1, sr=float(SR), prop_decrease=1.0, top_db=40.0, n_movemean=20, thresh_n_mult=1.3,
             sigmoid_slope=10.0)
    p.update(kw)
    g = _cabi.Gate(**p)
    g.set_window(torch.hann_window(p["win_length"]).numpy())
    return g


def test_cabi_error_codes(lib):
    for kw in (dict(stationary=1), dict(n_fft=1000, win_length=1000, hop_length=250)):      # stationary, generic
        g = torch_gate(lib, **kw)
        with pytest.raises(_cabi.GateError) as e:
            g.tstream_begin(1)
        assert e.value.code == _cabi.ERR_STATE
    g = _cabi.Gate(lib=lib, surface=0, stationary=0, n_fft=1024, win_length=1024, hop_length=256, sr=float(SR))
    with pytest.raises(_cabi.GateError) as e:
        g.tstream_begin(1)
    assert e.value.code == _cabi.ERR_STATE

    g = torch_gate(lib)
    x = signal(2, 6000).contiguous()
    y = torch.zeros(2, 8000)
    g.tstream_begin(2)
    with pytest.raises(_cabi.GateError) as e:                 # the other calls are blocked while the stream is open
        g.run_device(x.data_ptr(), y.data_ptr(), np.float32, 2, 6000, 6000, 8000)
    assert e.value.code == _cabi.ERR_STATE
    with pytest.raises(_cabi.GateError) as e:
        g.run_rows([(x.data_ptr(), y.data_ptr(), 6000, 1)], np.float32, True)
    assert e.value.code == _cabi.ERR_STATE
    with pytest.raises(_cabi.GateError) as e:
        g.torch_apply_masks_device(x.data_ptr(), y.data_ptr(), np.float32, 2, 6000, 6000, 8000)
    assert e.value.code == _cabi.ERR_STATE
    with pytest.raises(_cabi.GateError) as e:
        g.torch_apply_masks_rows([(x.data_ptr(), y.data_ptr(), 6000, 1)], np.float32, True)
    assert e.value.code == _cabi.ERR_STATE
    with pytest.raises(_cabi.GateError) as e:
        g.stream_begin(np.float32, 2)
    assert e.value.code == _cabi.ERR_STATE
    # too little output capacity: refused, nothing consumed
    with pytest.raises(_cabi.GateError) as e:
        g.tstream_push(x.data_ptr(), 6000, 6000, y.data_ptr(), 8000, 10)
    assert e.value.code == _cabi.ERR_ARG
    got = g.tstream_push(x.data_ptr(), 6000, 6000, y.data_ptr(), 8000, 8000)
    with pytest.raises(_cabi.GateError) as e:
        g.tstream_finish(y[:, got:].data_ptr(), 8000, 1)
    assert e.value.code == _cabi.ERR_ARG
    rest = g.tstream_finish(y[:, got:].data_ptr(), 8000, 8000 - got)
    assert got + rest == (6000 // HOP) * HOP
    tg = TorchGate(sr=SR, nonstationary=True)
    ref = tg(x, _lib=lib)
    assert torch.equal(y[:, :got + rest], ref)
    # the handle works normally after finish
    y2 = torch.zeros(2, ref.shape[1])
    g.run_device(x.data_ptr(), y2.data_ptr(), np.float32, 2, 6000, 6000, ref.shape[1])
    assert torch.equal(y2, ref)


# ---- H100 ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_256_rows_60s_20ms_blocks_side_stream():
    torch.manual_seed(0)
    B, L = 256, 60 * SR
    x = (torch.randn(B, L, device="cuda") * 0.1 + torch.sin(torch.arange(L, device="cuda") * 0.05)[None]).contiguous()
    tg = TorchGate(sr=SR, nonstationary=True).to("cuda")
    ref = tg(x)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        s = tg.stream(B)
        outs = [s.push(x[:, i:i + 320]) for i in range(0, L, 320)]
        outs.append(s.finish())
        y = torch.cat(outs, 1)
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(y, ref)


@pytest.mark.gpu
def test_gpu_random_blocks_one_row_and_memory():
    rng = np.random.default_rng(4)
    L = 10 * SR + 77
    x = torch.from_numpy(synth_torchgate(B=1, n=L, seed=4)).cuda()
    tg = TorchGate(sr=SR, nonstationary=True).to("cuda")
    ref = tg(x)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    alloc0 = torch.cuda.memory_allocated()
    for dtype in (torch.float32, torch.float16):
        xs = x.to(dtype)
        s = tg.stream(1)
        outs, i = [], 0
        while i < L:
            n = int(rng.integers(1, 2001))
            outs.append(s.push(xs[:, i:i + n]))
            i = min(i + n, L)
            assert s.samples_returned == s.returned_after(i)
        outs.append(s.finish())
        y = torch.cat(outs, 1)
        assert torch.equal(y, ref if dtype == torch.float32 else tg(xs))
        del outs, y, s
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= alloc0 + (1 << 20)       # (tg(xs) above is a new reference, not kept)
    torch.cuda.empty_cache()
    assert torch.cuda.mem_get_info()[0] >= free0 - (4 << 20)          # the stream's device state is released
