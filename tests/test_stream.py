"""NoiseReduceStream / b200gate_stream_*: a recording pushed block by block returns, concatenated, exactly what
reduce_noise() returns on the whole recording (shape, dtype, every bit), and after R samples exactly E(R) of them.

The simulator tests run the product's sources on the CPU (tests/cusim) with one chunk per slice, so long pushes are
sliced and the device window is compacted; the GPU tests use config 2's geometry on an H100."""
import ctypes

import numpy as np
import pytest

from noisereduce_b200 import _cabi
from tests.cusim_util import cusim_library
from tests.synth_host import synth_small

SR = 16000


def expected_emitted(R, cs, pad):
    return cs * max(0, (R - pad) // cs) if R > cs else 0


def schedules(N, cs, hop, seed=0):
    """One block; fixed blocks that do not divide chunk_size; seeded random sizes with 0, 1, < hop and multi-chunk."""
    fixed = [min(1700, N - i) for i in range(0, N, 1700)]
    rng = np.random.default_rng(seed)
    rand, left = [0, 1], N - 1
    picks = [0, 1, hop - 1, 3 * cs + 17, 7, cs // 3]
    while left > 0:
        n = int(picks[len(rand) % len(picks)] if len(rand) < 12 else rng.integers(0, 2 * cs))
        n = min(n, left)
        rand.append(n)
        left -= n
    return {"one": [N], "fixed": fixed, "random": rand}


def run_stream(nr, y, sizes, flat=False, **kw):
    C = None if flat else y.shape[0]
    s = nr.NoiseReduceStream(n_channels=C, **kw)
    cs, pad = s.chunk_size, s.padding
    outs, R = [], 0
    for n in sizes:
        blk = y[..., R:R + n]
        out = s.push(blk)
        R += n
        assert s.samples_returned == expected_emitted(R, cs, pad)
        assert out.shape[-1] % cs == 0 and out.dtype == y.dtype
        outs.append(out)
    assert R == y.shape[-1]
    last = s.finish()
    assert last.shape[-1] < cs + pad or R <= cs
    outs.append(last)
    return np.concatenate(outs, axis=-1)


@pytest.fixture(scope="module")
def lib():
    return cusim_library()


@pytest.fixture
def sim(lib, monkeypatch):
    monkeypatch.setattr(_cabi, "_LIB", lib)
    monkeypatch.setenv("B200GATE_STREAM_SLICE_CHUNKS", "1")       # slice long pushes, compact the window
    import noisereduce_b200 as nr
    return nr


def _noise(C, n, seed=7):
    return (0.05 * np.random.default_rng(seed).standard_normal((C, n))).astype(np.float32)


BASE = dict(sr=SR, chunk_size=2500, padding=400)
CASES = {
    "stationary_from_stream": (dict(stationary=True), 12000, np.float32),
    "stationary_y_noise_1d": (dict(stationary=True, y_noise=_noise(1, 5000)[0]), 9000, np.float32),
    "stationary_y_noise_2ch": (dict(stationary=True, y_noise=_noise(2, 3000)), 9000, np.float32),
    "stationary_y_noise_noclip": (dict(stationary=True, y_noise=_noise(2, 6000), clip_noise_stationary=False), 9000,
                                  np.float32),
    "nonstationary_1024": (dict(stationary=False, time_constant_s=0.3), 12000, np.float32),
    "nonstationary_2048": (dict(stationary=False, n_fft=2048, time_constant_s=0.3), 12000, np.float32),
    "general_512_400_100": (dict(stationary=True, n_fft=512, win_length=400, hop_length=100), 9000, np.float32),
    "int16": (dict(stationary=True), 9000, np.int16),
    "float64": (dict(stationary=False, time_constant_s=0.3), 9000, np.float64),
    "float16_promoted": (dict(stationary=True), 9000, np.float16),
    "int32_nonstationary_promoted": (dict(stationary=False, time_constant_s=0.3), 9000, np.int32),
    "pad601": (dict(stationary=True, padding=601), 12000, np.float32),
    "pad_ge_cs": (dict(stationary=True, chunk_size=1500, padding=1600), 9000, np.float32),
    "pad_lt_hop": (dict(stationary=False, padding=100, time_constant_s=0.3), 9000, np.float32),
    "n_le_cs": (dict(stationary=True), 2300, np.float32),
    "n_eq_k_cs": (dict(stationary=False, time_constant_s=0.3), 10000, np.float32),
    "n_k_cs_plus_1": (dict(stationary=True), 10001, np.float32),
    "stationary_short_clip": (dict(stationary=True), 800, np.float32),
    "prop_decrease": (dict(stationary=True, prop_decrease=0.7), 9000, np.float32),
    "smoothing_off": (dict(stationary=True, freq_mask_smooth_hz=None, time_mask_smooth_ms=None), 9000, np.float32),
}


def _signal(dtype, n, C=2):
    y = synth_small(C=C, n=n)
    if np.dtype(dtype) == np.int16 or np.dtype(dtype) == np.int32:
        return np.round(y / np.abs(y).max() * 20000).astype(dtype)
    return y.astype(dtype)


@pytest.mark.parametrize("case", sorted(CASES))
def test_stream_equals_reduce_noise_on_simulator(sim, case):
    extra, N, dtype = CASES[case]
    kw = dict(BASE)
    kw.update(extra)
    y = _signal(dtype, N)
    ref = sim.reduce_noise(y, **kw)
    assert ref.dtype == y.dtype
    hop = (kw.get("hop_length") or (kw.get("win_length") or kw.get("n_fft", 1024)) // 4)
    for name, sizes in schedules(N, kw["chunk_size"], hop).items():
        got = run_stream(sim, y, sizes, **kw)
        assert got.shape == ref.shape and got.dtype == ref.dtype, name
        assert np.array_equal(got, ref), (case, name)


def test_stream_flat_blocks_on_simulator(sim):
    y = synth_small(C=1, n=9000)[0]
    kw = dict(BASE, stationary=True)
    ref = sim.reduce_noise(y, **kw)
    for sizes in schedules(9000, 2500, 256).values():
        got = run_stream(sim, y, sizes, flat=True, **kw)
        assert got.shape == (9000,) and np.array_equal(got, ref)


def test_stream_default_slices_on_simulator(lib, monkeypatch):
    """The library's own slice size (whole pushes at these sizes): same bits."""
    monkeypatch.setattr(_cabi, "_LIB", lib)
    import noisereduce_b200 as nr
    y = synth_small(C=2, n=12000)
    kw = dict(BASE, stationary=True)
    ref = nr.reduce_noise(y, **kw)
    for sizes in schedules(12000, 2500, 256, seed=3).values():
        assert np.array_equal(run_stream(nr, y, sizes, **kw), ref)


def test_stream_rejects_what_reduce_noise_rejects(sim):
    """A stationary recording shorter than the window: reduce_noise() takes short-clip thresholds at 800 samples and
    raises scipy's noverlap error at 700; finish() does the same."""
    y = synth_small(C=2, n=800)
    kw = dict(BASE, stationary=True)
    assert np.array_equal(run_stream(sim, y, [300, 0, 500], **kw), sim.reduce_noise(y, **kw))
    with pytest.raises(ValueError, match="noverlap must be less than nperseg"):
        sim.reduce_noise(y[:, :700], **kw)
    s = sim.NoiseReduceStream(n_channels=2, **kw)
    assert s.push(y[:, :700]).shape == (2, 0)
    with pytest.raises(ValueError, match="noverlap must be less than nperseg"):
        s.finish()
    with pytest.raises(ValueError, match="closed"):
        s.push(y[:, :10])


# ---- the C ABI ----------------------------------------------------------------------------------------------------
def _gate(nr, **kw):
    return nr.NoiseReduceStream(n_channels=2, **dict(BASE, **kw))._gate


def test_device_pointer_pushes_on_simulator(sim):
    """is_device = 1 (simulator "device" pointers are host pointers): same bits, n_out known at once."""
    y = synth_small(C=2, n=12000)
    kw = dict(stationary=False, time_constant_s=0.3)
    ref = sim.reduce_noise(y, **dict(BASE, **kw))
    g = _gate(sim, **kw)
    g.stream_begin(np.float32, 2)
    got = np.zeros_like(y)
    done = 0
    for i in range(0, 12000, 3100):
        blk = y[:, i:i + 3100]                                    # a view: row stride 12000
        cap = blk.shape[1] + 2500
        dst = got[:, done:]
        m = g.stream_push(blk.ctypes.data, blk.shape[1], 12000, True, dst.ctypes.data, 12000, min(cap, 12000))
        done += m
    m = g.stream_finish(got[:, done:].ctypes.data, 12000, 12000)
    assert done + m == 12000
    assert np.array_equal(got, ref)


def test_stream_c_abi_errors_on_simulator(sim):
    y = synth_small(C=2, n=6000)
    g = _gate(sim, stationary=False, time_constant_s=0.3)
    g.stream_begin(np.float32, 2)
    out = np.full((2, 6000), 123.0, np.float32)
    # out_capacity below n + chunk_size: ERR_ARG, nothing written, nothing consumed
    with pytest.raises(_cabi.GateError) as e:
        g.stream_push(y.ctypes.data, 1000, 6000, False, out.ctypes.data, 6000, 3499)
    assert e.value.code == _cabi.ERR_ARG
    assert np.all(out == 123.0)
    assert g.stream_push(y.ctypes.data, 3000, 6000, False, out.ctypes.data, 6000, 6000) == 2500
    # b200gate_run while the stream is open: refused
    with pytest.raises(_cabi.GateError) as e:
        g.run_host(y)
    assert e.value.code == _cabi.ERR_STATE
    # finish with less than chunk_size + padding of room: ERR_ARG, the stream stays open
    with pytest.raises(_cabi.GateError) as e:
        g.stream_finish(out.ctypes.data, 6000, 2899)
    assert e.value.code == _cabi.ERR_ARG
    assert g.stream_finish(out.ctypes.data, 6000, 6000) == 500
    with pytest.raises(_cabi.GateError) as e:                      # closed
        g.stream_push(y.ctypes.data, 10, 6000, False, out.ctypes.data, 6000, 6000)
    assert e.value.code == _cabi.ERR_STATE
    g.run_host(y)                                                  # the handle runs offline again
    # a stationary stream without thresholds: the push that would return a chunk is refused (ERR_STATE)
    gs = _gate(sim, stationary=True)                               # (the class would set them from its pushes)
    gs.stream_begin(np.float32, 2)
    assert gs.stream_push(y.ctypes.data, 2000, 6000, False, out.ctypes.data, 6000, 4500) == 0
    with pytest.raises(_cabi.GateError) as e:
        gs.stream_push(y[:, 2000:].ctypes.data, 1000, 6000, False, out.ctypes.data, 6000, 6000)
    assert e.value.code == _cabi.ERR_STATE
    # b200gate_stream_begin resets: a fresh stream on the same handle
    g.stream_begin(np.float32, 2)
    assert g.stream_push(y.ctypes.data, 100, 6000, False, out.ctypes.data, 6000, 6000) == 0


def test_stream_python_errors(sim):
    with pytest.raises(ValueError, match="chunk_size"):
        sim.NoiseReduceStream(sr=SR, n_channels=2, chunk_size=None)
    with pytest.raises(ValueError, match="clip_noise_stationary"):
        sim.NoiseReduceStream(sr=SR, n_channels=2, stationary=True, clip_noise_stationary=False)
    with pytest.raises(ValueError, match="freq_mask_smooth_hz needs to be at least"):
        sim.NoiseReduceStream(sr=SR, n_channels=2, stationary=True, freq_mask_smooth_hz=10)
    s = sim.NoiseReduceStream(n_channels=2, **BASE)
    s.push(np.zeros((2, 3000), np.float32))
    with pytest.raises(ValueError, match="expected a \\[2, n\\] block"):
        s.push(np.zeros((3, 100), np.float32))
    with pytest.raises(ValueError, match="dtype"):
        s.push(np.zeros((2, 100), np.float64))
    with pytest.raises(ValueError, match="real-valued"):
        s.push(np.zeros((2, 100), np.complex64))
    s.finish()
    with pytest.raises(ValueError, match="closed"):
        s.push(np.zeros((2, 100), np.float32))
    with pytest.raises(ValueError, match="closed"):
        s.finish()
    s = sim.NoiseReduceStream(n_channels=None, **BASE)
    with pytest.raises(ValueError, match="1-D"):
        s.push(np.zeros((2, 100), np.float32))
    with pytest.raises(ValueError, match="zero-size array"):
        sim.NoiseReduceStream(n_channels=2, **BASE).finish()


# ---- H100 -------------------------------------------------------------------------------------------------------
SR48 = 48000


def _cfg2_signal(C, N, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(N) / SR48
    tone = 0.3 * np.sin(2 * np.pi * 440.0 * t) * (np.sin(2 * np.pi * 0.5 * t) > 0)
    return (tone[None, :] + 0.05 * rng.standard_normal((C, N))).astype(np.float32)


def _random_blocks(N, hi, seed):
    rng = np.random.default_rng(seed)
    out, left = [], N
    while left > 0:
        n = min(left, int(rng.integers(0, hi + 1)))
        out.append(n)
        left -= n
    return out


@pytest.mark.gpu
def test_stream_config2_geometry_on_gpu():
    import noisereduce_b200 as nr
    N = 2_000_000
    y = _cfg2_signal(3, N)
    kw = dict(sr=SR48, stationary=True)
    ref = nr.reduce_noise(y, **kw)
    for sizes in ([48000] * (N // 48000) + [N % 48000], _random_blocks(N, 700_000, 1)):
        got = run_stream(nr, y, sizes, **kw)
        assert np.array_equal(got, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["nonstationary_2048", "int16", "offset_rows"])
def test_stream_variants_on_gpu(case):
    import noisereduce_b200 as nr
    N = 1_500_000
    y = _cfg2_signal(3, N + 1, seed=2)
    kw = dict(sr=SR48, stationary=True)
    if case == "nonstationary_2048":
        y = y[:, :N]
        kw = dict(sr=SR48, stationary=False, n_fft=2048)
    elif case == "int16":
        y = np.round(y[:, :N] * 30000).astype(np.int16)
    else:
        y = y[:, 1:]                                             # rows that start 4 bytes past a 16-byte boundary
    ref = nr.reduce_noise(y, **kw)
    got = run_stream(nr, y, _random_blocks(N, 700_000, 5), **kw)
    assert got.dtype == ref.dtype and np.array_equal(got, ref)


@pytest.mark.gpu
def test_stream_device_tensors_on_gpu():
    """torch CUDA tensors through b200gate_stream_push with is_device = 1: the call only enqueues."""
    import torch
    import noisereduce_b200 as nr
    N = 1_300_000
    y = _cfg2_signal(3, N, seed=4)
    kw = dict(sr=SR48, stationary=False)
    ref = nr.reduce_noise(y, **kw)
    g = nr.NoiseReduceStream(n_channels=3, **kw)._gate
    g.stream_begin(np.float32, 3)
    cs, pad = 600000, 30000
    x = torch.from_numpy(y).cuda()
    out = torch.zeros((3, N + cs + pad), dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    R = done = 0
    for n in [0] + _random_blocks(N, 700_000, 9):
        blk, dst = x[:, R:], out[:, done:]
        done += g.stream_push(blk.data_ptr(), n, x.stride(0), True, dst.data_ptr(), out.stride(0), out.shape[1] - done, st)
        R += n
        assert done == expected_emitted(R, cs, pad)
    done += g.stream_finish(out[:, done:].data_ptr(), out.stride(0), out.shape[1] - done, st)
    torch.cuda.synchronize()
    assert done == N
    assert np.array_equal(out[:, :N].cpu().numpy(), ref)
