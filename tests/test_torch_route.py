"""reduce_noise(use_torch=True): the chunk grid as one library call on the chunked torch surface, CUDA tensors in and out,
and NoiseReduceStream(use_torch=True).

The yardstick is the reference's own loop, kept as StreamedTorchGate._get_traces_per_chunk(): one TorchGate call per
padded float64 chunk.  get_traces() must equal it in shape, dtype and every bit, and refuse what it refuses with the same
exception types.  On the CPU simulator (tests/cusim) a library with ``simulated_device`` set sends CPU tensors down the
device route.  tests/golden/torch_route.npz holds the unmodified reference's reduce_noise(use_torch=True, device="cpu")."""
import os

import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from noisereduce_b200.spectralgate.streamed_torch_gate import StreamedTorchGate
from tests.golden.make_golden_torch_route import SR as GOLDEN_SR, torch_route_cases

SR = 16000
HERE = os.path.dirname(os.path.abspath(__file__))
BASE = dict(chunk_size=3000, padding=1100, time_constant_s=0.2)


def _signal(C=2, n=9000, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    tone = np.sin(2 * np.pi * 440 * t)[None, :] * (t[None, :] > 0.12 * np.arange(1, C + 1)[:, None])
    return (0.4 * tone + 0.05 * rng.standard_normal((C, n))).astype(np.float32)


def _same(a, b):
    assert type(a) is type(b) and a.shape == b.shape and a.dtype == b.dtype
    a, b = (a.cpu().numpy(), b.cpu().numpy()) if isinstance(a, torch.Tensor) else (a, b)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


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


def _gate(y, lib, **kw):
    return StreamedTorchGate(y=y, sr=SR, **dict(BASE, **kw), _lib=lib)


def _outcome(f):
    try:
        return f()
    except Exception as e:          # noqa: BLE001 -- the exception type is the result
        return e


def _check_one_call(sg, *rng):
    want, got = _outcome(lambda: sg._get_traces_per_chunk(*rng)), _outcome(lambda: sg.get_traces(*rng))
    if isinstance(want, Exception):
        assert type(got) is type(want), (want, got)
    else:
        assert not isinstance(got, Exception), got
        _same(got, want)


Y = _signal()
CASES = {
    "stationary": dict(stationary=True),
    "nonstationary": dict(stationary=False, thresh_n_mult_nonstationary=1.5, sigmoid_slope_nonstationary=8),
    "noise_1d": dict(stationary=True, y_noise=Y[0, :4000]),
    "noise_rows": dict(stationary=True, y_noise=Y[:, 2000:7000]),
    "noise_longer_clipped": dict(stationary=True, y_noise=np.concatenate([Y, Y], 1)),
    "noise_longer_unclipped": dict(stationary=True, y_noise=np.concatenate([Y, Y], 1), clip_noise_stationary=False),
    "nonstationary_noise": dict(stationary=False, y_noise=Y[:, :5000]),
    "nfft2048": dict(stationary=True, n_fft=2048, chunk_size=5000),
    "nfft512_400_100": dict(stationary=False, n_fft=512, win_length=400, hop_length=100),
    "bluestein441": dict(stationary=True, n_fft=441),
    "chunk_none": dict(stationary=False, chunk_size=None),
    "single_chunk": dict(stationary=True, chunk_size=9000),
    "ragged_last": dict(stationary=True, chunk_size=4000),
    "padding0": dict(stationary=False, padding=0, chunk_size=3072),
    "len_not_hop_multiple": dict(stationary=True, padding=1001, chunk_size=2999),
    "prop_decrease": dict(stationary=True, prop_decrease=0.6),
    "smoothing_off": dict(stationary=False, freq_mask_smooth_hz=None, time_mask_smooth_ms=None),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_one_call_equals_loop(simlib, case):
    _check_one_call(_gate(Y, simlib, **CASES[case]))


@pytest.mark.parametrize("dtype", [np.float32, np.int16, np.float64, np.float16, np.int32])
def test_one_call_dtypes(simlib, dtype):
    y = (Y * 20000).astype(dtype) if np.dtype(dtype).kind == "i" else Y.astype(dtype)
    for stationary in (True, False):
        _check_one_call(_gate(y, simlib, stationary=stationary))


def test_flat_and_sub_ranges(simlib):
    _check_one_call(_gate(Y[0], simlib, stationary=True))
    sg = _gate(Y, simlib, stationary=False)
    for rng in ((500, 8200), (3000, 6001), (100, 2900), (0, 3000)):   # the chunked branch, then the single-chunk branch
        _check_one_call(sg, *rng)


def test_refused_inputs(simlib):
    """The loop's refusals, with its exception types: a padded chunk shorter than 2 win_length (TorchGate's Exception),
    a short or 3-D y_noise, a torch output shorter than padding + chunk_size (numpy's broadcast ValueError), an xn whose
    row count is neither 1 nor C (the library's error)."""
    for kw in (dict(chunk_size=600, padding=100), dict(y_noise=Y[:, :1000]), dict(y_noise=Y[None]),
               dict(padding=0, chunk_size=3001), dict(y_noise=np.concatenate([Y, Y])[:3])):
        sg = _gate(Y, simlib, stationary=True, **kw)
        want = _outcome(sg._get_traces_per_chunk)
        assert isinstance(want, Exception), kw
        _check_one_call(sg)
    with pytest.raises(ValueError):           # a short single chunk: the loop returns fewer samples, so does one call
        _gate(Y, simlib, stationary=False, padding=0, chunk_size=3001).get_traces(0, 10 ** 6)
    short = _gate(Y[:, :2900], simlib, stationary=False, padding=0, chunk_size=3001)
    _check_one_call(short)
    assert short.get_traces().shape[-1] < 2900


# ---- the device route on the simulator: CPU tensors through kernel_rows / b200gate_convert ------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.int16, torch.float16, torch.float64])
def test_device_route_matches_numpy_route(sim, dtype):
    y = torch.from_numpy(Y * (20000 if dtype == torch.int16 else 1)).to(dtype)
    for stationary in (True, False):
        kw = dict(BASE, stationary=stationary, use_torch=True)
        got = sim.reduce_noise(y, sr=SR, **kw)
        want = sim.reduce_noise(y.numpy(), sr=SR, **kw)
        assert isinstance(got, torch.Tensor) and isinstance(want, np.ndarray)
        _same(got.numpy(), want)
    wide = torch.zeros(2, 9003, dtype=dtype)                 # rows offset from a 16-byte boundary, read in place
    wide[:, 3:] = y
    got = sim.reduce_noise(wide[:, 3:], sr=SR, **dict(BASE, stationary=True, use_torch=True))
    _same(got.numpy(), sim.reduce_noise(y.numpy(), sr=SR, **dict(BASE, stationary=True, use_torch=True)))


def test_device_route_noise_and_device_args(sim):
    y = torch.from_numpy(Y)
    want = sim.reduce_noise(Y, sr=SR, y_noise=Y[:, :5000], stationary=True, use_torch=True, **BASE)
    for yn in (Y[:, :5000], torch.from_numpy(Y[:, :5000])):
        got = sim.reduce_noise(y, sr=SR, y_noise=yn, stationary=True, use_torch=True, **BASE)
        _same(got.numpy(), want)
    with pytest.raises(ValueError):
        sim.reduce_noise(y, sr=SR, use_torch=True, device="cuda:1", **BASE)
    with pytest.raises(ValueError, match="n_jobs"):
        sim.reduce_noise(y, sr=SR, use_torch=True, n_jobs=2, **BASE)


# ---- the stream ---------------------------------------------------------------------------------------------------
def _schedules(n):
    rng = np.random.default_rng(1)
    yield [n]
    yield [977] * (n // 977) + [n % 977]
    cuts = np.sort(rng.integers(0, n, 6))
    yield list(np.diff(np.concatenate([[0], cuts, [n]])))


def _stream(nr, y, schedule, sr=SR, **kw):
    s = nr.NoiseReduceStream(sr=sr, n_channels=y.shape[0], use_torch=True, **kw)
    outs, pos = [], 0
    for m in schedule:
        out = s.push(y[:, pos:pos + m])
        pos += m
        assert s.samples_returned == s.emitted() and out.shape[-1] == s.emitted() - sum(o.shape[-1] for o in outs)
        outs.append(out)
    outs.append(s.finish())
    cat = torch.cat if isinstance(y, torch.Tensor) else np.concatenate
    return cat(outs, -1), s


@pytest.mark.parametrize("case", ["stationary", "nonstationary", "noise_rows", "noise_longer_clipped",
                                  "noise_longer_unclipped", "bluestein441"])
def test_stream_equals_offline(sim, monkeypatch, case):
    monkeypatch.setenv("B200GATE_STREAM_SLICE_CHUNKS", "1")
    kw = dict(BASE, **CASES[case])
    want = sim.reduce_noise(Y, sr=SR, use_torch=True, **kw)
    for schedule in _schedules(Y.shape[1]):
        got, _ = _stream(sim, Y, schedule, **kw)
        _same(got, want)


def test_stream_noise_hold_back_and_short_recordings(sim):
    kw = dict(BASE, stationary=True, y_noise=Y[:, :7000])
    s = sim.NoiseReduceStream(sr=SR, n_channels=2, use_torch=True, **kw)
    assert s.push(Y[:, :6999]).shape == (2, 0) and s.emitted() == 0           # 6999 < len(y_noise): held back
    assert s.push(Y[:, 6999:7000]).shape == (2, s.emitted()) and s.emitted() == 3000
    got = np.concatenate([s.push(Y[:, 7000:]), s.finish()], 1)
    # recordings of at most chunk_size samples come back whole from finish(), the y_noise clip included
    for n in (2500, 3000):
        want = sim.reduce_noise(Y[:, :n], sr=SR, use_torch=True, **kw)
        got, s = _stream(sim, Y[:, :n], [n // 2, n - n // 2], **kw)
        _same(got, want)
    # a short recording with a longer y_noise, streamed on the device route
    y = torch.from_numpy(Y[:, :2600])
    got, _ = _stream(sim, y, [1000, 1600], **kw)
    _same(got.numpy(), sim.reduce_noise(Y[:, :2600], sr=SR, use_torch=True, **kw))


def test_stream_device_blocks(sim, monkeypatch):
    monkeypatch.setenv("B200GATE_STREAM_SLICE_CHUNKS", "1")
    kw = dict(BASE, stationary=False)
    got, _ = _stream(sim, torch.from_numpy(Y).to(torch.float16), [2000, 4500, 2500], **kw)
    _same(got.numpy(), sim.reduce_noise(Y.astype(np.float16), sr=SR, use_torch=True, **kw))
    with pytest.raises(ValueError):
        sim.NoiseReduceStream(sr=SR, n_channels=2, use_torch=True, device="cpu", **kw)


# ---- C ABI -----------------------------------------------------------------------------------------------------------
def test_cabi_chunked_torch_surface(simlib):
    base = dict(lib=simlib, surface=_cabi.SURFACE_TORCH_CHUNKED, stationary=1, n_fft=1024, win_length=1024,
                hop_length=256, std_ddof=1, chunk_size=3000, padding=1100, sr=float(SR), prop_decrease=1.0,
                n_std_thresh=1.5, top_db=40.0)
    with pytest.raises(_cabi.GateError, match="prop_decrease"):
        _cabi.Gate(**dict(base, prop_decrease=1.5))
    with pytest.raises(_cabi.GateError, match="unknown surface"):
        _cabi.Gate(**dict(base, surface=3))
    g = _cabi.Gate(**base)
    x = np.ascontiguousarray(Y)
    out = np.zeros((2, 9000), np.float32)
    # streams: no thresholds needed on this surface (each unit takes its own statistics)
    g.stream_begin(np.float32, 2)
    assert g.stream_push(x.ctypes.data, 9000, 9000, False, out.ctypes.data, 12000, 12000) == 6000
    with pytest.raises(_cabi.GateError, match="out_capacity"):
        g.stream_finish(out.ctypes.data, 100, 100)                  # refused before anything is written
    assert g.stream_finish(out.ctypes.data, 9000, 9000) == 3000
    with pytest.raises(_cabi.GateError, match="no open stream"):
        g.stream_finish(out.ctypes.data, 9000, 9000)
    # a padded chunk shorter than 2 win_length, and a torch output shorter than padding + chunk_size
    for kw in (dict(chunk_size=500, padding=100), dict(chunk_size=3001, padding=0)):
        g2 = _cabi.Gate(**dict(base, **kw))
        with pytest.raises(_cabi.GateError, match="bigger than|broadcast"):
            g2.run_host(x)
    # the whole-row torch surface still refuses streams
    g3 = _cabi.Gate(**dict(base, surface=_cabi.SURFACE_TORCH, chunk_size=0, padding=0))
    with pytest.raises(_cabi.GateError, match="streaming"):
        g3.stream_begin(np.float32, 2)


# ---- the reference's own route -------------------------------------------------------------------------------------------
def _golden_check(nr, to_input=lambda a: a):
    gold = np.load(os.path.join(HERE, "golden", "torch_route.npz"))
    for name, (y, y_noise, kw) in torch_route_cases().items():
        got = nr.reduce_noise(to_input(y), sr=GOLDEN_SR, y_noise=y_noise, use_torch=True, **kw)
        got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
        want = gold[name]
        assert got.shape == want.shape and got.dtype == want.dtype, name
        assert np.array_equal(np.isnan(got), np.isnan(want)), name
        g, w = got.astype(np.float64), want.astype(np.float64)
        ok = ~np.isnan(w)
        assert np.abs(g[ok] - w[ok]).max() / np.abs(w[ok]).max() < 5e-7, name


def test_golden_reference_route(sim):
    _golden_check(sim)


# ---- H100 ----------------------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


@gpu
def test_gpu_one_call_equals_loop_config2_slice():
    """Config 2's geometry (48 kHz, chunk 600000, padding 30000) on an 8 ch x 2 min slice."""
    rng = np.random.default_rng(7)
    n = 48000 * 120
    t = np.arange(n) / 48000
    y = (0.3 * np.sin(2 * np.pi * 440 * t)[None, :] * (rng.random((8, 1)) + 0.2)
         + 0.05 * rng.standard_normal((8, n))).astype(np.float32)
    for stationary in (True, False):
        sg = StreamedTorchGate(y=y, sr=48000, stationary=stationary)
        _same(sg.get_traces(), sg._get_traces_per_chunk())


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.int16, torch.float16])
def test_gpu_cuda_tensor_route(dtype):
    import noisereduce_b200 as nr
    rng = np.random.default_rng(3)
    y = (0.3 * rng.standard_normal((4, 48000 * 20))).astype(np.float32)
    yt = torch.from_numpy(y * (20000 if dtype == torch.int16 else 1)).to(dtype)
    for stationary in (True, False):
        want = nr.reduce_noise(yt.numpy(), sr=48000, stationary=stationary, use_torch=True)
        got = nr.reduce_noise(yt.cuda(), sr=48000, stationary=stationary, use_torch=True)
        assert got.is_cuda
        _same(got.cpu().numpy(), want)
        wide = torch.zeros(4, yt.shape[1] + 3, dtype=dtype, device="cuda")
        wide[:, 3:] = yt.cuda()
        _same(nr.reduce_noise(wide[:, 3:], sr=48000, stationary=stationary, use_torch=True).cpu().numpy(), want)


@gpu
def test_gpu_cuda_stream_equals_offline():
    import noisereduce_b200 as nr
    rng = np.random.default_rng(5)
    y = torch.from_numpy((0.3 * rng.standard_normal((4, 48000 * 40))).astype(np.float32)).cuda()
    for stationary in (True, False):
        want = nr.reduce_noise(y, sr=48000, stationary=stationary, use_torch=True)
        got, _ = _stream(nr, y, [48000] * 40, sr=48000, stationary=stationary)
        _same(got.cpu().numpy(), want.cpu().numpy())


@gpu
def test_gpu_golden_reference_route():
    import noisereduce_b200 as nr
    _golden_check(nr)
    _golden_check(nr, lambda a: torch.from_numpy(a).cuda())
