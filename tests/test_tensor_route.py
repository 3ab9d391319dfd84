"""reduce_noise() / the mirror classes / NoiseReduceStream on torch CUDA tensors: a tensor on the samples' device comes
back, with the same shape, dtype and bits as the numpy route on ``y.cpu().numpy()`` (NaN where it has NaN).

On the CPU simulator (tests/cusim) the library's "device" pointers are host pointers; a simulator library with
``simulated_device`` set sends CPU tensors down the device route, so every step of it -- the conversion kernels
included -- runs here.  The GPU tests use config 2's geometry on an H100."""
import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from tests.golden.edge_cases import cases, refused
from tests.synth_host import synth_small
from tests.test_stream import expected_emitted, schedules

SR = 16000
_BITS = {torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}


def assert_same(got, ref):
    """`got` (a tensor) equals the numpy route's `ref`: shape, dtype, every bit outside NaN, and the NaN pattern."""
    assert isinstance(got, torch.Tensor), type(got)
    ref = torch.from_numpy(np.ascontiguousarray(ref))
    got = got.cpu().contiguous()
    assert got.shape == ref.shape and got.dtype == ref.dtype, (got.shape, got.dtype, ref.shape, ref.dtype)
    if got.dtype in _BITS:
        nan = torch.isnan(ref)
        assert torch.equal(torch.isnan(got), nan)
        assert torch.equal(got.view(_BITS[got.dtype])[~nan], ref.view(_BITS[ref.dtype])[~nan])
    else:
        assert torch.equal(got, ref)


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


def _signal(dtype, n, C=2):
    y = synth_small(C=C, n=n)
    if np.dtype(dtype).kind in "iu":
        return np.round(y / np.abs(y).max() * 100 + (128 if np.dtype(dtype).kind == "u" else 0)).astype(dtype)
    return y.astype(dtype)


# ---- the edge cases of the numpy route, replayed through the tensor route ---------------------------------------
@pytest.mark.parametrize("name", sorted(cases()))
def test_edge_cases_on_simulator(sim, name):
    y, kw = cases()[name]
    ref = sim.reduce_noise(y, sr=SR, **kw)
    got = sim.reduce_noise(torch.from_numpy(y), sr=SR, **kw)        # (from_numpy keeps Fortran order and strides)
    assert_same(got, ref)


@pytest.mark.parametrize("name", sorted(refused()))
def test_refused_inputs_on_simulator(sim, name):
    y, kw, exc, _ = refused()[name]
    with pytest.raises(exc):
        sim.reduce_noise(y, sr=SR, **kw)
    with pytest.raises(exc):
        sim.reduce_noise(torch.from_numpy(y), sr=SR, **kw)


def test_other_refusals_on_simulator(sim):
    y = torch.from_numpy(synth_small(C=2, n=4000))
    with pytest.raises(ValueError, match="shape"):
        sim.reduce_noise(y[None], sr=SR)
    with pytest.raises(ValueError, match="real-valued"):
        sim.reduce_noise(y.to(torch.complex64), sr=SR)
    with pytest.raises(TypeError):
        sim.reduce_noise(y.to(torch.bfloat16), sr=SR)


def test_cpu_tensors_keep_the_numpy_route(monkeypatch):
    """With a library that is not the simulator's device stand-in (the product's case), a CPU tensor goes through
    np.asarray and returns a numpy array, as before."""
    from tests.cusim import build_cusim
    monkeypatch.setattr(_cabi, "_LIB", _cabi.GateLibrary(build_cusim.build()))
    import noisereduce_b200 as nr
    y = synth_small(C=2, n=6000)
    got = nr.reduce_noise(torch.from_numpy(y), sr=SR, stationary=True, chunk_size=2500, padding=400)
    assert isinstance(got, np.ndarray)
    assert np.array_equal(got, nr.reduce_noise(y, sr=SR, stationary=True, chunk_size=2500, padding=400))


# ---- gates, geometries, dtypes, layouts -----------------------------------------------------------------------
BASE = dict(sr=SR, chunk_size=2500, padding=400)
GEOMETRIES = {
    "stationary_1024": dict(stationary=True),
    "nonstationary_1024": dict(stationary=False, time_constant_s=0.3),
    "nonstationary_2048": dict(stationary=False, n_fft=2048, time_constant_s=0.3),
    "general_512_400_100": dict(stationary=True, n_fft=512, win_length=400, hop_length=100),
    "general_441": dict(stationary=False, n_fft=441, time_constant_s=0.3),
    "prop_decrease": dict(stationary=True, prop_decrease=0.6),
    "smoothing_off": dict(stationary=False, freq_mask_smooth_hz=None, time_mask_smooth_ms=None, time_constant_s=0.3),
    "unchunked": dict(stationary=True, chunk_size=None),
}


@pytest.mark.parametrize("geo", sorted(GEOMETRIES))
def test_geometries_on_simulator(sim, geo):
    kw = dict(BASE, **GEOMETRIES[geo])
    y = synth_small(C=2, n=7000)
    assert_same(sim.reduce_noise(torch.from_numpy(y), **kw), sim.reduce_noise(y, **kw))
    assert_same(sim.reduce_noise(torch.from_numpy(y[1]), **kw), sim.reduce_noise(y[1], **kw))     # 1-D stays 1-D


DTYPES = ["bool", "int8", "uint8", "int16", "uint16", "int32", "uint32", "int64", "uint64", "float16", "float32",
          "float64"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("stationary", [True, False])
def test_dtypes_on_simulator(sim, dtype, stationary):
    y = synth_small(C=2, n=6000) > 0.05 if dtype == "bool" else _signal(dtype, 6000)
    kw = dict(BASE, stationary=stationary, time_constant_s=0.3)
    assert_same(sim.reduce_noise(torch.from_numpy(y), **kw), sim.reduce_noise(y, **kw))


@pytest.mark.parametrize("layout", ["column_slice", "row_step", "fortran", "transposed_odd_dtype"])
def test_layouts_on_simulator(sim, layout):
    y = synth_small(C=4, n=9000)
    t = torch.from_numpy(y)
    kw = dict(BASE, stationary=True)
    if layout == "column_slice":                 # read in place: row stride 9000, rows 4 bytes past an aligned start
        t, ref_in = t[:, 1:8001], y[:, 1:8001]
    elif layout == "row_step":                   # read in place: every other row
        t, ref_in = t[::2], y[::2]
    elif layout == "fortran":                    # copied to contiguous rows
        t = t.t().contiguous().t()
        ref_in = np.asfortranarray(y)
    else:
        h = y.astype(np.float16)
        t, ref_in = torch.from_numpy(h.T.copy()).t(), np.asfortranarray(h)
    assert_same(sim.reduce_noise(t, **kw), sim.reduce_noise(ref_in, **kw))


def test_channel_adjacent_odd_dtype_clip_is_the_row_major_mean(sim):
    """numpy sums a Fortran-order clip pairwise over its contiguous channel axis; the tensor route sums in channel
    order, i.e. it equals the numpy route on the row-major copy (the contract stated in install_noise_thresholds)."""
    y = (synth_small(C=12, n=6000) * 3).astype(np.float16)
    kw = dict(BASE, stationary=True)
    t = torch.from_numpy(y.T.copy()).t()                             # channels adjacent in memory
    assert_same(sim.reduce_noise(t, **kw), sim.reduce_noise(np.ascontiguousarray(y), **kw))


# ---- y_noise ------------------------------------------------------------------------------------------------
def _noise(C, n, dtype=np.float32, seed=5):
    return (0.05 * np.random.default_rng(seed).standard_normal((C, n))).astype(dtype)


Y_NOISE = {
    "1d": (_noise(1, 3000)[0], True),
    "2d": (_noise(3, 3000), True),
    "longer_than_chunk_clipped": (_noise(2, 6000), True),
    "longer_than_chunk_unclipped": (_noise(2, 6000), False),
    "short_clip": (_noise(2, 900), True),
    "float16": (_noise(3, 4000, np.float16), True),
    "int32": ((_noise(3, 4000) * 30000).astype(np.int32), True),
}


@pytest.mark.parametrize("as_tensor", [False, True])
@pytest.mark.parametrize("case", sorted(Y_NOISE))
def test_y_noise_on_simulator(sim, case, as_tensor):
    yn, clip = Y_NOISE[case]
    y = synth_small(C=2, n=8000)
    kw = dict(BASE, stationary=True, clip_noise_stationary=clip)
    ref = sim.reduce_noise(y, y_noise=yn, **kw)
    got = sim.reduce_noise(torch.from_numpy(y), y_noise=torch.from_numpy(yn) if as_tensor else yn, **kw)
    assert_same(got, ref)


def test_unclipped_self_noise_on_simulator(sim):
    y = synth_small(C=2, n=8000).astype(np.float16)
    kw = dict(BASE, stationary=True, clip_noise_stationary=False)
    assert_same(sim.reduce_noise(torch.from_numpy(y), **kw), sim.reduce_noise(y, **kw))


# ---- the mirror classes -------------------------------------------------------------------------------------
def _classes(nr, y, stationary):
    args = dict(sr=SR, chunk_size=2500, padding=400, n_fft=1024, win_length=None, hop_length=None,
                time_constant_s=0.3, freq_mask_smooth_hz=500, time_mask_smooth_ms=50, tmp_folder=None,
                prop_decrease=1.0, use_tqdm=False, n_jobs=1)
    if stationary:
        return nr.spectralgate.SpectralGateStationary(y=y, y_noise=None, n_std_thresh_stationary=1.5, clip_noise_stationary=True,
                                         **args)
    return nr.spectralgate.SpectralGateNonStationary(y=y, thresh_n_mult_nonstationary=2, sigmoid_slope_nonstationary=10, **args)


@pytest.mark.parametrize("dtype", ["float32", "uint8"])
@pytest.mark.parametrize("stationary", [True, False])
def test_get_traces_ranges_on_simulator(sim, stationary, dtype):
    y = _signal(dtype, 9000)
    sg_np, sg_t = _classes(sim, y, stationary), _classes(sim, torch.from_numpy(y), stationary)
    for a, b in [(None, None), (1000, 7000), (2600, 5100), (3000, 4000), (0, 2000), (0, 9000), (5000, 9000)]:
        assert_same(sg_t.get_traces(a, b), sg_np.get_traces(a, b))
    if stationary:
        for attr in ("mean_freq_noise", "std_freq_noise", "noise_thresh"):
            assert isinstance(getattr(sg_t, attr), np.ndarray)
            assert np.array_equal(getattr(sg_t, attr), getattr(sg_np, attr))
        assert np.array_equal(sg_t.y_noise, sg_np.y_noise)


# ---- streams of tensor blocks -------------------------------------------------------------------------------
def run_tensor_stream(nr, y, sizes, **kw):
    s = nr.NoiseReduceStream(n_channels=y.shape[0], **kw)
    outs, R = [], 0
    for n in sizes:
        out = s.push(y[:, R:R + n])
        R += n
        assert isinstance(out, torch.Tensor) and out.device == y.device
        assert s.samples_returned == expected_emitted(R, s.chunk_size, s.padding)
        outs.append(out)
    outs.append(s.finish())
    return torch.cat(outs, dim=1)


STREAMS = {
    "stationary_float32": (dict(stationary=True), np.float32),
    "stationary_float16": (dict(stationary=True), np.float16),
    "nonstationary_int16": (dict(stationary=False, time_constant_s=0.3), np.int16),
    "stationary_uint8": (dict(stationary=True), np.uint8),
    "y_noise_tensor": (dict(stationary=True, y_noise="tensor"), np.float32),
    "y_noise_numpy": (dict(stationary=True, y_noise="numpy"), np.float32),
}


@pytest.mark.parametrize("case", sorted(STREAMS))
def test_tensor_stream_on_simulator(sim, monkeypatch, case):
    monkeypatch.setenv("B200GATE_STREAM_SLICE_CHUNKS", "1")
    extra, dtype = STREAMS[case]
    kw = dict(BASE, **extra)
    noise = _noise(2, 3000)
    if kw.get("y_noise") is not None:
        kw["y_noise"] = torch.from_numpy(noise) if kw["y_noise"] == "tensor" else noise
    y = _signal(dtype, 9000)
    ref = sim.reduce_noise(y, **dict(kw, y_noise=noise if "y_noise" in extra else None))
    for sizes in schedules(9000, 2500, 256).values():
        assert_same(run_tensor_stream(sim, torch.from_numpy(y), sizes, **kw), ref)


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
def test_tensor_stream_results_hold_only_their_samples_on_simulator(sim, dtype):
    """A push that returns nothing returns a tensor without storage, and a returned chunk holds its own columns only,
    not the push's [C, n + chunk_size] output buffer: a caller keeping every result must not keep those buffers."""
    y = torch.from_numpy(_signal(dtype, 9000))
    s = sim.NoiseReduceStream(n_channels=2, **dict(BASE, stationary=False, time_constant_s=0.3))
    es = y.element_size()
    for a, b in [(0, 100), (100, 2000), (2000, 3000), (3000, 3100), (3100, 9000)]:
        out = s.push(y[:, a:b])
        assert out.untyped_storage().nbytes() == out.numel() * es, (a, b, out.shape)
        if out.shape[1] == 0:
            assert out.untyped_storage().nbytes() == 0
    out = s.finish()
    assert out.shape[1] > 0 and out.untyped_storage().nbytes() == out.numel() * es


def test_tensor_stream_flat_and_mixing_errors_on_simulator(sim):
    y = synth_small(C=1, n=6000)[0]
    kw = dict(BASE, stationary=True)
    s = sim.NoiseReduceStream(**kw)
    got = torch.cat([s.push(torch.from_numpy(y[:4000])), s.push(torch.from_numpy(y[4000:])), s.finish()])
    assert_same(got, sim.reduce_noise(y, **kw))
    s = sim.NoiseReduceStream(n_channels=1, **kw)
    s.push(torch.from_numpy(y[None, :100]))
    with pytest.raises(ValueError, match="memory space"):
        s.push(y[None, 100:200])
    with pytest.raises(ValueError, match="dtype"):
        s.push(torch.from_numpy(y[None, 100:200].astype(np.float64)))
    s = sim.NoiseReduceStream(n_channels=1, **kw)
    s.push(y[None, :100])
    with pytest.raises(ValueError, match="memory space"):
        s.push(torch.from_numpy(y[None, 100:200]))


# ---- the conversion kernels ---------------------------------------------------------------------------------
CRAFTED = np.array([np.nan, -np.nan, np.inf, -np.inf, 2.0 ** 31, -2.0 ** 31, 2.0 ** 31 - 0.5, -2.0 ** 31 - 1, 2.0 ** 32,
                    2.0 ** 63, -2.0 ** 63, 2.0 ** 64, 1.5 * 2 ** 63, -1.5, 255.9, 256.0, 65535.5, 65536.0, -0.7, 127.9,
                    128.0, -129.0, 2.0 ** 53, 2.0 ** 53 + 2, 1e300, -1e300, 3e9, -3e9, 0.0, -0.0, 0.5, 1e-8,
                    65519.0, 65520.0, 2.0 ** -25, 3 * 2.0 ** -26, 5.960464477539063e-08, 6.103515625e-05])
# float64 values one float32 rounding away from a float16 tie: rounding through float32 lands on the tie and then on
# the even neighbour; numpy's single rounding does not (1 + 2^-11 + 2^-40 -> 1.001 in numpy, 1.0 through float32)
DOUBLE_ROUNDING = np.array([1 + 2.0 ** -11 + 2.0 ** -40, 1 + 3 * 2.0 ** -11 - 2.0 ** -40, -(1 + 2.0 ** -11 + 2.0 ** -40),
                            2048 + 1 + 2.0 ** -30, 2.0 ** -14 * (1 + 2.0 ** -11 + 2.0 ** -40)])


WIDE_I64 = np.array([2 ** 53 + 1, 2 ** 53 + 3, -(2 ** 53) - 1, 2 ** 63 - 1, -(2 ** 63), 2 ** 62 + 2 ** 9,
                     2 ** 62 + 2 ** 9 + 1, 2 ** 62 + 3 * 2 ** 9, 12345, -7], dtype=np.int64)
WIDE_U64 = np.array([2 ** 53 + 1, 2 ** 64 - 1, 2 ** 63, 2 ** 63 + 2 ** 10, 2 ** 63 + 2 ** 10 + 1, 2 ** 63 + 3 * 2 ** 10,
                     2 ** 63 - 1, 0, 1], dtype=np.uint64)


def convert_cast(lib, x64, np_dtype, device):
    """x64 (float64 numpy [C, N]) -> np_dtype through b200gate_convert on `device` tensors."""
    src = torch.from_numpy(x64).to(device)
    tdt = torch.from_numpy(np.empty(0, np_dtype)).dtype
    dst = torch.empty(src.shape, dtype=tdt, device=device)
    st = torch.cuda.current_stream(device).cuda_stream if src.is_cuda else None
    _cabi.convert(lib, _cabi.CONVERT_CAST, src.data_ptr(), np.float64, src.shape[1], dst.data_ptr(), np_dtype,
                  src.shape[1], src.shape[0], src.shape[1], st)
    back = torch.empty(src.shape, dtype=torch.float64, device=device)
    _cabi.convert(lib, _cabi.CONVERT_CAST, dst.data_ptr(), np_dtype, src.shape[1], back.data_ptr(), np.float64,
                  src.shape[1], src.shape[0], src.shape[1], st)
    return dst.cpu().numpy(), back.cpu().numpy()


def check_conversions(lib, device):
    x = np.stack([CRAFTED, CRAFTED[::-1]])
    for name in DTYPES:
        dt = np.dtype(name)
        with np.errstate(all="ignore"):
            want = x.astype(dt)
        got, back = convert_cast(lib, x, dt, device)
        assert got.dtype == dt
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), name          # every bit, NaN included
        with np.errstate(all="ignore"):
            assert np.array_equal(back.view(np.uint8), want.astype(np.float64).view(np.uint8)), name
    # 64-bit integers beyond 2^53 round to nearest even on the way to float64, as numpy's cast does
    for dt, vals in ((np.int64, WIDE_I64), (np.uint64, WIDE_U64)):
        src = torch.from_numpy(vals[None, :]).to(device)
        dst = torch.empty(src.shape, dtype=torch.float64, device=device)
        st = torch.cuda.current_stream(device).cuda_stream if src.is_cuda else None
        _cabi.convert(lib, _cabi.CONVERT_CAST, src.data_ptr(), dt, vals.size, dst.data_ptr(), np.float64, vals.size, 1,
                      vals.size, st)
        want = vals.astype(np.float64)
        assert np.array_equal(dst.cpu().numpy()[0], want), dt
        with np.errstate(all="ignore"):
            assert not np.array_equal(want.astype(dt), vals)      # some of them do round
    x = DOUBLE_ROUNDING[None, :]
    got, _ = convert_cast(lib, x, np.float16, device)
    assert np.array_equal(got.view(np.uint16), x.astype(np.float16).view(np.uint16))
    assert not np.array_equal(x.astype(np.float32).astype(np.float16), x.astype(np.float16))   # the vector bites


def check_channel_mean(lib, device):
    for name in DTYPES:
        dt = np.dtype(name)
        y = _signal(dt, 3000, C=5) if name != "bool" else synth_small(C=5, n=3000) > 0
        if name == "float16":
            y = (synth_small(C=5, n=3000) * 7).astype(np.float16)
        t = torch.from_numpy(y).to(device)
        out = torch.empty(3000, dtype=torch.float64, device=device)
        st = torch.cuda.current_stream(device).cuda_stream if t.is_cuda else None
        _cabi.convert(lib, _cabi.CONVERT_CHANNEL_MEAN, t.data_ptr(), dt, 3000, out.data_ptr(), np.float64, 0, 5, 3000, st)
        want = np.mean(y, axis=0).astype(np.float64)
        assert np.array_equal(out.cpu().numpy(), want), name


def test_conversion_kernels_on_simulator(simlib):
    check_conversions(simlib, "cpu")


def test_channel_mean_kernel_on_simulator(simlib):
    check_channel_mean(simlib, "cpu")


def test_convert_rejects_bad_arguments_on_simulator(simlib):
    x = torch.zeros((2, 8), dtype=torch.float64)
    with pytest.raises(_cabi.GateError, match="float64"):             # neither side float64
        _cabi.convert(simlib, _cabi.CONVERT_CAST, x.data_ptr(), np.float32, 8, x.data_ptr(), np.int16, 8, 2, 8)
    with pytest.raises(_cabi.GateError):                              # row stride below N
        _cabi.convert(simlib, _cabi.CONVERT_CAST, x.data_ptr(), np.float64, 4, x.data_ptr(), np.float32, 8, 2, 8)
    with pytest.raises(TypeError):
        _cabi.format_code(np.complex64)


# ---- H100 -------------------------------------------------------------------------------------------------------
SR48 = 48000


def _cfg2(C, N, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(N) / SR48
    tone = 0.3 * np.sin(2 * np.pi * 440.0 * t) * (np.sin(2 * np.pi * 0.5 * t) > 0)
    return (tone[None, :] + 0.05 * rng.standard_normal((C, N))).astype(np.float32)


GPU_CASES = {
    "float32_stationary": (np.float32, dict(stationary=True)),
    "float32_nonstationary_2048": (np.float32, dict(stationary=False, n_fft=2048)),
    "int16_stationary": (np.int16, dict(stationary=True)),
    "float16_stationary": (np.float16, dict(stationary=True)),
    "uint8_nonstationary": (np.uint8, dict(stationary=False)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GPU_CASES))
def test_config2_geometry_on_gpu(case):
    import noisereduce_b200 as nr
    dtype, kw = GPU_CASES[case]
    y = _cfg2(8, 1_300_000)
    if dtype == np.int16:
        y = np.round(y * 30000).astype(np.int16)
    elif dtype == np.uint8:
        y = np.round(y * 100 + 128).astype(np.uint8)
    else:
        y = y.astype(dtype)
    t = torch.from_numpy(y).cuda()
    got = nr.reduce_noise(t, sr=SR48, **kw)
    assert got.is_cuda and got.device == t.device
    assert_same(got, nr.reduce_noise(t.cpu().numpy(), sr=SR48, **kw))


@pytest.mark.gpu
def test_tensor_stream_config2_on_gpu():
    import noisereduce_b200 as nr
    from tests.test_stream import _random_blocks
    N = 1_300_000
    y = torch.from_numpy(_cfg2(4, N, seed=3)).cuda()
    kw = dict(sr=SR48, stationary=True)
    ref = nr.reduce_noise(y.cpu().numpy(), **kw)
    assert_same(run_tensor_stream(nr, y, _random_blocks(N, 700_000, 11), **kw), ref)


@pytest.mark.gpu
def test_tensor_stream_with_host_y_noise_on_gpu():
    """Host y_noise: the thresholds are computed at construction; the handle moves to the blocks' device with them."""
    import noisereduce_b200 as nr
    from tests.test_stream import _random_blocks
    N = 1_300_000
    y = torch.from_numpy(_cfg2(2, N, seed=5)).cuda()
    noise = _cfg2(2, 200_000, seed=6) * np.float32(0.2)
    kw = dict(sr=SR48, stationary=True, y_noise=noise)
    ref = nr.reduce_noise(y.cpu().numpy(), **kw)
    assert_same(run_tensor_stream(nr, y, _random_blocks(N, 500_000, 2), **kw), ref)
    # a stream built before torch initialised CUDA does not know its handle's device: the first CUDA block remakes
    # the handle there, with the thresholds copied over
    s = nr.NoiseReduceStream(n_channels=2, **kw)
    s._gate_device = None
    outs = [s.push(y[:, :700_000]), s.push(y[:, 700_000:]), s.finish()]
    assert_same(torch.cat(outs, dim=1), ref)


@pytest.mark.gpu
def test_runs_on_the_current_stream_on_gpu():
    """Work queued on a side stream before the call (a long sleep, then an in-place write of the input) must be
    seen by reduce_noise() called inside that stream's context."""
    import noisereduce_b200 as nr
    y_np = _cfg2(2, 700_000, seed=9)
    x = torch.zeros(y_np.shape, dtype=torch.float32, device="cuda")
    src = torch.from_numpy(y_np).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                 # ~0.1 s of spinning on the side stream
        x.copy_(src)
        got = nr.reduce_noise(x, sr=SR48, stationary=False)
    side.synchronize()
    assert_same(got, nr.reduce_noise(y_np, sr=SR48, stationary=False))
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        x.mul_(0.5)
        got = nr.reduce_noise(x, sr=SR48, stationary=True)
    side.synchronize()
    assert_same(got, nr.reduce_noise(y_np * np.float32(0.5), sr=SR48, stationary=True))


@pytest.mark.gpu
def test_conversion_kernels_on_gpu(capsys):
    lib = _cabi.library()
    check_conversions(lib, "cuda")
    check_channel_mean(lib, "cuda")
    # record torch's own CUDA cast of the double-rounding vector (the reason the route has its own kernels)
    x = torch.from_numpy(DOUBLE_ROUNDING).cuda()
    torch_cast = x.to(torch.float16).cpu().numpy()
    with capsys.disabled():
        print("\nfloat64 -> float16 of", DOUBLE_ROUNDING.tolist())
        print("  numpy astype      :", DOUBLE_ROUNDING.astype(np.float16).tolist())
        print("  torch CUDA .to()  :", torch_cast.tolist())
        with np.errstate(all="ignore"):
            v = torch.from_numpy(CRAFTED).cuda()
            for dt in (torch.uint8, torch.int16, torch.int32):
                print(f"  torch CUDA {dt} of crafted:", v.to(dt).cpu().tolist())
