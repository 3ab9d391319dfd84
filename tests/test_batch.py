"""reduce_noise_batch(): a list of recordings of different lengths through one handle and one b200gate_run_rows call.

The contract is bit-identity: outs[i] equals reduce_noise(ys[i], sr, ...) in every bit (NaN pattern included), whatever
else is in the list.  On the CPU simulator (tests/cusim) the .cu sources run on the host, and CPU tensors take the
device route; the gpu-marked tests repeat the comparison on the nvcc build at the sizes the feature is for."""
import ctypes
import math

import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from tests.synth_host import synth_small

SR = 16000
CS, PAD = 5000, 600          # small chunks so that the simulator stays fast
N_FFT, HOP = 1024, 256


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


def clip(n, C=None, seed=0, dtype=np.float32):
    y = synth_small(C=C or 1, n=n, seed=seed) if n >= 64 else \
        (0.1 * np.random.default_rng(seed).standard_normal((C or 1, n))).astype(np.float32)
    y = y if C else y[0]
    if dtype == np.int16:
        return np.round(y * 20000).astype(np.int16)
    return y.astype(dtype)


NOISE = clip(4000, seed=99) * 0.3
# every branch of the chunk grid: shorter than n_fft, between n_fft and 2 n_fft, off the hop grid, exactly chunk_size,
# chunk_size + 1, several chunks with a ragged last one
LENGTHS = (700, 1500, 2077, CS, CS + 1, 2 * CS + 1234, 256)


def loop(nr, ys, **kw):
    return [nr.reduce_noise(y, SR, **kw) for y in ys]


def assert_same(outs, refs, ys):
    assert len(outs) == len(refs) == len(ys)
    for i, (o, r, y) in enumerate(zip(outs, refs, ys)):
        assert type(o) is type(r) and o.shape == r.shape == y.shape and o.dtype == r.dtype == y.dtype, i
        if isinstance(o, torch.Tensor):
            assert o.device == y.device and torch.equal(torch.nan_to_num(o, nan=7.0), torch.nan_to_num(r, nan=7.0)), i
        else:
            assert np.array_equal(o, r, equal_nan=True), i


def gate_kw(stationary):
    return dict(stationary=True, y_noise=NOISE, chunk_size=CS, padding=PAD) if stationary else \
        dict(chunk_size=CS, padding=PAD)


@pytest.mark.parametrize("stationary", [False, True], ids=["nonstationary", "stationary"])
@pytest.mark.parametrize("padding", [0, 100, PAD, CS + 500])
def test_lengths_and_paddings(sim, stationary, padding):
    ys = [clip(n, seed=i) for i, n in enumerate(LENGTHS)]
    if padding == 0:
        ys = [y for y in ys if y.shape[-1] >= 1500]       # (shorter single chunks have no frame reduce_noise() can use)
    kw = dict(gate_kw(stationary), padding=padding)
    outs = sim.reduce_noise_batch(ys, SR, **kw)
    assert_same(outs, loop(sim, ys, **kw), ys)
    assert any(np.abs(o).max() > 0 for o in outs)


@pytest.mark.parametrize("stationary", [False, True], ids=["nonstationary", "stationary"])
@pytest.mark.parametrize("dtype", [np.float32, np.int16, np.float64])
def test_layouts_and_dtypes_numpy(sim, stationary, dtype):
    ys = [clip(3000, seed=1, dtype=dtype), clip(CS + 700, C=3, seed=2, dtype=dtype),
          np.asfortranarray(clip(2100, C=2, seed=3, dtype=dtype)), clip(1300, C=1, seed=4, dtype=dtype)]
    kw = gate_kw(stationary)
    assert_same(sim.reduce_noise_batch(ys, SR, **kw), loop(sim, ys, **kw), ys)


@pytest.mark.parametrize("stationary", [False, True], ids=["nonstationary", "stationary"])
def test_tensor_route_strided_rows(sim, stationary):
    big = torch.from_numpy(clip(CS + 900, C=5, seed=7))
    ys = [big[::2, 3:],                                   # row stride 2 N, rows starting off a 16-byte boundary
          big[1, 100:3000],                               # 1-D view at an offset
          torch.from_numpy(clip(2 * CS + 10, C=3, seed=8))[:, ::2],     # sample stride 2: copied to contiguous rows
          torch.from_numpy(clip(900, seed=9))]
    kw = gate_kw(stationary)
    if stationary:
        kw["y_noise"] = torch.from_numpy(NOISE)
    assert_same(sim.reduce_noise_batch(ys, SR, **kw), loop(sim, ys, **kw), ys)


@pytest.mark.parametrize("stationary", [False, True], ids=["nonstationary", "stationary"])
@pytest.mark.parametrize("smooth", [dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None),
                                    dict(freq_mask_smooth_hz=450, time_mask_smooth_ms=70),      # nf = 14: the tap loops
                                    dict(prop_decrease=0.6)], ids=["none", "nf14", "blend"])
def test_smoothing_settings(sim, stationary, smooth):
    ys = [clip(n, seed=i) for i, n in enumerate((1800, CS + 300, 3333))]
    kw = dict(gate_kw(stationary), **smooth)
    assert_same(sim.reduce_noise_batch(ys, SR, **kw), loop(sim, ys, **kw), ys)


def test_follower_regenerates_and_stores_in_one_batch(sim):
    """k_iir_sigmoid's two variants round differently: each unit takes the one its own frame count selects."""
    tc = 0.05
    tfr = tc * SR / HOP
    b = (math.sqrt(1.0 + 4.0 * tfr * tfr) - 1.0) / (2.0 * tfr * tfr)
    t_switch = int(math.floor((29.0 * math.log(2.0) - math.log(2.5) + math.log(b)) / (2.0 * -math.log1p(-b))))
    frames = [t_switch - 6, t_switch, t_switch + 1, t_switch + 9]
    assert frames[0] > 8
    ys = []
    for i, T in enumerate(frames):                       # single padded chunks: T = (n + 2 pad) // hop + 1
        n = (T - 1) * HOP - 2 * PAD + 17
        y = clip(n, seed=20 + i)
        y[: n // 2] *= 1e-4                              # quiet, then loud: where the two variants differ
        ys.append(y)
    kw = dict(chunk_size=4 * CS, padding=PAD, time_constant_s=tc)
    outs = sim.reduce_noise_batch(ys, SR, **kw)
    assert_same(outs, loop(sim, ys, **kw), ys)
    assert_same(sim.reduce_noise_batch(ys[::-1], SR, **kw), outs[::-1], ys[::-1])


def _rows_call(lib, params, ys, y_noise=None):
    """b200gate_run_rows on host rows packed in one buffer; returns (outputs, stats)."""
    gate = _cabi.Gate(lib=lib, **params)
    if y_noise is not None:
        gate.noise_stats_host(y_noise)
    total = sum(y.size for y in ys)
    buf = np.zeros(2 * total, ys[0].dtype)
    rows, off = [], 0
    for y in ys:
        buf[off: off + y.size] = y
        rows.append((buf.ctypes.data + off * y.itemsize, buf.ctypes.data + (total + off) * y.itemsize, y.size, 1))
        off += y.size
    gate.run_rows(rows, ys[0].dtype, False)
    st = gate.stats()
    gate.close()
    outs, off = [], total
    for y in ys:
        outs.append(buf[off: off + y.size].copy())
        off += y.size
    return outs, st


def stationary_params(**kw):
    p = dict(surface=_cabi.SURFACE_NUMPY, stationary=1, n_fft=N_FFT, win_length=N_FFT, hop_length=HOP, n_grad_freq=15,
             n_grad_time=3, chunk_size=CS, padding=PAD, sr=float(SR), prop_decrease=1.0, top_db=80.0, std_ddof=0,
             n_std_thresh=1.5, clip_noise=1)
    p.update(kw)
    return p


def test_stationary_exactness_machinery_per_unit(sim, simlib):
    """A loud tone (its top_db floor lifts rows: the row-maximum fallback runs for the batch) next to quiet items and
    an all-zero one; then a wide guard band, so that many bins go through the FP64 re-decision."""
    n = 6000
    t = np.arange(n) / SR
    rng = np.random.default_rng(5)
    tone = (1e-5 * rng.standard_normal(n) + 0.9 * np.sin(2 * np.pi * 1000 * t)).astype(np.float32)
    quiet = (1e-5 * rng.standard_normal(4000)).astype(np.float32)
    ys = [quiet[:2500], tone, np.zeros(3000, np.float32), quiet[500:3100]]
    kw = dict(stationary=True, y_noise=quiet, chunk_size=CS, padding=PAD)
    assert_same(sim.reduce_noise_batch(ys, SR, **kw), loop(sim, ys, **kw), ys)

    outs, st = _rows_call(simlib, stationary_params(), ys, quiet[None, :])
    for o, y in zip(outs, ys):
        g = _cabi.Gate(lib=simlib, **stationary_params())
        g.noise_stats_host(quiet[None, :])
        assert np.array_equal(o, g.run_host(y[None, :])[0], equal_nan=True)
        g.close()
    units = [1 if y.size <= CS else (y.size - 1) // CS + 1 for y in ys]
    frames = sum(((min(y.size, CS) + 2 * PAD) // HOP + 1) * u for y, u in zip(ys, units))
    assert st["units"] == sum(units) and st["frames"] == frames
    assert st["rowfloor_flags"] > 0 and st["bins_unresolved"] == 0

    ys = [clip(n_, seed=i) for i, n_ in enumerate((2000, CS + 200))]
    wide = stationary_params(debug_guard_scale=100000)
    outs, st = _rows_call(simlib, wide, ys, NOISE[None, :])
    assert st["bins_rechecked_fp64"] > 100 and st["bins_unresolved"] == 0
    rechecked = 0
    for o, y in zip(outs, ys):
        g = _cabi.Gate(lib=simlib, **wide)
        g.noise_stats_host(NOISE[None, :])
        assert np.array_equal(o, g.run_host(y[None, :])[0])
        rechecked += g.stats()["bins_rechecked_fp64"]
        g.close()
    assert st["bins_rechecked_fp64"] == rechecked


@pytest.mark.parametrize("stationary", [False, True], ids=["nonstationary", "stationary"])
def test_workspace_batches_order_and_single_item(sim, simlib, stationary, monkeypatch):
    ys = [clip(n, seed=i) for i, n in enumerate((2 * CS + 100, 1200, 3100, CS))]
    kw = gate_kw(stationary)
    outs = sim.reduce_noise_batch(ys, SR, **kw)
    perm = [2, 0, 3, 1]
    assert_same(sim.reduce_noise_batch([ys[i] for i in perm], SR, **kw), [outs[i] for i in perm], [ys[i] for i in perm])
    assert_same(sim.reduce_noise_batch(ys[:1], SR, **kw), loop(sim, ys[:1], **kw), ys[:1])
    # a workspace limit of about two units: several workspace batches, same bits
    real_gate = _cabi.Gate
    seen = []

    def small_workspace(**params):
        g = real_gate(workspace_limit_bytes=2.2 * 27 * (1024 * 8 + 2 * 544 * 4 * 2), **params)
        seen.append(g)
        return g

    monkeypatch.setattr(_cabi, "Gate", small_workspace)
    stats = []
    monkeypatch.setattr(real_gate, "close", lambda self, _c=real_gate.close: (stats.append(self.stats()), _c(self))[1])
    assert_same(sim.reduce_noise_batch(ys, SR, **kw), outs, ys)
    assert len(seen) == 1 and stats[-1]["units"] == 6          # one handle for the whole call


def test_refusals_before_any_handle(sim, monkeypatch):
    def no_handle(**kw):
        raise AssertionError("a handle was created")

    monkeypatch.setattr(_cabi, "Gate", no_handle)
    ys = [clip(2000), clip(3000, seed=1)]
    tens = [torch.from_numpy(y) for y in ys]
    for kw in (dict(use_torch=True), dict(stationary=True), dict(n_fft=2048), dict(n_fft=512), dict(hop_length=128),
               dict(win_length=512), dict(stationary=True, y_noise=NOISE, time_mask_smooth_ms=300),
               dict(stationary=True, y_noise=NOISE, freq_mask_smooth_hz=600),
               dict(time_mask_smooth_ms=1600)):
        with pytest.raises(NotImplementedError, match="|".join(kw)):
            sim.reduce_noise_batch(ys, SR, **kw)
    with pytest.raises(NotImplementedError, match="float16"):
        sim.reduce_noise_batch([y.astype(np.float16) for y in ys], SR)
    with pytest.raises(NotImplementedError, match="int32"):
        sim.reduce_noise_batch([y.astype(np.int32) for y in ys], SR)
    with pytest.raises(NotImplementedError, match="grad"):
        sim.reduce_noise_batch([tens[0], tens[1].clone().requires_grad_()], SR)
    # what reduce_noise() refuses, with its exception type
    for bad in (np.zeros(0, np.float32), np.zeros((2, 2, 100), np.float32), ys[0].astype(np.complex64)):
        with pytest.raises(ValueError):
            sim.reduce_noise(bad, SR)
        with pytest.raises(ValueError):
            sim.reduce_noise_batch([ys[0].astype(bad.dtype), bad], SR)
    with pytest.raises(ValueError):
        sim.reduce_noise_batch(ys, SR, freq_mask_smooth_hz=1)
    with pytest.raises(ValueError):
        sim.reduce_noise_batch([], SR)
    with pytest.raises(TypeError):
        sim.reduce_noise_batch(ys[0], SR)
    with pytest.raises(TypeError):
        sim.reduce_noise_batch([ys[0], tens[1]], SR)
    with pytest.raises(TypeError):
        sim.reduce_noise_batch([ys[0], ys[1].astype(np.float64)], SR)
    with pytest.raises(ValueError):
        sim.reduce_noise_batch([tens[0], tens[1].to("meta")], SR)


def test_cabi_error_codes(simlib):
    y = clip(3000)
    out = np.empty_like(y)
    row = (y.ctypes.data, out.ctypes.data, y.size, 1)

    def code(gate, rows, dtype=np.float32):
        with pytest.raises(_cabi.GateError) as e:
            gate.run_rows(rows, dtype, False)
        return e.value.code

    nonstat = dict(stationary_params(), stationary=0, time_constant_s=2.0, thresh_n_mult=2.0, sigmoid_slope=10.0)
    for params in (dict(nonstat, n_fft=2048, win_length=2048, hop_length=512), dict(nonstat, hop_length=128),
                   dict(nonstat, path_flags=64), dict(stationary_params(), n_grad_time=20)):
        g = _cabi.Gate(lib=simlib, **params)
        if params["stationary"]:
            g.noise_stats_host(NOISE[None, :])
        assert code(g, [row]) == _cabi.ERR_ARG
        g.close()
    g = _cabi.Gate(lib=simlib, **stationary_params())
    assert code(g, [row]) == _cabi.ERR_STATE                    # no thresholds yet
    g.close()
    g = _cabi.Gate(lib=simlib, **dict(nonstat, surface=_cabi.SURFACE_TORCH_CHUNKED, top_db=40.0, std_ddof=1, n_movemean=20))
    assert code(g, [row]) == _cabi.ERR_STATE
    g.close()

    g = _cabi.Gate(lib=simlib, **nonstat)
    assert code(g, [(y.ctypes.data, out.ctypes.data, 0, 1)]) == _cabi.ERR_ARG
    assert code(g, [(None, out.ctypes.data, y.size, 1)]) == _cabi.ERR_ARG
    assert code(g, [(y.ctypes.data, y.ctypes.data + 400, y.size, 1)]) == _cabi.ERR_ARG      # out overlaps in
    assert code(g, [(y.ctypes.data, out.ctypes.data, y.size, 0)]) == _cabi.ERR_ARG
    assert g.lib.dll.b200gate_run_rows(g._h, None, 1, _cabi.F32, 0, None) == _cabi.ERR_ARG
    g.set_range(1, 0, 0)
    assert code(g, [row]) == _cabi.ERR_STATE
    g.set_range(0)
    store = np.empty(1 << 20, np.uint8)
    g.set_mask_store(store.ctypes.data, store.size)
    assert code(g, [row]) == _cabi.ERR_STATE
    g.set_mask_store(None)
    g.stream_begin(np.float32, 1)
    assert code(g, [row]) == _cabi.ERR_STATE
    tail = np.empty(CS + PAD, np.float32)
    g.stream_finish(ctypes.c_void_p(tail.ctypes.data), tail.size, tail.size)
    # the handle is still usable: rows, then an ordinary run, agree
    buf = np.concatenate([y, np.zeros_like(y)])
    g.run_rows([(buf.ctypes.data, buf.ctypes.data + y.nbytes, y.size, 1)], np.float32, False)
    assert np.array_equal(buf[y.size:], g.run_host(y[None, :])[0]) and np.abs(buf[y.size:]).max() > 0
    g.close()


# ---- on the GPU ------------------------------------------------------------------------------------------------------
def _gpu_clips(n_clips, lo_s, hi_s, sr, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lens = torch.randint(int(lo_s * sr), int(hi_s * sr) + 1, (n_clips,), generator=torch.Generator().manual_seed(seed)).tolist()
    ys = []
    for n in lens:
        t = torch.arange(n, device="cuda", dtype=torch.float32) / sr
        y = 0.05 * torch.randn(n, device="cuda", generator=g)
        y += 0.3 * ((t % 1.0) < 0.4) * torch.sin(2 * math.pi * 440.0 * t)
        ys.append(y)
    return ys


@pytest.mark.gpu
@pytest.mark.parametrize("stationary", [False, True], ids=["nonstationary", "stationary"])
def test_gpu_512_clips_equal_the_loop(stationary):
    import noisereduce_b200 as nr
    sr = 48000
    ys = _gpu_clips(512, 1.0, 30.0, sr, seed=3)
    kw = dict(stationary=True, y_noise=ys[0][: 2 * sr].clone()) if stationary else {}
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        outs = nr.reduce_noise_batch(ys, sr, **kw)
    assert [o.shape for o in outs] == [y.shape for y in ys]
    order = sorted(range(len(ys)), key=lambda i: ys[i].numel())
    subset = [order[round(k * (len(order) - 1) / 31)] for k in range(32)]
    for i in subset:
        assert torch.equal(outs[i], nr.reduce_noise(ys[i], sr, **kw)), i
    assert all(float(o.abs().max()) > 0 for o in outs[:8])
    del outs, ys, kw
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= base - 512 * 48000 * 4      # inputs and results are gone, nothing else stayed


@pytest.mark.gpu
def test_gpu_int16_numpy_batch_equals_the_loop():
    import noisereduce_b200 as nr
    sr = 48000
    rng = np.random.default_rng(11)
    ys = [np.round(3000 * rng.standard_normal((C, n))).astype(np.int16)
          for C, n in ((1, 700_001), (2, 90_000), (3, 1_250_000), (1, 20_000))]
    ys[0] = ys[0][0]
    noise = ys[1][0, :48000]
    for kw in ({}, dict(stationary=True, y_noise=noise)):
        outs = nr.reduce_noise_batch(ys, sr, **kw)
        assert_same(outs, [nr.reduce_noise(y, sr, **kw) for y in ys], ys)
        assert any(np.abs(o).max() > 0 for o in outs)
