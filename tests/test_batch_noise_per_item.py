"""reduce_noise_batch(..., stationary=True, y_noise_per_item=...): every recording with thresholds of its own.

The contract is bit-identity with a loop of reduce_noise(): a None entry is reduce_noise(y, sr, stationary=True, ...)
(the item's first chunk is its noise clip), a clip is reduce_noise(y, sr, stationary=True, y_noise=clip, ...).  On the
CPU simulator (tests/cusim) the .cu sources run on the host and CPU tensors take the device route; the gpu-marked tests
repeat the comparison on the nvcc build at the sizes the feature is for."""
import math

import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from tests.test_batch import CS, HOP, NOISE, PAD, SR, assert_same, clip, stationary_params

# item lengths: between the hop overlap and the window (their own clip takes the shortened-window path), between n_fft
# and 2 n_fft, off the hop grid, exactly chunk_size, chunk_size + 1, several chunks with a ragged last one
LENGTHS = (900, 1500, 2077, CS, CS + 1, 2 * CS + 1234)


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


def loop(nr, ys, clips, **kw):
    return [nr.reduce_noise(y, SR, stationary=True, **kw) if c is None else
            nr.reduce_noise(y, SR, stationary=True, y_noise=c, **kw) for y, c in zip(ys, clips)]


def check(nr, ys, clips, **kw):
    kw = dict(dict(chunk_size=CS, padding=PAD), **kw)
    outs = nr.reduce_noise_batch(ys, SR, stationary=True, y_noise_per_item=clips, **kw)
    assert_same(outs, loop(nr, ys, clips, **kw), ys)
    return outs


@pytest.mark.parametrize("clip_noise, order", [(True, "C"), (False, "F")], ids=["clipped-C", "whole-F"])
def test_none_entries_every_length(sim, clip_noise, order):
    ys = [clip(n, seed=i) for i, n in enumerate(LENGTHS)]
    ys += [np.asarray(clip(n, C=3, seed=10 + i), order=order) for i, n in enumerate((2077, CS + 1, 2 * CS + 300))]
    outs = check(sim, ys, [None] * len(ys), clip_noise_stationary=clip_noise)
    assert all(np.abs(o).max() > 0 for o in outs)


@pytest.mark.parametrize("dtype", [np.float32, np.int16, np.float64])
def test_explicit_clips_and_fallbacks(sim, dtype):
    ys = [clip(n, C=C, seed=i, dtype=dtype) for i, (C, n) in enumerate(((1, 3000), (2, CS + 700), (1, 1300), (3, 2100),
                                                                        (1, 2600), (1, 4000), (2, 1800)))]
    clips = [NOISE,                                         # a shared clip of the item dtype group, mono
             clip(CS + 2000, C=2, seed=40, dtype=dtype),     # clipped to chunk_size, two channels
             None,
             clip(900, seed=41),                            # shorter than the window: the one-clip path
             clip(3000, seed=42).astype(np.float16),        # another dtype: np.mean's rules, the one-clip path
             clip(2500, C=2, seed=43).astype(np.float64),   # a kernel dtype of its own: a second batched group
             np.asfortranarray(clip(2200, C=3, seed=44, dtype=dtype))]
    check(sim, ys, clips)
    check(sim, ys, tuple(clips), clip_noise_stationary=False)


def test_tensor_items(sim):
    big = torch.from_numpy(clip(CS + 900, C=5, seed=7))
    ys = [big[::2, 3:],                                   # row stride 2 N, rows off a 16-byte boundary
          big[1, 100:3000],
          torch.from_numpy(clip(2 * CS + 10, C=3, seed=8))[:, ::2],     # sample stride 2: copied
          torch.from_numpy(clip(2400, seed=9)),
          torch.from_numpy(clip(1900, seed=10))]
    clips = [None, torch.from_numpy(NOISE),               # a "device" clip, read in place
             None,
             NOISE[:2000],                                # a numpy clip with device items: host statistics
             torch.from_numpy(clip(3000, C=2, seed=11))[:, ::3]]      # strided device clip
    check(sim, ys, clips)


@pytest.mark.parametrize("smooth", [dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None),
                                    dict(freq_mask_smooth_hz=540, time_mask_smooth_ms=208),     # 17 bins, 13 frames
                                    dict(prop_decrease=0.6)], ids=["none", "limits", "blend"])
def test_smoothing_settings(sim, smooth):
    ys = [clip(n, seed=i) for i, n in enumerate((1800, CS + 300, 3333))]
    check(sim, ys, [None, NOISE, None], **smooth)


def test_nan_sample(sim):
    ys = [clip(n, seed=i) for i, n in enumerate((2600, CS + 400, 3100))]
    ys[1][77] = np.nan
    check(sim, ys, [None, None, NOISE])


def _tone(n, amp, seed):
    t = np.arange(n) / SR
    rng = np.random.default_rng(seed)
    return (1e-5 * rng.standard_normal(n) + amp * np.sin(2 * np.pi * 1000 * t)).astype(np.float32)


def test_each_unit_reads_its_own_tables(sim, simlib):
    """A quiet item next to a loud one (one table for all would gate one of them wrongly); a tone whose quiet clip lets its
    top_db floor lift rows next to items that lift none; then a wide guard band, so that many bins are re-decided in
    float64 -- outputs and counters equal the per-item runs."""
    quiet = (1e-4 * np.random.default_rng(3).standard_normal(CS + 2000)).astype(np.float32)
    loud = clip(CS + 2000, seed=4) * 30
    ys = [quiet, loud]
    outs = check(sim, ys, [None, None])
    shared = sim.reduce_noise(quiet, SR, stationary=True, y_noise=loud, chunk_size=CS, padding=PAD)
    assert not np.array_equal(outs[0], shared)             # the quiet item's own thresholds matter

    tone = _tone(6000, 0.9, 5)
    ys = [tone, clip(2500, seed=6), np.zeros(3000, np.float32), clip(CS + 200, seed=7)]
    clips = [quiet[:3000], None, NOISE, None]
    check(sim, ys, clips)

    def per_item(params):
        rows_thr, outs_ref, st_ref = [], [], dict(rowfloor_flags=0, bins_rechecked_fp64=0)
        for y, c in zip(ys, clips):
            g = _cabi.Gate(lib=simlib, **params)
            g.noise_stats_host((y if c is None else c)[None, :])
            rows_thr.append(g.noise_threshold())
            outs_ref.append(g.run_host(y[None, :])[0])
            for k in st_ref:
                st_ref[k] += g.stats()[k]
            g.close()
        return np.array(rows_thr), outs_ref, st_ref

    for params in (stationary_params(), stationary_params(debug_guard_scale=100000)):
        thr, outs_ref, st_ref = per_item(params)
        outs, st = _rows_call(simlib, params, ys, thr)
        for o, r in zip(outs, outs_ref):
            assert np.array_equal(o, r, equal_nan=True)
        assert st["rowfloor_flags"] == st_ref["rowfloor_flags"]
        assert st["bins_rechecked_fp64"] == st_ref["bins_rechecked_fp64"] and st["bins_unresolved"] == 0
    assert st_ref["bins_rechecked_fp64"] > 100
    assert per_item(stationary_params())[2]["rowfloor_flags"] > 0


def _rows_call(lib, params, ys, thr, channels=None):
    """b200gate_run_rows on mono host rows packed in one buffer, with per-recording thresholds; (outputs, stats)."""
    gate = _cabi.Gate(lib=lib, **params)
    gate.set_noise_threshold_rows(thr)
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
    return [buf[total + o - y.size: total + o].copy() for y, o in zip(ys, np.cumsum([y.size for y in ys]))], st


def test_workspace_batches(sim, simlib, monkeypatch):
    """A limit of about two units and two clips: units and statistics groups both span several batches."""
    ys = [clip(n, seed=i) for i, n in enumerate((2 * CS + 100, 1200, 3100, CS, 2700))]
    clips = [None, NOISE, None, clip(CS + 50, C=2, seed=30), None]
    ref = loop(sim, ys, clips, chunk_size=CS, padding=PAD)
    real_gate = _cabi.Gate
    seen = []

    def small_workspace(**params):
        g = real_gate(workspace_limit_bytes=3.0e5, **params)
        seen.append(g)
        return g

    monkeypatch.setattr(_cabi, "Gate", small_workspace)
    outs = sim.reduce_noise_batch(ys, SR, stationary=True, y_noise_per_item=clips, chunk_size=CS, padding=PAD)
    assert_same(outs, ref, ys)
    assert len(seen) == 1
    # the statistics groups alone: rows equal the one-clip statistics
    g = real_gate(lib=simlib, **stationary_params(workspace_limit_bytes=3.0e5))
    cl = [clip(n, seed=50 + i) for i, n in enumerate((CS + 10, 4000, 1024, 2500, 7000))]
    keep = [np.ascontiguousarray(c[None, :]) for c in cl]
    thr = g.noise_stats_rows([(k.ctypes.data, 1, k.shape[1], k.shape[1]) for k in keep], np.float32, False)
    for k, t in zip(keep, thr):
        g.noise_stats_host(k)
        assert np.array_equal(g.noise_threshold(), t)
    g.close()


@pytest.mark.parametrize("dtype", [np.float32, np.int16, np.float64])
@pytest.mark.parametrize("is_device", [False, True], ids=["host", "device"])
def test_cabi_noise_stats_rows_equal_one_clip(simlib, dtype, is_device):
    params = stationary_params()
    cl = [clip(n, C=C, seed=60 + i, dtype=dtype) for i, (C, n) in enumerate(((1, 1024), (3, CS + 900), (2, 4000), (1, 1025)))]
    big = np.zeros((2, 6000), dtype)                      # a clip in rows of a longer buffer: row stride 6000
    big[:, :3500] = clip(3500, C=2, seed=70, dtype=dtype)
    specs = [(c.ctypes.data, c.shape[0], c.shape[1], c.shape[1]) for c in cl] + [(big.ctypes.data, 2, 3500, 6000)]
    for clip_noise in (1, 0):
        g = _cabi.Gate(lib=simlib, **dict(params, clip_noise=clip_noise))
        thr = g.noise_stats_rows(specs, dtype, is_device)
        for (ptr, C, n, stride), t in zip(specs, thr):
            g.noise_stats_device(ptr, dtype, C, n, stride) if is_device else \
                g.noise_stats_host((big[:, :n] if stride == 6000 else next(c for c in cl if c.ctypes.data == ptr)))
            assert np.array_equal(g.noise_threshold(), t, equal_nan=True)
        g.close()


def test_cabi_error_codes_and_state(simlib):
    params = stationary_params()
    ys = [clip(3000, seed=1), clip(2000, seed=2)]
    g = _cabi.Gate(lib=simlib, **params)
    short = clip(1000)
    for specs in ([(short.ctypes.data, 1, 1000, 1000)], [(None, 1, 1000, 1000)], [(ys[0].ctypes.data, 2, 3000, 100)]):
        with pytest.raises(_cabi.GateError) as e:
            g.noise_stats_rows(specs, np.float32, False)
        assert e.value.code == _cabi.ERR_ARG
    thr = g.noise_stats_rows([(y.ctypes.data, 1, y.size, y.size) for y in ys], np.float32, False)
    for bad in (thr[:, :100], thr[:0]):
        with pytest.raises(_cabi.GateError) as e:
            g.set_noise_threshold_rows(bad)
        assert e.value.code == _cabi.ERR_ARG
    g.set_noise_threshold_rows(thr)
    buf = np.concatenate([ys[0], ys[0], ys[1], np.zeros(8000, np.float32)])
    p = buf.ctypes.data

    def code(rows):
        with pytest.raises(_cabi.GateError) as e:
            g.run_rows(rows, np.float32, False)
        return e.value.code

    out = p + 8000 * 4
    assert code([(p, out, 3000, 1)]) == _cabi.ERR_ARG                                      # 1 recording, 2 rows
    assert code([(p, out, 3000, 1), (p + 12000, out + 12000, 3000, 1), (p + 24000, out + 24000, 2000, 1)]) == _cabi.ERR_ARG
    assert code([(p, out, 3000, 2), (p + 24000, out + 24000, 2000, 2)]) == _cabi.ERR_ARG      # unequal n in a recording
    assert code([(p, out, 3000, 2), (p + 12000, out + 12000, 3000, 1)]) == _cabi.ERR_ARG      # unequal channels
    assert code([(p, out, 3000, 1), (p + 24000, out + 24000, 2000, 3)]) == _cabi.ERR_ARG      # runs past the last row
    with pytest.raises(_cabi.GateError) as e:
        g.run_host(ys[0][None, :])
    assert e.value.code == _cabi.ERR_STATE
    with pytest.raises(_cabi.GateError) as e:
        g.noise_threshold()
    assert e.value.code == _cabi.ERR_STATE
    s = _cabi.Gate(lib=simlib, **params)                 # a stationary stream returns no chunk with them
    s.set_noise_threshold_rows(thr)
    s.stream_begin(np.float32, 1)
    x, sink = clip(CS + 2 * PAD + 10), np.empty(3 * CS, np.float32)
    with pytest.raises(_cabi.GateError) as e:
        s.stream_push(x.ctypes.data, x.size, x.size, False, sink.ctypes.data, sink.size, sink.size)
    assert e.value.code == _cabi.ERR_STATE
    s.close()
    # mono recordings with their own thresholds: the rows equal the one-set runs
    two = np.concatenate([ys[0], ys[1], np.zeros(5000, np.float32)])
    q = two.ctypes.data
    g.run_rows([(q, q + 5000 * 4, 3000, 1), (q + 3000 * 4, q + 8000 * 4, 2000, 1)], np.float32, False)
    for k, (y, t) in enumerate(zip(ys, thr)):
        h = _cabi.Gate(lib=simlib, **params)
        h.set_noise_threshold(t)
        assert np.array_equal(two[5000 + 3000 * k: 5000 + 3000 * k + y.size], h.run_host(y[None, :])[0])
        h.close()
    # back to one set: the shared-threshold behaviour
    g.set_noise_threshold(thr[1])
    assert np.array_equal(g.noise_threshold(), thr[1])
    two[5000:] = 0
    g.run_rows([(q, q + 5000 * 4, 3000, 1), (q + 3000 * 4, q + 8000 * 4, 2000, 1)], np.float32, False)
    for k, y in enumerate(ys):
        assert np.array_equal(two[5000 + 3000 * k: 5000 + 3000 * k + y.size], g.run_host(y[None, :])[0])
    g.close()
    nonstat = dict(params, stationary=0, time_constant_s=2.0, thresh_n_mult=2.0, sigmoid_slope=10.0)
    h = _cabi.Gate(lib=simlib, **nonstat)
    with pytest.raises(_cabi.GateError) as e:
        h.set_noise_threshold_rows(thr)
    assert e.value.code == _cabi.ERR_ARG
    h.close()


def test_refusals(sim, monkeypatch):
    ys = [clip(2000), clip(3000, seed=1)]
    kw = dict(chunk_size=CS, padding=PAD)

    def no_handle(**kw):
        raise AssertionError("a handle was created")

    real_gate = _cabi.Gate
    monkeypatch.setattr(_cabi, "Gate", no_handle)
    for bad in (dict(stationary=True, y_noise=NOISE, y_noise_per_item=[None, None]),
                dict(y_noise_per_item=[None, None]),
                dict(stationary=True, y_noise_per_item=[None]),
                dict(stationary=True, y_noise_per_item=[None, None, NOISE])):
        with pytest.raises(ValueError, match="y_noise_per_item"):
            sim.reduce_noise_batch(ys, SR, **kw, **bad)
    with pytest.raises(NotImplementedError, match="stationary"):
        sim.reduce_noise_batch(ys, SR, stationary=True)
    # clips reduce_noise() refuses: the same exception type, before any handle
    for c in (np.zeros(0, np.float32), clip(700), torch.from_numpy(NOISE).to("meta"), clip(600, C=2)):
        monkeypatch.setattr(_cabi, "Gate", real_gate)
        with pytest.raises(Exception) as ref:
            sim.reduce_noise(torch.from_numpy(ys[0]), SR, stationary=True, y_noise=c, **kw)
        monkeypatch.setattr(_cabi, "Gate", no_handle)
        with pytest.raises(ref.type):
            sim.reduce_noise_batch([torch.from_numpy(y) for y in ys], SR, stationary=True, y_noise_per_item=[None, c], **kw)
    with pytest.raises(ValueError, match="noverlap"):
        sim.reduce_noise_batch([clip(700), ys[1]], SR, stationary=True, y_noise_per_item=[None, None], **kw)
    # a "device" clip with host items: what reduce_noise() does with it (np.array), exception type included
    meta = torch.from_numpy(NOISE).to("meta")
    monkeypatch.setattr(_cabi, "Gate", real_gate)
    with pytest.raises(Exception) as ref:
        sim.reduce_noise(ys[0], SR, stationary=True, y_noise=meta, **kw)
    with pytest.raises(ref.type):
        sim.reduce_noise_batch(ys, SR, stationary=True, y_noise_per_item=[meta, None], **kw)
    tens = torch.from_numpy(NOISE)
    check(sim, ys, [tens, None])                        # (a CPU tensor with host items: numpy's copy, as reduce_noise())


# ---- on the GPU ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_512_clips_own_thresholds_equal_the_loop():
    import noisereduce_b200 as nr
    from tests.test_batch import _gpu_clips
    sr = 48000
    ys = _gpu_clips(512, 1.0, 30.0, sr, seed=5)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        outs = nr.reduce_noise_batch(ys, sr, stationary=True, y_noise_per_item=[None] * len(ys))
    assert [o.shape for o in outs] == [y.shape for y in ys]
    order = sorted(range(len(ys)), key=lambda i: ys[i].numel())
    subset = [order[round(k * (len(order) - 1) / 31)] for k in range(32)]
    for i in subset:
        assert torch.equal(outs[i], nr.reduce_noise(ys[i], sr, stationary=True)), i
    assert all(float(o.abs().max()) > 0 for o in outs[:8])
    del outs, ys
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= base - 512 * 48000 * 4


@pytest.mark.gpu
def test_gpu_int16_numpy_multichannel_mixed_clips():
    import noisereduce_b200 as nr
    sr = 48000
    rng = np.random.default_rng(12)
    ys = [np.round(3000 * rng.standard_normal((C, n))).astype(np.int16)
          for C, n in ((1, 700_001), (2, 90_000), (3, 1_250_000), (1, 20_000), (2, 650_000))]
    ys[0] = ys[0][0]
    clips = [None, ys[1][0, :48000], None, np.round(500 * rng.standard_normal((2, 30_000))).astype(np.int16),
             rng.standard_normal(9000).astype(np.float32)]
    outs = nr.reduce_noise_batch(ys, sr, stationary=True, y_noise_per_item=clips)
    assert_same(outs, [nr.reduce_noise(y, sr, stationary=True, y_noise=c) for y, c in zip(ys, clips)], ys)
    assert all(np.abs(o).max() > 0 for o in outs)
