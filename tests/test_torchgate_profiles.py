"""TorchGate.sessions(profiles=...): every row of one sessions object gated with its own profile's sample rate and gate
strength.

The contract is bit-identity per session: everything returned for a session on profile k equals
TorchGate(nonstationary=True, **module settings overridden by profile k)(x_s[None])[0], however the session was cut and
whatever the other rows and their profiles did.  On the CPU simulator (tests/cusim) the .cu sources run on the host with
CPU tensors; the gpu-marked test repeats the comparison on the nvcc build with 256 rows on three sample rates."""
import ctypes

import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from noisereduce_b200.torchgate import TorchGate
from tests.cusim_util import cusim_library
from tests.synth_host import synth_torchgate

SR, HOP = 16000, 256
NO_SMOOTHING = dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None)
# extents (nf, nt): 8 kHz (32, 1) and 16 kHz (16, 3) smooth with k_smooth_stream, 48 kHz (5, 9) with k_smooth_box<5>
MIXED = [dict(sr=8000, n_movemean_nonstationary=1), dict(n_movemean_nonstationary=7, prop_decrease=0.6),
         dict(sr=48000, n_movemean_nonstationary=40), dict(n_movemean_nonstationary=20, **NO_SMOOTHING)]


@pytest.fixture(scope="module")
def lib():
    return cusim_library()


def signal(B, L, seed=7):
    return torch.from_numpy(synth_torchgate(B=B, n=L, seed=seed))


def profile_gate(tg, profile):
    """The TorchGate a session on this profile equals."""
    kw = dict(sr=tg.sr, n_thresh_nonstationary=tg.n_thresh_nonstationary, temp_coeff_nonstationary=tg.temp_coeff_nonstationary,
              n_movemean_nonstationary=tg.n_movemean_nonstationary, prop_decrease=tg.prop_decrease,
              freq_mask_smooth_hz=tg.freq_mask_smooth_hz, time_mask_smooth_ms=tg.time_mask_smooth_ms)
    kw.update(profile)
    return TorchGate(nonstationary=True, **kw)


class Driver:
    """Feeds a TorchGateSessions with profiles and keeps, per session, its profile, samples and output; checks the
    documented counts of each row's profile after every call."""

    def __init__(self, tg, n_rows, profiles, lib, dtype=torch.float32):
        self.tg, self.profiles = tg, profiles
        self.ss = tg.sessions(n_rows, profiles=profiles, _lib=lib)
        self.lib, self.dtype, self.B = lib, dtype, n_rows
        self.prof = [0] * n_rows
        self.x = [[] for _ in range(n_rows)]
        self.y = [[] for _ in range(n_rows)]
        self.done = []                                   # (profile, samples, output) of every ended session

    def assign(self, rows, k):
        self.ss.assign(rows, k)
        for b in rows:
            self.prof[b] = k

    def push(self, blocks):
        n = [int(v.shape[0]) for v in blocks]
        block = torch.zeros((self.B, max(n)), dtype=self.dtype)
        for b, v in enumerate(blocks):
            block[b, :n[b]] = v
        before = self.ss.samples_returned
        y, m = self.ss.push(block, n)
        assert y.dtype == self.dtype and y.shape == (self.B, max(m))
        for b in range(self.B):
            self.x[b].append(blocks[b])
            self.y[b].append(y[b, :m[b]])
            R = self.ss.samples_received[b]
            assert self.ss.samples_returned[b] == before[b] + m[b] == self.ss.returned_after(R, profile=self.prof[b])
            assert 0 <= R - self.ss.samples_returned[b] <= self.ss.latency_samples_per_profile[self.prof[b]]

    def end(self, rows):
        y, m = self.ss.end(rows)
        for i, b in enumerate(rows):
            xs, out = torch.cat(self.x[b]), torch.cat(self.y[b] + [y[i, :m[i]]])
            assert out.shape[0] == (xs.shape[0] // HOP) * HOP
            self.done.append((self.prof[b], xs, out))
            self.x[b], self.y[b] = [], []

    def reset(self, rows):
        self.ss.reset(rows)
        for b in rows:
            self.x[b], self.y[b] = [], []

    def check(self, min_sessions):
        assert len(self.done) >= min_sessions
        gates = [profile_gate(self.tg, p) for p in self.profiles]
        for k, xs, out in self.done:
            assert torch.equal(out, gates[k](xs[None], _lib=self.lib)[0]), k


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_mixed_profiles_bit_identical(lib, dtype):
    """Six rows on four profiles (8 / 16 / 48 kHz and smoothing off; n_movemean 1, 7, 40, 20; prop_decrease 0.6 and 1.0)
    in seeded random per-tick lengths; sessions end and restart on another profile, and one is dropped by reset()."""
    tg = TorchGate(sr=SR, nonstationary=True)
    rng = np.random.default_rng(21)
    x = signal(6, 60000, seed=4).to(dtype)
    d = Driver(tg, 6, MIXED, lib, dtype)
    d.assign([1, 4], 1)
    d.assign([2], 2)
    d.assign([3, 5], 3)
    pos = [0] * 6
    choices = [0, 1, 100, 255, 257, 320, 700, 960, 4500]
    for tick in range(36):
        n = rng.choice(choices, size=6)
        d.push([x[b, pos[b]:pos[b] + n[b]] for b in range(6)])
        pos = [pos[b] + int(n[b]) for b in range(6)]
        if tick in (11, 23):
            rows = [b for b in range(6) if d.ss.samples_received[b] >= 2048][:3]
            d.end(rows)
            for b in rows:                                  # the row's next session is on the next profile
                d.assign([b], (d.prof[b] + 1) % 4)
        if tick == 17:
            d.reset([5])
            d.assign([5], 2)
    d.end([b for b in range(6) if d.ss.samples_received[b] >= 2048])
    d.ss.close()
    d.check(min_sessions=8)
    assert {k for k, _, _ in d.done} == {0, 1, 2, 3}


def same(outs):
    """Every (y, m) of outs returns what the first does (row i's y[i, :m[i]])."""
    y0, m0 = outs[0]
    for y, m in outs[1:]:
        assert m == m0 and all(torch.equal(y[i, :k], y0[i, :k]) for i, k in enumerate(m))


def test_single_profile_equals_plain_sessions(lib):
    """profiles=[{}] (and a profile repeating the module's sample rate) give today's sessions() in every bit."""
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(3, 16000, seed=8)
    objs = [tg.sessions(3, _lib=lib), tg.sessions(3, profiles=[{}], _lib=lib),
            tg.sessions(3, profiles=[dict(sr=SR)], _lib=lib)]
    assert all(o.latency_samples == objs[0].latency_samples for o in objs)
    cuts = [(0, 0, 0), (700, 1, 3000), (5000, 2500, 3001), (9000, 9000, 9999), (16000, 12000, 16000)]
    for a, b in zip(cuts, cuts[1:]):
        n = [b[r] - a[r] for r in range(3)]
        blk = torch.zeros(3, max(n))
        for r in range(3):
            blk[r, :n[r]] = x[r, a[r]:b[r]]
        outs = [o.push(blk, n) for o in objs]
        same(outs)
    same([o.end([2, 0, 1]) for o in objs])
    for o in objs:
        o.close()


def test_counts_and_latency_per_profile(lib):
    tg = TorchGate(sr=SR, nonstationary=True)
    ss = tg.sessions(2, profiles=MIXED, _lib=lib)
    lat = []
    for p in MIXED:
        one = profile_gate(tg, p).sessions(1, _lib=lib)
        lat.append(one.latency_samples)
        for R in (0, 511, 512, 3000, 7777, 20000):
            assert ss.returned_after(R, profile=len(lat) - 1) == one.returned_after(R)
    assert ss.latency_samples_per_profile == lat and ss.latency_samples == max(lat)
    assert ss.returned_after(9000) == ss.returned_after(9000, profile=0)
    for bad in (-1, 4, 1.0, True):
        with pytest.raises(ValueError, match="profile"):
            ss.returned_after(9000, profile=bad)


def _bytes_in_use():
    """Heap bytes allocated and not freed: the main arena's plus the mmapped blocks'.  The sum does not depend on where
    glibc puts a large block, which moves with its dynamic mmap threshold (raised whenever an mmapped block is freed)."""
    class MallInfo2(ctypes.Structure):
        _fields_ = [(n, ctypes.c_size_t) for n in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                                   "uordblks", "fordblks", "keepcost")]
    libc = ctypes.CDLL(None)
    libc.mallinfo2.restype = MallInfo2
    m = libc.mallinfo2()
    return m.uordblks + m.hblkhd


def test_state_fixed_and_sized_by_largest_profile(lib):
    """The simulator's device buffers are host allocations made by the pushing thread.  An object whose second profile
    has the longest moving mean holds what a single-profile object of that setting holds, far more than the default's;
    and what it holds stays the same over 600 pushes with sessions ending, restarting on the other profile and being
    dropped.  (Tolerance: the transient host allocations of a push, a few KB.)"""
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(2, 320 * 600, seed=1)
    long_mm = dict(n_movemean_nonstationary=300)

    def opened(ss):
        h0 = _bytes_in_use()
        ss.push(x[:, :320], [320, 320])
        return ss, _bytes_in_use() - h0

    opened(tg.sessions(2, profiles=[{}, long_mm], _lib=lib))[0].close()     # (one-time allocations of the library)
    small_ss, small = opened(tg.sessions(2, _lib=lib))
    big_ss, big = opened(profile_gate(tg, long_mm).sessions(2, _lib=lib))
    ss, both = opened(tg.sessions(2, profiles=[{}, long_mm], _lib=lib))
    small_ss.close()
    big_ss.close()
    assert big > small + (4 << 20)
    assert abs(both - big) <= 64 << 10
    after = None
    for k in range(1, 600):
        blk = x[:, 320 * k:320 * (k + 1)]
        ss.push(blk, [320, 160 + (k % 3) * 80])
        if k % 20 == 19:
            row = k // 20 % 2
            ss.end([row])
            ss.assign([row], (k // 40) % 2)
        elif k % 40 == 25:
            ss.reset([1])
        if k == 10:
            after = _bytes_in_use()
    assert abs(_bytes_in_use() - after) <= 64 << 10
    ss.close()


# ---- refusals -------------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_handles(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("a library handle was made")
    monkeypatch.setattr(_cabi, "Gate", boom)


@pytest.mark.parametrize("kw,profiles,match", [
    (dict(), [{}], "nonstationary"),
    (dict(nonstationary=True, n_fft=512), [{}], "n_fft"),
    (dict(nonstationary=True), [{}, dict(time_mask_smooth_ms=400)], "profile 1: .*time_mask_smooth_ms"),
    (dict(nonstationary=True), [dict(sr=4000, time_mask_smooth_ms=3000)], "profile 0: .*time_mask_smooth_ms")])
def test_not_implemented_before_any_handle(no_handles, kw, profiles, match):
    tg = TorchGate(sr=SR, **kw)
    with pytest.raises(NotImplementedError, match=match):
        tg.sessions(2, profiles=profiles)


@pytest.mark.parametrize("profiles,match", [
    ([], "non-empty list"), (dict(sr=8000), "non-empty list"), ([8000], "profile 0: a profile is a dict"),
    ([{}, dict(n_fft=512)], "profile 1: unknown key"), ([dict(nonstationary=False)], "profile 0: unknown key"),
    ([dict(prop_decrease=1.5)], "profile 0: prop_decrease"), ([{}, dict(prop_decrease=-0.1)], "profile 1: prop_decrease"),
    ([{}, {}, dict(n_movemean_nonstationary=0)], "profile 2: n_movemean_nonstationary"),
    ([dict(sr=48000, freq_mask_smooth_hz=50)], "profile 0: freq_mask_smooth_hz needs to be at least 93"),
    ([{}, dict(sr=8000, time_mask_smooth_ms=20)], "profile 1: time_mask_smooth_ms needs to be at least 32"),
    ([dict(temp_coeff_nonstationary=0)], "profile 0: temp_coeff")])
def test_bad_profiles_before_any_handle(no_handles, profiles, match):
    with pytest.raises(ValueError, match=match):
        TorchGate(sr=SR, nonstationary=True).sessions(2, profiles=profiles)


@pytest.mark.parametrize("block,exc,match", [(torch.zeros(2, 10, dtype=torch.float64), NotImplementedError, "float64"),
                                             (torch.zeros(2, 10, requires_grad=True), NotImplementedError, "grad")])
def test_bad_blocks_before_any_handle(no_handles, block, exc, match):
    ss = TorchGate(sr=SR, nonstationary=True).sessions(2, profiles=MIXED, _lib=object())
    with pytest.raises(exc, match=match):
        ss.push(block, [1, 1])


def test_assign_refusals(no_handles):
    ss = TorchGate(sr=SR, nonstationary=True).sessions(3, profiles=MIXED[:2], _lib=object())
    for rows, k, match in (([3], 1, "range"), ([-1], 1, "range"), ([0, 0], 1, "repeat"), ([0.5], 1, "ints"),
                           ([0], 2, "profile"), ([0], -1, "profile"), ([0], 1.0, "profile")):
        with pytest.raises(ValueError, match=match):
            ss.assign(rows, k)
    ss.assign([0, 2], 1)                                  # no handle yet: recorded for the first push


def test_assign_on_a_live_session_changes_nothing(lib):
    tg = TorchGate(sr=SR, nonstationary=True)
    d = Driver(tg, 2, MIXED[:3], lib)
    d.assign([1], 2)                                      # before the handle exists
    x = signal(2, 9000, seed=6)
    d.push([x[0, :3000], x[1, :0]])
    with pytest.raises(ValueError, match=r"rows \[0\] hold a session"):
        d.ss.assign([1, 0], 1)
    d.assign([1], 1)                                      # row 1 is still empty: allowed
    d.push([x[0, 3000:], x[1, :9000]])
    d.end([0, 1])
    d.ss.close()
    with pytest.raises(ValueError, match="after close"):
        d.ss.assign([0], 1)
    d.check(min_sessions=2)
    assert [k for k, _, _ in d.done] == [0, 1]


def test_stream_takes_no_profiles():
    with pytest.raises(TypeError):
        TorchGate(sr=SR, nonstationary=True).stream(2, profiles=[{}])


# ---- C ABI ----------------------------------------------------------------------------------------------------------------
def torch_gate(lib):
    g = _cabi.Gate(lib=lib, surface=_cabi.SURFACE_TORCH, stationary=0, n_fft=1024, win_length=1024, hop_length=256,
                   n_grad_freq=16, n_grad_time=3, std_ddof=1, sr=float(SR), prop_decrease=1.0, top_db=40.0, n_movemean=20,
                   thresh_n_mult=1.3, sigmoid_slope=10.0)
    g.set_window(torch.hann_window(1024).numpy())
    return g


def i64(*v):
    return np.array(v, dtype=np.int64)


def code(call):
    with pytest.raises(_cabi.GateError) as e:
        call()
    return e.value.code


P16 = (16, 3, 20, 1.3, 10.0, 1.0)                         # the module's own settings
P48 = (5, 9, 7, 1.3, 10.0, 0.7)                           # 48 kHz, n_movemean 7, prop_decrease 0.7


def test_cabi_profile_errors(lib):
    g = torch_gate(lib)
    assert code(lambda: g.tstream_set_profiles([])) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_set_profiles([P16, (16, 200, 20, 1.3, 10.0, 1.0)])) == _cabi.ERR_ARG   # nt: shared memory
    assert code(lambda: g.tstream_set_profiles([P16, (-1, 3, 20, 1.3, 10.0, 1.0)])) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_set_profiles([P16, (16, 3, 0, 1.3, 10.0, 1.0)])) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_set_profiles([(16, 3, 20, 1.3, 10.0, 1.01)])) == _cabi.ERR_ARG
    g.tstream_set_profiles([P16, P48])
    g.tstream_begin(2)
    assert code(lambda: g.tstream_set_profiles([P16])) == _cabi.ERR_STATE                # while a stream is open
    x = signal(2, 6000).contiguous()
    y = torch.zeros(2, 8000)
    xp, yp = x.data_ptr(), y.data_ptr()
    # the lockstep calls refuse a stream of several profiles, before any change
    assert code(lambda: g.tstream_push(xp, 100, 6000, yp, 8000, 8000)) == _cabi.ERR_STATE
    assert code(lambda: g.tstream_finish(yp, 8000, 8000)) == _cabi.ERR_STATE
    assert code(lambda: g.tstream_assign_rows(i64(1), 2)) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_assign_rows(i64(1), -1)) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_assign_rows(i64(1, 1), 1)) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_assign_rows(i64(2), 1)) == _cabi.ERR_ARG
    g.tstream_assign_rows(i64(1), 1)
    got = g.tstream_push_rows(xp, i64(3000, 2500), 6000, yp, 8000, 8000)
    # a row holding samples keeps its profile: nothing changes, not even the other listed row
    assert code(lambda: g.tstream_assign_rows(i64(0, 1), 0)) == _cabi.ERR_ARG
    x1 = x[:, 3000:].contiguous()
    y2 = torch.zeros(2, 8000)
    got2 = g.tstream_push_rows(x1.data_ptr(), i64(3000, 3000), 3000, y2.data_ptr(), 8000, 8000)
    yt = torch.zeros(2, 8000)
    tail = g.tstream_end_rows(i64(1, 0), yt.data_ptr(), 8000, 8000)
    tg = TorchGate(sr=SR, nonstationary=True)
    gates = {0: tg, 1: TorchGate(sr=48000, nonstationary=True, n_movemean_nonstationary=7, prop_decrease=0.7)}
    for i, b in enumerate((1, 0)):
        xs = torch.cat([x[b, :(3000, 2500)[b]], x1[b]])
        out = torch.cat([y[b, :got[b]], y2[b, :got2[b]], yt[i, :tail[i]]])
        assert torch.equal(out, gates[b](xs[None], _lib=lib)[0])
    g.close()


def test_cabi_one_set_profile_runs_lockstep(lib):
    """A single profile given by b200gate_tstream_set_profiles is what the lockstep calls gate with."""
    g = torch_gate(lib)
    g.tstream_set_profiles([P48])
    g.tstream_begin(2)
    x = signal(2, 5000).contiguous()
    y = torch.zeros(2, 6000)
    m = g.tstream_push(x.data_ptr(), 5000, 5000, y.data_ptr(), 6000, 6000)
    yt = torch.zeros(2, 6000)
    t = g.tstream_finish(yt.data_ptr(), 6000, 6000)
    ref = TorchGate(sr=48000, nonstationary=True, n_movemean_nonstationary=7, prop_decrease=0.7)(x, _lib=lib)
    assert torch.equal(torch.cat([y[:, :m], yt[:, :t]], 1), ref)
    g.close()


# ---- H100 ---------------------------------------------------------------------------------------------------------------
def _outside_torch():
    """Device memory in use outside torch's caching allocator (the library's allocations)."""
    free, total = torch.cuda.mem_get_info()
    return total - free - torch.cuda.memory_reserved()


@pytest.mark.gpu
def test_gpu_256_rows_three_sample_rates_side_stream():
    """256 rows on three profiles (8 / 16 / 48 kHz, the 48 kHz one at prop_decrease 0.7); sessions of 5-60 s start and
    end at seeded ticks, each on a random profile, in 10-30 ms jittered blocks at its own rate, pushed on a side
    stream.  Every completed session equals its profile's TorchGate in every bit."""
    rng = np.random.default_rng(1)
    B, ticks = 256, 800
    profiles = [dict(sr=8000), dict(sr=16000), dict(sr=48000, prop_decrease=0.7)]
    rates = np.array([8000, 16000, 48000])
    tg = TorchGate(sr=SR, nonstationary=True).to("cuda")
    gates = [profile_gate(tg, p).to("cuda") for p in profiles]
    torch.cuda.synchronize()
    alloc0 = torch.cuda.memory_allocated()
    L = 61 * 48000
    src = (torch.randn(B, L, device="cuda") * 0.1 + torch.sin(torch.arange(L, device="cuda") * 0.05)[None]).contiguous()
    prof = rng.integers(0, 3, size=B)
    want = (rng.uniform(5, 60, size=B) * rates[prof]).astype(np.int64)
    want[: B // 4] = (rng.uniform(5, 12, size=B // 4) * rates[prof[: B // 4]]).astype(np.int64)   # (some end early)
    start = rng.integers(0, 100, size=B)
    got_x = [[] for _ in range(B)]
    got_y = [[] for _ in range(B)]
    pos = np.zeros(B, dtype=np.int64)
    done, ye = [], None
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        warm = tg.sessions(B, profiles=profiles)             # (loads the kernels this test runs)
        warm.assign(list(range(B)), 2)
        for i in range(8):
            warm.push(src[:, 960 * i:960 * (i + 1)].contiguous(), [960] * B)
        warm.end(list(range(B)))
        warm.close()
        torch.cuda.synchronize()
        lib0 = _outside_torch()
        ss = tg.sessions(B, profiles=profiles)
        for k in range(3):
            ss.assign(np.nonzero(prof == k)[0].tolist(), k)
        for k in range(ticks):
            n = (rng.uniform(0.010, 0.030, size=B) * rates[prof]).astype(np.int64)
            n[start > k] = 0
            n = np.minimum(n, want - pos)
            width = int(n.max())
            off = rng.integers(0, L - width, size=B)
            idx = torch.from_numpy(off[:, None] + np.arange(max(width, 1))[None, :]).cuda()
            block = torch.gather(src, 1, idx)[:, :width].contiguous()
            y, m = ss.push(block, n)
            for b in np.nonzero(n)[0]:
                got_x[b].append(block[b, :n[b]])
            for b in np.nonzero(m)[0]:
                got_y[b].append(y[b, :m[b]])
            pos += n
            ending = [int(b) for b in np.nonzero(pos >= want)[0]]
            if ending:
                ye, me = ss.end(ending)
                for i, b in enumerate(ending):
                    done.append((int(prof[b]), torch.cat(got_x[b]), torch.cat(got_y[b] + [ye[i, :me[i]]])))
                    got_x[b], got_y[b] = [], []
                    pos[b] = 0
                    prof[b] = rng.integers(0, 3)
                    ss.assign([b], int(prof[b]))
                    want[b] = int(rng.uniform(5, 60) * rates[prof[b]])
                    start[b] = k + 1 + rng.integers(0, 50)
        ss.close()
        assert _outside_torch() <= lib0 + (4 << 20)              # the stream's device state is released by close()
    torch.cuda.current_stream().wait_stream(side)
    assert len(done) >= 32
    assert {k for k, _, _ in done} == {0, 1, 2}
    for k, xs, out in done:
        assert torch.equal(out, gates[k](xs[None])[0]), k
    del done, got_x, got_y, y, ye, block, idx, src, xs, out
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= alloc0
