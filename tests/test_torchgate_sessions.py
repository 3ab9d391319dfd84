"""TorchGate.sessions(): many live sessions in one stream, each row starting, receiving samples and ending at its own pace.

The contract is bit-identity per session: the concatenation of everything returned for a session, by pushes and by its
end(), equals tg(x_s[None])[0] for the session's samples x_s, however the session was cut, whatever the other rows did
and whichever row it used.  On the CPU simulator (tests/cusim) the .cu sources run on the host with CPU tensors; the
gpu-marked tests repeat the comparison on the nvcc build with 256 rows of sessions that start and end at random ticks."""
import ctypes

import numpy as np
import pytest
import torch

from noisereduce_b200 import _cabi
from noisereduce_b200.torchgate import TorchGate, TorchGateSessions
from tests.cusim_util import cusim_library
from tests.synth_host import synth_torchgate

SR, HOP = 16000, 256
NO_SMOOTHING = dict(freq_mask_smooth_hz=None, time_mask_smooth_ms=None)


@pytest.fixture(scope="module")
def lib():
    return cusim_library()


def signal(B, L, seed=7):
    return torch.from_numpy(synth_torchgate(B=B, n=L, seed=seed))


class Driver:
    """Feeds the rows of a TorchGateSessions from per-row sample sources and keeps, per session, its samples and what was
    returned for it; checks the documented counts after every call."""

    def __init__(self, tg, n_rows, lib=None, dtype=torch.float32, device="cpu"):
        self.tg, self.ss = tg, tg.sessions(n_rows, _lib=lib)
        assert isinstance(self.ss, TorchGateSessions)
        self.lib, self.dtype, self.device, self.B = lib, dtype, device, n_rows
        self.x = [[] for _ in range(n_rows)]             # the current session's blocks, per row
        self.y = [[] for _ in range(n_rows)]
        self.done = []                                   # (samples, output) of every ended session

    def push(self, blocks):
        """blocks[b]: the 1-D samples row b receives (possibly empty)."""
        n = [int(v.shape[0]) for v in blocks]
        width = max(n) if n else 0
        block = torch.zeros((self.B, width), dtype=self.dtype, device=self.device)
        for b, v in enumerate(blocks):
            block[b, :n[b]] = v
        before = self.ss.samples_returned
        y, m = self.ss.push(block, n)
        assert isinstance(m, list) and y.dtype == self.dtype and y.shape == (self.B, max(m))
        for b in range(self.B):
            self.x[b].append(blocks[b])
            self.y[b].append(y[b, :m[b]])
            R = self.ss.samples_received[b]
            assert R == sum(int(v.shape[0]) for v in self.x[b])
            assert self.ss.samples_returned[b] == before[b] + m[b] == self.ss.returned_after(R)
            assert 0 <= R - self.ss.samples_returned[b] <= self.ss.latency_samples

    def end(self, rows):
        y, m = self.ss.end(rows)
        assert y.shape == (len(rows), max(m, default=0))
        for i, b in enumerate(rows):
            xs = torch.cat(self.x[b])
            out = torch.cat(self.y[b] + [y[i, :m[i]]])
            assert out.shape[0] == (xs.shape[0] // HOP) * HOP
            self.done.append((xs, out))
            self.x[b], self.y[b] = [], []
            assert self.ss.samples_received[b] == self.ss.samples_returned[b] == 0

    def reset(self, rows):
        self.ss.reset(rows)
        for b in rows:
            self.x[b], self.y[b] = [], []

    def check(self):
        """Every ended session equals tg on its own samples, in every bit."""
        assert self.done
        for xs, out in self.done:
            assert torch.equal(out, self.tg(xs[None], _lib=self.lib)[0])


def test_random_lengths_four_rows(lib):
    """Four rows, 40 pushes of seeded per-row lengths: zeros, single samples, lengths off the hop grid and pushes longer
    than the 4096-sample slice; each row one session."""
    tg = TorchGate(sr=SR, nonstationary=True)
    rng = np.random.default_rng(11)
    choices = [0, 0, 1, 1, 100, 255, 257, 320, 513, 700]
    lens = rng.choice(choices, size=(40, 4))
    lens[5, 1] = lens[17, 3] = 4097
    lens[23, 0] = 6000
    x = signal(4, int(lens.sum(0).max()) + 1, seed=3)
    d = Driver(tg, 4, lib)
    pos = [0] * 4
    for k in range(40):
        d.push([x[b, pos[b]:pos[b] + lens[k, b]] for b in range(4)])
        pos = [pos[b] + int(lens[k, b]) for b in range(4)]
    d.end([0, 1, 2, 3])
    d.check()


def test_sessions_join_and_leave(lib):
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(4, 20000, seed=5)
    e = torch.from_numpy(synth_torchgate(B=1, n=6000, seed=9)[0])
    d = Driver(tg, 4, lib)
    z = x[0, :0]
    # staggered starts: rows 1..3 begin later
    d.push([x[0, :1000], z, z, z])
    d.push([x[0, 1000:1500], x[1, :700], z, z])
    d.push([x[0, 1500:2047], x[1, 700:3000], x[2, :2048], x[3, :300]])
    # row 0 holds 2047 samples: its end is refused before any work, and no row changes
    with pytest.raises(Exception, match="x must be bigger than 2048"):
        d.ss.end([2, 0])
    assert d.ss.samples_received == [2047, 3000, 2048, 300]
    # a session of exactly 2048 samples ends while the others continue; its row is reused at once
    d.end([2])
    d.push([x[0, 2047:4000], x[1, 3000:3400], e[:900], x[3, 300:2500]])
    # row 3 is dropped without output and starts over
    d.reset([3])
    d.push([x[0, 4000:6000], x[1, 3400:9000], e[900:3300], x[3, 2500:5000]])
    d.end([1])
    d.push([x[0, 6000:6100], x[1, 9000:12000], e[3300:6000], x[3, 5000:9000]])
    d.end([3, 0, 2, 1])
    d.check()
    assert len(d.done) == 6


@pytest.mark.parametrize("kw", [dict(n_movemean_nonstationary=7), dict(n_movemean_nonstationary=1), NO_SMOOTHING,
                                dict(time_mask_smooth_ms=239), dict(prop_decrease=0.6),
                                dict(n_movemean_nonstationary=8, time_mask_smooth_ms=32)],
                         ids=["movemean7", "movemean1", "no-smoothing", "largest-nt", "prop0.6", "even-right+nt"])
def test_gate_parameters(lib, kw):
    tg = TorchGate(sr=SR, nonstationary=True, **kw)
    x = signal(2, 7000, seed=5)
    d = Driver(tg, 2, lib)
    cuts = [(0, 0), (333, 1500), (4000, 1501), (7000, 5000), (7000, 7000)]
    for (a0, a1), (b0, b1) in zip(cuts, cuts[1:]):
        d.push([x[0, a0:b0], x[1, a1:b1]])
    d.end([1, 0])
    d.check()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_precision(lib, dtype):
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(2, 7000, seed=9).to(dtype)
    d = Driver(tg, 2, lib, dtype=dtype)
    d.push([x[0, :3000], x[1, :100]])
    d.push([x[0, 3000:], x[1, 100:5000]])
    d.end([0])
    d.push([x[0, :2500], x[1, 5000:]])
    d.end([0, 1])
    d.check()


def test_equal_lengths_match_stream_and_forward(lib):
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(3, 6100, seed=2)
    ss, st = tg.sessions(3, _lib=lib), tg.stream(3, _lib=lib)
    ys, yt = [], []
    for i in range(0, 6100, 700):
        blk = x[:, i:i + 700]
        y, m = ss.push(blk, [blk.shape[1]] * 3)
        assert len(set(m)) == 1
        ys.append(y)
        yt.append(st.push(blk))
        assert torch.equal(ys[-1], yt[-1])
    ys.append(ss.end([0, 1, 2])[0])
    yt.append(st.finish())
    ss.close()
    y = torch.cat(ys, 1)
    assert torch.equal(y, torch.cat(yt, 1))
    assert torch.equal(y, tg(x, _lib=lib))


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
    size are the same after 10 pushes and after 1000, with sessions ending, being dropped and starting all along."""
    tg = TorchGate(sr=SR, nonstationary=True)
    x = signal(2, 320 * 1000, seed=1)
    ss = tg.sessions(2, _lib=lib)
    for k in range(1000):
        blk = x[:, 320 * k:320 * (k + 1)]
        ss.push(blk, [320, 160 + (k % 3) * 80])
        if k % 20 == 19:
            ss.end([k // 20 % 2])
        elif k % 40 == 25:
            ss.reset([1])
        if k == 9:
            after_10 = _heap_bytes()
    assert _heap_bytes() == after_10
    ss.close()


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
        tg.sessions(1)


@pytest.mark.parametrize("block,lengths,exc,match", [
    (torch.zeros(2, 10, dtype=torch.float64), [1, 1], NotImplementedError, "float64"),
    (torch.zeros(2, 10, requires_grad=True), [1, 1], NotImplementedError, "grad"),
    (torch.zeros(3, 10), [1, 1], ValueError, "2, n"),
    (torch.zeros(2, 10, dtype=torch.int16), [1, 1], ValueError, "float32"),
    (torch.zeros(2, 10), [1], ValueError, "entries"),
    (torch.zeros(2, 10), [1, -1], ValueError, "lengths must lie"),
    (torch.zeros(2, 10), [1, 11], ValueError, "lengths must lie"),
    (torch.zeros(2, 10), [1.0, 2.0], ValueError, "ints"),
    (torch.zeros(2, 10), [True, False], ValueError, "ints"),
    (torch.zeros(2, 10), torch.tensor([1.0, 2.0]), ValueError, "ints")])
def test_bad_pushes_before_any_handle(no_handles, block, lengths, exc, match):
    ss = TorchGate(sr=SR, nonstationary=True).sessions(2, _lib=object())
    with pytest.raises(exc, match=match):
        ss.push(block, lengths)


def test_bad_rows_and_use_after_close(lib):
    tg = TorchGate(sr=SR, nonstationary=True)
    ss = tg.sessions(3, _lib=lib)
    x = signal(3, 2500)
    ss.push(x, torch.tensor([2500, 2500, 10]))
    for rows, match in (([3], "range"), ([-1], "range"), ([0, 0], "repeat"), ([0.5], "ints")):
        with pytest.raises(ValueError, match=match):
            ss.end(rows)
        with pytest.raises(ValueError, match=match):
            ss.reset(rows)
    with pytest.raises(Exception, match="x must be bigger than 2048"):
        ss.end([0, 2])
    assert ss.samples_received == [2500, 2500, 10]
    assert ss.end([]) [1] == []
    ss.close()
    ss.close()
    for call in (lambda: ss.push(x, [1, 1, 1]), lambda: ss.end([0]), lambda: ss.reset([0])):
        with pytest.raises(ValueError, match="after close"):
            call()


def test_cuda_only_without_lib():
    ss = TorchGate(sr=SR, nonstationary=True).sessions(1)
    with pytest.raises(ValueError, match="CUDA"):
        ss.push(torch.zeros(1, 10), [10])


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


def test_cabi_error_codes(lib):
    x = signal(2, 6000).contiguous()
    y = torch.zeros(2, 8000)
    g = torch_gate(lib)
    g.tstream_begin(2)
    xp, yp = x.data_ptr(), y.data_ptr()
    # argument errors change nothing
    assert code(lambda: g.tstream_push_rows(xp, i64(10, -1), 6000, yp, 8000, 8000)) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_push_rows(xp, i64(10, 6000), 5000, yp, 8000, 8000)) == _cabi.ERR_ARG   # in_stride
    assert code(lambda: g.tstream_push_rows(xp, i64(6000, 10), 6000, yp, 8000, 10)) == _cabi.ERR_ARG     # out_capacity
    got = g.tstream_push_rows(xp, i64(3000, 2000), 6000, yp, 8000, 8000)
    assert code(lambda: g.tstream_end_rows(i64(0, 1), yp, 8000, 8000)) == _cabi.ERR_ARG                  # row 1: 2000 < 2048
    assert code(lambda: g.tstream_end_rows(i64(2), yp, 8000, 8000)) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_end_rows(i64(0, 0), yp, 8000, 8000)) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_end_rows(i64(0), yp, 8000, 1)) == _cabi.ERR_ARG
    assert code(lambda: g.tstream_reset_rows(i64(-1))) == _cabi.ERR_ARG
    # the lockstep calls are refused on a per-row stream
    assert code(lambda: g.tstream_push(xp, 10, 6000, yp, 8000, 8000)) == _cabi.ERR_STATE
    assert code(lambda: g.tstream_finish(yp, 8000, 8000)) == _cabi.ERR_STATE
    # none of the refused calls changed the stream: the rest of both rows gives tg's result
    x1 = x[:, 3000:].contiguous()
    y2 = torch.zeros(2, 8000)
    got2 = g.tstream_push_rows(x1.data_ptr(), i64(3000, 3000), 3000, y2.data_ptr(), 8000, 8000)
    yt = torch.zeros(2, 8000)
    tail = g.tstream_end_rows(i64(1, 0), yt.data_ptr(), 8000, 8000)
    tg = TorchGate(sr=SR, nonstationary=True)
    for i, b in enumerate((1, 0)):
        xs = torch.cat([x[b, :(3000, 2000)[b]], x1[b]])
        out = torch.cat([y[b, :got[b]], y2[b, :got2[b]], yt[i, :tail[i]]])
        assert torch.equal(out, tg(xs[None], _lib=lib)[0])
    g.close()


def test_cabi_mixing_and_in_stride(lib):
    g = torch_gate(lib)
    x = signal(2, 3000).contiguous()
    y = torch.zeros(2, 4000)
    g.tstream_begin(2)
    assert code(lambda: g.tstream_push_rows(x.data_ptr(), i64(10, 3001), 3000, y.data_ptr(), 4000, 4000)) == _cabi.ERR_ARG
    g.tstream_push(x.data_ptr(), 3000, 3000, y.data_ptr(), 4000, 4000)
    assert code(lambda: g.tstream_push_rows(x.data_ptr(), i64(1, 1), 3000, y.data_ptr(), 4000, 4000)) == _cabi.ERR_STATE
    assert code(lambda: g.tstream_end_rows(i64(0), y.data_ptr(), 4000, 4000)) == _cabi.ERR_STATE
    assert code(lambda: g.tstream_reset_rows(i64(0))) == _cabi.ERR_STATE
    g.tstream_finish(y.data_ptr(), 4000, 4000)
    g.tstream_begin(2)                                            # a new stream may take either kind
    g.tstream_reset_rows(i64(1))
    g.close()


# ---- H100 ---------------------------------------------------------------------------------------------------------------
def _outside_torch():
    """Device memory in use outside torch's caching allocator (the library's allocations)."""
    free, total = torch.cuda.mem_get_info()
    return total - free - torch.cuda.memory_reserved()


@pytest.mark.gpu
def test_gpu_256_rows_random_sessions_side_stream():
    """256 rows; sessions of 5-60 s start and end at random ticks; 10-30 ms jittered blocks pushed on a side stream."""
    rng = np.random.default_rng(0)
    B, ticks = 256, 3000                                          # 3000 ticks of 20 ms nominal
    tg = TorchGate(sr=SR, nonstationary=True).to("cuda")
    torch.cuda.synchronize()
    alloc0 = torch.cuda.memory_allocated()
    src = (torch.randn(B, 70 * SR, device="cuda") * 0.1 +
           torch.sin(torch.arange(70 * SR, device="cuda") * 0.05)[None]).contiguous()
    want = rng.integers(5 * SR, 60 * SR + 1, size=B)              # each row's current session length
    start = rng.integers(0, 400, size=B)                          # the tick it starts at
    got_x = [[] for _ in range(B)]
    got_y = [[] for _ in range(B)]
    pos = np.zeros(B, dtype=np.int64)
    done, ye = [], None
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        warm = tg.sessions(B)                                     # (loads the kernels this test runs)
        for i in range(8):
            idx = torch.from_numpy(np.arange(320 * i, 320 * (i + 1))[None, :].repeat(B, 0)).cuda()
            warm.push(torch.gather(src, 1, idx).contiguous(), [320] * B)
        warm.end(list(range(B)))
        warm.close()
        torch.cuda.synchronize()
        lib0 = _outside_torch()
        ss = tg.sessions(B)
        for k in range(ticks):
            n = rng.integers(160, 481, size=B)
            n[start > k] = 0
            n = np.minimum(n, want - pos)
            width = int(n.max())
            off = rng.integers(0, 70 * SR - width, size=B)
            idx = torch.from_numpy(off[:, None] + np.arange(max(width, 1))[None, :]).cuda()
            block = torch.gather(src, 1, idx)[:, :width].contiguous()
            y, m = ss.push(block, n)
            if k == 0:
                assert _outside_torch() > lib0 + B * (1 << 19)   # the stream's device state: over 0.5 MB per row
            for b in np.nonzero(n)[0]:
                got_x[b].append(block[b, :n[b]])
            for b in np.nonzero(m)[0]:
                got_y[b].append(y[b, :m[b]])
            pos += n
            ending = [int(b) for b in np.nonzero(pos >= want)[0]]
            if ending:
                ye, me = ss.end(ending)
                for i, b in enumerate(ending):
                    done.append((torch.cat(got_x[b]), torch.cat(got_y[b] + [ye[i, :me[i]]])))
                    got_x[b], got_y[b] = [], []
                    pos[b] = 0
                    want[b] = rng.integers(5 * SR, 60 * SR + 1)
                    start[b] = k + 1 + rng.integers(0, 50)
        ss.close()
        assert _outside_torch() <= lib0 + (4 << 20)              # ... released by close()
    torch.cuda.current_stream().wait_stream(side)
    assert len(done) >= B // 2
    for xs, out in done:
        assert torch.equal(out, tg(xs[None])[0])
    del done, got_x, got_y, y, ye, block, idx, src, xs, out
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() <= alloc0


@pytest.mark.gpu
def test_gpu_random_blocks_one_row():
    rng = np.random.default_rng(4)
    L = 10 * SR + 77
    x = torch.from_numpy(synth_torchgate(B=1, n=L, seed=4)).cuda()
    tg = TorchGate(sr=SR, nonstationary=True).to("cuda")
    for dtype in (torch.float32, torch.float16):
        xs = x.to(dtype)
        ss = tg.sessions(1)
        outs, i = [], 0
        while i < L:
            n = int(rng.integers(0, 2001))
            y, m = ss.push(xs[:, i:i + n], [min(n, L - i)])
            outs.append(y[0, :m[0]])
            i = min(i + n, L)
            assert ss.samples_returned[0] == ss.returned_after(i)
        outs.append(ss.end([0])[0][0])
        ss.close()
        assert torch.equal(torch.cat(outs), tg(xs)[0])
