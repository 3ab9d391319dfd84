"""TorchGate -- drop-in for noisereduce/torchgate/torchgate.py:7 on libb200gate.

Same constructor signature, attributes, registered ``smoothing_filter`` buffer (so ``state_dict``
round-trips), ``forward(x, xn)`` contract and exceptions as the reference.  The arithmetic is not
torch ops: forward() hands the tensors' device pointers to the C ABI on the current CUDA stream.
CUDA tensors only -- there is no CPU path.
"""
from typing import Optional, Union

import numpy as np
import torch

from .. import _cabi


class TorchGate(torch.nn.Module):
    @torch.no_grad()
    def __init__(
        self,
        sr: int,
        nonstationary: bool = False,
        n_std_thresh_stationary: float = 1.5,
        n_thresh_nonstationary: float = 1.3,
        temp_coeff_nonstationary: float = 0.1,
        n_movemean_nonstationary: int = 20,
        prop_decrease: float = 1.0,
        n_fft: int = 1024,
        win_length: int = None,
        hop_length: int = None,
        freq_mask_smooth_hz: float = 500,
        time_mask_smooth_ms: float = 50,
    ):
        super().__init__()
        self.sr = sr
        self.nonstationary = nonstationary
        assert 0.0 <= prop_decrease <= 1.0                                     # torchgate.py:52
        self.prop_decrease = prop_decrease
        self.n_fft = n_fft
        self.win_length = self.n_fft if win_length is None else win_length      # torchgate.py:56-58
        self.hop_length = self.win_length // 4 if hop_length is None else hop_length
        self.n_std_thresh_stationary = n_std_thresh_stationary
        self.temp_coeff_nonstationary = temp_coeff_nonstationary
        self.n_movemean_nonstationary = n_movemean_nonstationary
        self.n_thresh_nonstationary = n_thresh_nonstationary
        self.freq_mask_smooth_hz = freq_mask_smooth_hz
        self.time_mask_smooth_ms = time_mask_smooth_ms
        self._extents = (0, 0)
        self.register_buffer("smoothing_filter", self._generate_mask_smoothing_filter())
        self._gate = None

    @torch.no_grad()
    def _generate_mask_smoothing_filter(self) -> Union[torch.Tensor, None]:
        """torchgate.py:74-124: (1, 1, 2 nf + 1, 2 nt + 1) float32 buffer, or None when disabled.
        The kernels use only the extents (the taps are (n+1-|k|) / (n+1)^2)."""
        if self.freq_mask_smooth_hz is None and self.time_mask_smooth_ms is None:
            return None
        nf = 1 if self.freq_mask_smooth_hz is None else int(self.freq_mask_smooth_hz / (self.sr / (self.n_fft / 2)))
        if nf < 1:
            raise ValueError(f"freq_mask_smooth_hz needs to be at least {int((self.sr / (self.n_fft / 2)))} Hz")
        nt = 1 if self.time_mask_smooth_ms is None else int(self.time_mask_smooth_ms / ((self.hop_length / self.sr) * 1000))
        if nt < 1:
            raise ValueError(f"time_mask_smooth_ms needs to be at least {int((self.hop_length / self.sr) * 1000)} ms")
        if nt == 1 and nf == 1:
            return None
        self._extents = (nf, nt)

        def tri(n):
            k = torch.arange(-n, n + 1, dtype=torch.float32)
            return (n + 1 - k.abs()) / (n + 1)

        filt = torch.outer(tri(nf), tri(nt))[None, None]
        return filt / filt.sum()

    def _params(self):
        return (int(self.sr), bool(self.nonstationary), float(self.n_std_thresh_stationary), float(self.n_thresh_nonstationary),
                float(self.temp_coeff_nonstationary), int(self.n_movemean_nonstationary), float(self.prop_decrease),
                int(self.n_fft), int(self.win_length), int(self.hop_length))

    def _get_gate(self, lib, device, f64):
        """One library handle per (library, device, sample type, parameter values): the handle's tables live on the
        device that was current when it was created, and the reference reads its attributes on every forward."""
        key = (id(lib), str(device), bool(f64), self._params())
        if self._gate is None:
            self._gate = {}
        gate = self._gate.get(key)
        if gate is None:
            nf, nt = self._extents if self.smoothing_filter is not None else (0, 0)
            gate = _cabi.Gate(
                lib=lib, surface=_cabi.SURFACE_TORCH, stationary=0 if self.nonstationary else 1,
                n_fft=int(self.n_fft), win_length=int(self.win_length), hop_length=int(self.hop_length),
                n_grad_freq=nf, n_grad_time=nt, std_ddof=1, chunk_size=0, padding=0, sr=float(self.sr),
                prop_decrease=float(self.prop_decrease), n_std_thresh=float(self.n_std_thresh_stationary),
                top_db=40.0,                                                   # torchgate/utils.py:6
                n_movemean=int(self.n_movemean_nonstationary), thresh_n_mult=float(self.n_thresh_nonstationary),
                sigmoid_slope=1.0 / float(self.temp_coeff_nonstationary),
                path_flags=4 if f64 else 0)           # float64 input: the float64 general-geometry family (complex128 like the reference)
            # the reference's own window table (torchgate.py:231): torch.hann_window, float32
            gate.set_window(torch.hann_window(self.win_length).numpy())
            self._gate[key] = gate
        return gate

    def forward(self, x: torch.Tensor, xn: Optional[torch.Tensor] = None, lengths=None, _lib=None) -> torch.Tensor:
        """Gate the rows of x ([B, L]); xn: noise clip(s) for the stationary thresholds ([Ln], [1, Ln] or [B, Ln]).

        lengths: a zero-padded batch of rows of different lengths (one int per row, a 1-D integer tensor or a sequence).
        Row b is then gated as the signal x[b, :lengths[b]] alone: its first (lengths[b] // hop) * hop output samples
        equal forward(x[b:b+1, :lengths[b]], xn_b)[0] in every bit (xn_b = xn, or its row b when xn has B rows), the
        rest of the row is zero, samples of x past lengths[b] are never read, and the gradient past lengths[b] is zero.
        The output keeps the shape of forward(x).  2 * win_length <= lengths[b] <= L.  A CUDA tensor of lengths is
        read back to the host once, which waits for its stream; a CPU tensor or a list does not wait.  Covered: the
        default STFT geometry (n_fft = win_length = 1024, hop 256), float32 / float16 / bfloat16 x, both gates; other
        inputs raise NotImplementedError.  forward(x, lengths=[L] * B) is promised to equal forward(x) to float32
        rounding only: the last bit at synthesis work-item seams may depend on how many rows share a call."""
        assert x.ndim == 2                                                      # torchgate.py:214-220
        if x.shape[-1] < self.win_length * 2:
            raise Exception(f"x must be bigger than {self.win_length * 2}")
        assert xn is None or xn.ndim == 1 or xn.ndim == 2
        if xn is not None and xn.shape[-1] < self.win_length * 2:
            raise Exception(f"xn must be bigger than {self.win_length * 2}")
        if _lib is None and not x.is_cuda:
            raise RuntimeError("noisereduce_b200.TorchGate runs on CUDA tensors only (no CPU fallback)")
        if lengths is not None:
            lengths = self._row_lengths(x, lengths)
        if torch.is_grad_enabled() and x.requires_grad:
            # torchgate.py:223-262: the masks are built under no_grad, the gradient flows through stft -> * mask -> istft
            return _GateFunction.apply(x, self, xn, lengths, _lib)
        return self._forward_impl(x, xn, lengths, _lib)[0]

    def _tuned(self):
        return self.n_fft == 1024 and self.win_length == 1024 and self.hop_length == 256

    def _row_lengths(self, x, lengths):
        """The checked lengths= of forward() as a list of ints; raises before any library handle is made."""
        if not self._tuned():
            raise NotImplementedError("TorchGate.forward(lengths=...) needs the default STFT geometry (n_fft = win_length "
                                      f"= 1024, hop_length = 256), not n_fft={self.n_fft}, win_length={self.win_length}, "
                                      f"hop_length={self.hop_length}")
        if x.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            raise NotImplementedError(f"TorchGate.forward(lengths=...) takes float32 / float16 / bfloat16 x, not {x.dtype}")
        nf, nt = self._extents if self.smoothing_filter is not None else (0, 0)
        reason = _rows_smoothing_refusal(nf, nt, self.nonstationary)
        if reason:
            raise NotImplementedError(f"TorchGate.forward(lengths=...): freq_mask_smooth_hz={self.freq_mask_smooth_hz} / "
                                      f"time_mask_smooth_ms={self.time_mask_smooth_ms} give smoothing extents ({nf}, {nt}) "
                                      f"bins / frames, {reason}")
        if isinstance(lengths, torch.Tensor):
            if lengths.ndim != 1 or lengths.dtype.is_floating_point or lengths.dtype.is_complex or lengths.dtype == torch.bool:
                raise ValueError(f"lengths must be a 1-D integer tensor, got {tuple(lengths.shape)} {lengths.dtype}")
            lengths = lengths.tolist()                          # (a CUDA tensor: one device -> host copy)
        else:
            try:
                lengths = list(lengths)
            except TypeError:
                raise ValueError("lengths must be a 1-D integer tensor or a sequence of ints") from None
            if not all(isinstance(n, (int, np.integer)) and not isinstance(n, (bool, np.bool_)) for n in lengths):
                raise ValueError("lengths must be integers")
            lengths = [int(n) for n in lengths]
        B, L = x.shape
        if len(lengths) != B:
            raise ValueError(f"lengths has {len(lengths)} entries, x has {B} rows")
        if max(lengths) > L:
            raise ValueError(f"lengths ({max(lengths)}) beyond the {L} samples of x")
        if min(lengths) < self.win_length * 2:
            raise Exception(f"x must be bigger than {self.win_length * 2}")
        return lengths

    def _forward_impl(self, x, xn, lengths, _lib):
        f64 = x.dtype == torch.float64
        work_t, np_t = (torch.float64, np.float64) if f64 else (torch.float32, np.float32)
        ctx = torch.cuda.device(x.device) if x.is_cuda else _NullCtx()
        with ctx:
            gate = self._get_gate(_lib, x.device, f64)
            stream = torch.cuda.current_stream(x.device).cuda_stream if x.is_cuda else None
            xf = x.detach().to(work_t).contiguous()
            if xn is not None and not self.nonstationary:
                xnf = xn.detach().to(device=x.device, dtype=work_t)
                xnf = (xnf[None, :] if xnf.ndim == 1 else xnf).contiguous()
                gate.torch_set_noise(xnf.data_ptr(), xnf.shape[0], xnf.shape[1], xnf.stride(0), True, stream, dtype=np_t)
            else:
                gate.torch_set_noise(None, 0, 0, 0, True, stream)
            B, L = xf.shape
            Lo = (L // self.hop_length) * self.hop_length + (self.n_fft & 1)     # torch.istft(center=True) length
            if lengths is None:
                y = torch.empty((B, Lo), dtype=work_t, device=x.device)
                gate.run_device(xf.data_ptr(), y.data_ptr(), np_t, B, L, xf.stride(0), y.stride(0), stream)
            else:                                               # b200gate_run_rows: row b is x[b, :lengths[b]] alone
                y = torch.zeros((B, Lo), dtype=work_t, device=x.device)
                gate.run_rows(_rows(xf, y, lengths), np_t, True, stream)
            gate._fwd_serial = getattr(gate, "_fwd_serial", 0) + 1
        return y.to(dtype=x.dtype), gate                                        # torchgate.py:264

    def _ola_envelope(self, L, device):
        """sum_t w^2 of torch.istft(center=True) for T = 1 + L // hop frames, on the output's Lo samples."""
        N, H = self.n_fft, self.hop_length
        T = 1 + L // H
        w2 = torch.hann_window(self.win_length, device=device, dtype=torch.float32) ** 2
        env = torch.zeros(N + H * (T - 1), device=device, dtype=torch.float32)
        idx = (torch.arange(T, device=device) * H)[:, None] + torch.arange(N, device=device)[None, :]
        env.index_add_(0, idx.reshape(-1), w2.repeat(T))
        return env[N // 2: N // 2 + (L // H) * H]

    def _adjoint_rows(self, g, gate, serial, L, lengths, _lib):
        """_adjoint of forward(x, lengths=...): row b is the map of its own lengths[b] samples, so its envelope is
        _ola_envelope(lengths[b]) -- the single-row path's divisor -- and b200gate_torch_apply_masks_rows applies the
        forward's masks row by row.  Input samples past a row's output length get a zero gradient."""
        if getattr(gate, "_fwd_serial", 0) != serial:
            raise RuntimeError("TorchGate.backward: another forward ran on this module since the forward being "
                               "differentiated (its masks were overwritten); call backward first or use a second module")
        B, Lo = g.shape
        H = self.hop_length
        env = torch.ones((B, Lo), dtype=torch.float32, device=g.device)
        envs = {}
        for b, n in enumerate(lengths):                         # one envelope per frame count
            T = n // H
            if T not in envs:
                envs[T] = self._ola_envelope(n, g.device)
            env[b, :T * H] = envs[T]
        own = torch.arange(Lo, device=g.device)[None, :] < torch.tensor([(n // H) * H for n in lengths], device=g.device)[:, None]
        z = torch.zeros((B, L), dtype=torch.float32, device=g.device)
        z[:, :Lo] = torch.where(own, g.to(torch.float32) / env, 0.0)
        out = torch.zeros((B, Lo), dtype=torch.float32, device=g.device)
        ctx = torch.cuda.device(g.device) if g.is_cuda else _NullCtx()
        with ctx:
            stream = torch.cuda.current_stream(g.device).cuda_stream if g.is_cuda else None
            gate.torch_apply_masks_rows(_rows(z, out, lengths), np.float32, True, stream)
        grad = torch.zeros((B, L), dtype=torch.float32, device=g.device)
        grad[:, :Lo] = out * env
        return grad

    def _adjoint(self, g, gate, serial, L, _lib):
        """Gradient of forward with respect to x (masks fixed): the gate is  y = OLA(w B(w frame(x))) / env  with a
        symmetric B (a real mask between rfft and irfft), so  dL/dx = env * gate(g / env)  with the SAME masks --
        one more analysis + synthesis through b200gate_torch_apply_masks.  Input samples beyond the output length
        ((L // hop) * hop) get a zero gradient."""
        if getattr(gate, "_fwd_serial", 0) != serial:
            raise RuntimeError("TorchGate.backward: another forward ran on this module since the forward being "
                               "differentiated (its masks were overwritten); call backward first or use a second module")
        B, Lo = g.shape
        env = self._ola_envelope(L, g.device)
        z = torch.zeros((B, L), dtype=torch.float32, device=g.device)
        z[:, :Lo] = g.to(torch.float32) / env
        out = torch.empty((B, Lo), dtype=torch.float32, device=g.device)
        ctx = torch.cuda.device(g.device) if g.is_cuda else _NullCtx()
        with ctx:
            stream = torch.cuda.current_stream(g.device).cuda_stream if g.is_cuda else None
            gate.torch_apply_masks_device(z.data_ptr(), out.data_ptr(), np.float32, B, L, z.stride(0), out.stride(0), stream)
        grad = torch.zeros((B, L), dtype=torch.float32, device=g.device)
        grad[:, :Lo] = out * env
        return grad

    def stream(self, n_rows: int, _lib=None) -> "TorchGateStream":
        """Gate live audio of n_rows rows as it arrives: the non-stationary gate, bit-identical to forward() on the whole
        rows.  See TorchGateStream."""
        return TorchGateStream(self, n_rows, _lib)

    def sessions(self, n_rows: int, _lib=None) -> "TorchGateSessions":
        """Gate many live sessions in one stream of n_rows rows, each row starting, receiving samples and ending at its
        own pace: the non-stationary gate, each session bit-identical to forward() on its own samples.  See
        TorchGateSessions."""
        return TorchGateSessions(self, n_rows, _lib)


class _LiveGate:
    """What TorchGate.stream() and TorchGate.sessions() share: the refusals, the closed-form counts, the library handle
    and the checks of a block.  _api / _cls name the public call and class in messages."""
    _api, _cls = "TorchGate.stream()", "TorchGateStream"

    def __init__(self, tg: "TorchGate", n_rows: int, _lib=None):
        if not tg.nonstationary:
            raise NotImplementedError(f"{self._api} needs nonstationary=True: the stationary gate's top_db floor and "
                                      "thresholds are taken over all of a row's frames, so no sample is final before the end")
        if not tg._tuned():
            raise NotImplementedError(f"{self._api} needs the default STFT geometry (n_fft = win_length = 1024, "
                                      f"hop_length = 256), not n_fft={tg.n_fft}, win_length={tg.win_length}, "
                                      f"hop_length={tg.hop_length}")
        nf, nt = tg._extents if tg.smoothing_filter is not None else (0, 0)
        reason = _rows_smoothing_refusal(nf, nt, True)
        if reason:
            raise NotImplementedError(f"{self._api}: freq_mask_smooth_hz={tg.freq_mask_smooth_hz} / "
                                      f"time_mask_smooth_ms={tg.time_mask_smooth_ms} give smoothing extents ({nf}, {nt}) "
                                      f"bins / frames, {reason}")
        if isinstance(n_rows, bool) or not isinstance(n_rows, (int, np.integer)) or n_rows < 1:
            raise ValueError(f"n_rows must be a positive int, got {n_rows!r}")
        n = int(tg.n_movemean_nonstationary)
        if n < 1:
            raise ValueError(f"n_movemean_nonstationary must be at least 1, got {n}")
        self.n_rows = int(n_rows)
        self._gate_kw = dict(nf=nf, nt=nt, params=tg._params(), window=torch.hann_window(tg.win_length).numpy())
        self._lib = _lib
        self._hop, self._n_fft, self._win = tg.hop_length, tg.n_fft, tg.win_length
        self._right, self._nt = n - 1 - (n - 1) // 2, nt
        e = 1 if (self._right + nt) % 2 == 0 else 0
        self.latency_samples = self._n_fft // 2 + self._hop * (self._right + nt + 4 + e) - 1
        self._gate = None
        self._device = self._dtype = None

    def returned_after(self, R: int) -> int:
        """samples_returned after R samples per row (the closed form above)."""
        if R < self._n_fft // 2:
            return 0
        c = (R - self._n_fft // 2) // self._hop + 1
        nS = (c - c % 2) - 1 - self._right - self._nt
        hb = nS - nS % 2
        return self._hop * max(0, hb - 2)

    def _open(self, block):
        sr, _, _, n_thresh, temp, n_mm, prop, n_fft, win, hop = self._gate_kw["params"]
        gate = _cabi.Gate(
            lib=self._lib, surface=_cabi.SURFACE_TORCH, stationary=0, n_fft=n_fft, win_length=win, hop_length=hop,
            n_grad_freq=self._gate_kw["nf"], n_grad_time=self._gate_kw["nt"], std_ddof=1, chunk_size=0, padding=0,
            sr=float(sr), prop_decrease=prop, top_db=40.0, n_movemean=n_mm, thresh_n_mult=n_thresh,
            sigmoid_slope=1.0 / temp, path_flags=0)
        gate.set_window(self._gate_kw["window"])
        gate.tstream_begin(self.n_rows)
        self._gate = gate

    def _ctx(self):
        return torch.cuda.device(self._device) if self._device.type == "cuda" else _NullCtx()

    def _stream(self):
        return torch.cuda.current_stream(self._device).cuda_stream if self._device.type == "cuda" else None

    def _check_block(self, block):
        if not isinstance(block, torch.Tensor) or block.ndim != 2 or block.shape[0] != self.n_rows:
            shape = tuple(block.shape) if isinstance(block, torch.Tensor) else type(block).__name__
            raise ValueError(f"a block must be a [{self.n_rows}, n] tensor, got {shape}")
        if block.dtype == torch.float64:
            raise NotImplementedError(f"{self._cls}.push() takes float32 / float16 / bfloat16 blocks, not float64")
        if block.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            raise ValueError(f"a block must be float32 / float16 / bfloat16, got {block.dtype}")
        if block.requires_grad:
            raise NotImplementedError(f"{self._cls} has no backward pass: push blocks that do not require grad")
        if self._lib is None and not block.is_cuda:
            raise ValueError(f"noisereduce_b200.{self._cls} runs on CUDA tensors only (no CPU fallback)")
        if self._device is None:
            self._device, self._dtype = block.device, block.dtype
        elif block.device != self._device:
            raise ValueError(f"every block of a stream must be on {self._device}, got {block.device}")
        elif block.dtype != self._dtype:
            raise ValueError(f"every block of a stream must be {self._dtype}, got {block.dtype}")


class TorchGateStream(_LiveGate):
    """The non-stationary TorchGate on rows that arrive block by block (TorchGate.stream(n_rows)).

    push(block) takes a [n_rows, n] CUDA tensor (any n >= 0) and returns the [n_rows, m] output samples that have become
    final; finish() returns the rest.  torch.cat of everything returned, along dim 1, equals tg(x) in every bit, where x
    is the concatenation of the blocks, however x is cut into blocks.  The rows advance together.

    Every stage of the gate looks ahead a bounded distance (stft frames n_fft / 2 samples, the moving mean `right`
    frames, the smoothing nt frames, the overlap-add one window), so after R samples per row exactly
        samples_returned = hop * max(0, hb - 2),   hb = 2 floor(nS / 2),   nS = 2 floor(c / 2) - 1 - right - nt,
        c = floor((R - n_fft / 2) / hop) + 1
    have been returned (right = n - 1 - (n - 1) // 2 for n = n_movemean_nonstationary, nt the smoothing's time extent in
    frames, 0 without smoothing; frames are analysed and synthesised in pairs).  The most samples held back is
        latency_samples = n_fft / 2 + hop * (right + nt + 4 + e) - 1,   e = 1 if right + nt is even, else 0
    (4863 samples, 0.304 s, at 16 kHz with the defaults).

    push() enqueues on the current CUDA stream of the blocks' device and never waits for the device; keep the pushes of a
    stream on one CUDA stream.  The stream has its own library handle, made at the first push on that block's device and
    released by finish() (releasing it waits for the device, as destroying any handle does).  The TorchGate's attributes
    are read once, by stream().  Covered: the non-stationary gate at n_fft = win_length = 1024, hop 256, float32 /
    float16 / bfloat16 blocks (the output has the block's dtype), smoothing extents the lengths= form of forward()
    runs; other settings raise NotImplementedError, before any library handle is made."""

    def __init__(self, tg: "TorchGate", n_rows: int, _lib=None):
        super().__init__(tg, n_rows, _lib)
        self.samples_received = 0
        self.samples_returned = 0
        self._finished = False

    @torch.no_grad()
    def push(self, block: torch.Tensor) -> torch.Tensor:
        """Append block ([n_rows, n] samples of every row) and return the [n_rows, m] output samples now final."""
        if self._finished:
            raise ValueError("TorchGateStream.push() after finish()")
        self._check_block(block)
        n = block.shape[1]
        m = self.returned_after(self.samples_received + n) - self.samples_returned
        with self._ctx():
            if self._gate is None:
                self._open(block)
            y = torch.empty((self.n_rows, m), dtype=torch.float32, device=self._device)
            if n > 0:
                xf = block.detach().to(torch.float32).contiguous()
                got = self._gate.tstream_push(xf.data_ptr(), n, xf.stride(0), y.data_ptr() if m else None, max(m, 1), m,
                                              self._stream())
                assert got == m, (got, m)
        self.samples_received += n
        self.samples_returned += m
        return y.to(dtype=self._dtype)

    @torch.no_grad()
    def finish(self) -> torch.Tensor:
        """The rest of the output, [n_rows, (R // hop) * hop - samples_returned]; closes the stream."""
        if self._finished:
            raise ValueError("TorchGateStream.finish() called twice")
        R = self.samples_received
        if R < 2 * self._win:
            raise Exception(f"x must be bigger than {self._win * 2}")
        m = (R // self._hop) * self._hop - self.samples_returned
        with self._ctx():
            y = torch.empty((self.n_rows, m), dtype=torch.float32, device=self._device)
            got = self._gate.tstream_finish(y.data_ptr(), max(m, 1), m, self._stream())
            assert got == m, (got, m)
            self._gate.close()
        self._gate = None
        self._finished = True
        self.samples_returned += m
        return y.to(dtype=self._dtype)


class TorchGateSessions(_LiveGate):
    """Many live sessions in one stream (TorchGate.sessions(n_rows)): every row holds its own session, which starts,
    receives samples and ends at its own pace.

    push(block, lengths) appends block[b, :lengths[b]] to row b's session for every row b (0 <= lengths[b] <= n for a
    [n_rows, n] block) and returns (y, m): row b's new output is y[b, :m[b]], y is [n_rows, max(m)] in the block's dtype,
    m a host list.  end(rows) ends the session in each listed row and returns its tail the same way (y[i, :m[i]] for
    rows[i]); the row is then empty and its next samples start a new session.  reset(rows) drops the sessions in the
    listed rows without output.  close() releases the library handle.

    A session is the samples a row receives between its start (the creation of the object, or the end() / reset() that
    last emptied the row) and its end().  For a session x_s of at least 2 * win_length samples, the concatenation of
    everything returned for it, by pushes and by its end(), equals tg(x_s[None])[0] in every bit, however the session
    was cut, whatever the other rows did meanwhile and whichever row it used.  After R samples of a session exactly
    returned_after(R) of its output samples have been returned, and at most latency_samples are held back (the closed
    forms of TorchGateStream).  samples_received / samples_returned are those counts for each row's current session.

    push() and end() enqueue on the current CUDA stream of the blocks' device and never wait for the device, except that
    the per-row tables travel through a ring of 16 pinned slots: a call waits when the device is 16 slices behind (a push
    is one slice per 4096 samples of its longest row, an end() one).  Keep the calls of one object on one CUDA stream.
    The library handle is made at the first push; its device memory is fixed then, by n_rows and the parameters, however
    many sessions pass through.  close() waits for the device, as destroying any handle does.  Covered and refused as
    TorchGate.stream(): NotImplementedError for other settings, before any library handle is made.  ValueError, before
    any work: bad lengths (count, negative, larger than n, not integers), rows out of range or repeated, use after
    close().  end() of a row holding fewer than 2 * win_length samples raises the reference's
    Exception("x must be bigger than 2048") and changes no row."""
    _api, _cls = "TorchGate.sessions()", "TorchGateSessions"

    def __init__(self, tg: "TorchGate", n_rows: int, _lib=None):
        super().__init__(tg, n_rows, _lib)
        self._R = np.zeros(self.n_rows, dtype=np.int64)
        self._E = np.zeros(self.n_rows, dtype=np.int64)
        self._closed = False

    @property
    def samples_received(self) -> list:
        return self._R.tolist()

    @property
    def samples_returned(self) -> list:
        return self._E.tolist()

    def _returned_after_rows(self, R: np.ndarray) -> np.ndarray:
        """returned_after of every entry of R."""
        c = (R - self._n_fft // 2) // self._hop + 1
        nS = (c - c % 2) - 1 - self._right - self._nt
        hb = nS - nS % 2
        return np.where(R < self._n_fft // 2, 0, self._hop * np.maximum(0, hb - 2))

    def _live(self, what):
        if self._closed:
            raise ValueError(f"TorchGateSessions.{what}() after close()")

    def _ints(self, v, what):
        """v as a 1-D int64 numpy array (a sequence of ints or a 1-D integer tensor)."""
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().numpy()                 # (a CUDA tensor: one device -> host copy)
        try:
            a = np.asarray(v)
        except Exception:
            a = None
        if a is None or a.ndim != 1 or (a.size and a.dtype.kind not in "iu"):
            raise ValueError(f"{what} must be a 1-D sequence of ints, got {v!r}")
        return np.ascontiguousarray(a, dtype=np.int64)

    def _rows(self, rows):
        r = self._ints(rows, "rows")
        if r.size and (r.min() < 0 or r.max() >= self.n_rows):
            raise ValueError(f"rows out of range [0, {self.n_rows}): {r.tolist()}")
        if np.unique(r).size != r.size:
            raise ValueError(f"rows must not repeat, got {r.tolist()}")
        return r

    @torch.no_grad()
    def push(self, block: torch.Tensor, lengths):
        """Append block[b, :lengths[b]] to row b's session; returns (y, m), row b's new output being y[b, :m[b]]."""
        self._live("push")
        self._check_block(block)
        n = self._ints(lengths, "lengths")
        if n.size != self.n_rows:
            raise ValueError(f"lengths has {n.size} entries, the stream has {self.n_rows} rows")
        if n.size and (n.min() < 0 or n.max() > block.shape[1]):
            raise ValueError(f"lengths must lie in [0, {block.shape[1]}] (the block's samples), got {n.tolist()}")
        m = self._returned_after_rows(self._R + n) - self._E
        m_max = int(m.max())
        with self._ctx():
            if self._gate is None:
                self._open(block)
            y = torch.empty((self.n_rows, m_max), dtype=torch.float32, device=self._device)
            if n.max() > 0:
                xf = block.detach().to(torch.float32).contiguous()
                got = self._gate.tstream_push_rows(xf.data_ptr(), n, xf.stride(0), y.data_ptr() if m_max else None,
                                                   max(m_max, 1), m_max, self._stream())
                assert np.array_equal(got, m), (got, m)
        self._R += n
        self._E += m
        return y.to(dtype=self._dtype), m.tolist()

    @torch.no_grad()
    def end(self, rows):
        """End the sessions in rows; returns (y, m), the tail of rows[i] being y[i, :m[i]].  The rows are empty again."""
        self._live("end")
        r = self._rows(rows)
        short = [int(b) for b in r if self._R[b] < 2 * self._win]
        if short:
            raise Exception(f"x must be bigger than {self._win * 2}")
        m = (self._R[r] // self._hop) * self._hop - self._E[r]
        m_max = int(m.max()) if m.size else 0
        dtype = self._dtype or torch.float32
        if not r.size:
            return torch.empty((0, 0), dtype=dtype, device=self._device), []
        with self._ctx():
            y = torch.empty((r.size, m_max), dtype=torch.float32, device=self._device)
            got = self._gate.tstream_end_rows(r, y.data_ptr() if m_max else None, max(m_max, 1), m_max, self._stream())
            assert np.array_equal(got, m), (got, m)
        self._R[r] = 0
        self._E[r] = 0
        return y.to(dtype=dtype), m.tolist()

    def reset(self, rows):
        """Drop the sessions in rows without output; the rows are empty again."""
        self._live("reset")
        r = self._rows(rows)
        if self._gate is not None and r.size:
            self._gate.tstream_reset_rows(r)
        self._R[r] = 0
        self._E[r] = 0

    def close(self):
        """Release the library handle (waits for the device).  Calling it again does nothing."""
        if self._gate is not None:
            with self._ctx():
                self._gate.close()
        self._gate = None
        self._closed = True


class _GateFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, module, xn, lengths, lib):
        if not module._tuned() or x.dtype == torch.float64:
            raise NotImplementedError("noisereduce_b200.TorchGate: the backward pass exists for float32 / float16 input at the "
                                      "default STFT geometry (n_fft 1024, hop 256); use torch.no_grad() otherwise")
        y, gate = module._forward_impl(x, xn, lengths, lib)
        ctx.module, ctx.gate, ctx.lib, ctx.lengths = module, gate, lib, lengths
        ctx.serial, ctx.L, ctx.dtype = gate._fwd_serial, x.shape[-1], x.dtype
        return y

    @staticmethod
    def backward(ctx, g):
        if ctx.lengths is None:
            grad = ctx.module._adjoint(g.contiguous(), ctx.gate, ctx.serial, ctx.L, ctx.lib)
        else:
            grad = ctx.module._adjoint_rows(g.contiguous(), ctx.gate, ctx.serial, ctx.L, ctx.lengths, ctx.lib)
        return grad.to(ctx.dtype), None, None, None, None


def _rows(x, y, lengths):
    """b200gate_row tuples (in, out, n, channels = 1) for float32 rows of x and y with unit sample stride."""
    xs, ys = x.stride(0) * 4, y.stride(0) * 4
    return [(x.data_ptr() + b * xs, y.data_ptr() + b * ys, int(n), 1) for b, n in enumerate(lengths)]


def _rows_smoothing_refusal(nf, nt, nonstationary, f_pad=544, smem=200 * 1024):
    """Why the rows form cannot smooth extents (nf, nt), or None.  (1) A filter whose integer numerators outgrow 16 bits
    sends the library handle to the float64 general family, which has no rows form (big_filter in b200gate_create).
    (2) The non-stationary gate's streaming smoothing keeps a ring of 2 nt + 1 mask rows in shared memory (k_smooth_box
    for 1 <= nf <= 12, else k_smooth_stream; smoothb_smem_bytes / smooths_smem_bytes in gate_kernels.cuh)."""
    if nf > 64 or nt > 64 or (nf + 1) ** 2 * (nt + 1) ** 2 > 65535:
        return "beyond the 16-bit mask numerators of the n_fft 1024 kernels ((nf + 1)^2 (nt + 1)^2 <= 65535, at most 64 a side)"
    box = ((2 * nt + 1) * f_pad + (f_pad + 32) + (f_pad + 16)) * 4
    stream = ((2 * nt + 1) * f_pad + f_pad + 2 * nf + 8) * 4
    if nonstationary and not ((1 <= nf <= 12 and box <= smem) or stream <= smem):
        return "beyond the shared-memory ring of the non-stationary gate's smoothing"
    return None


class _NullCtx:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
