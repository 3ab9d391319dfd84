"""Host-side mirror of noisereduce/spectralgate/base.py:32 (class SpectralGate).

Same constructor arguments, attributes, defaults and exceptions as the reference; the chunk loop,
joblib fan-out and temp-file memmap (base.py:167-226) are replaced by ONE call into libb200gate,
which runs every (chunk, channel) unit of the reference's chunk table on the GPU.

Samples that are a torch CUDA tensor take the device route: they are read where they are, the result is a tensor on
the same device, and every call is enqueued on that device's current torch stream (see `SpectralGate`).  torch is never
imported here; a tensor is recognised through ``sys.modules``.
"""
import contextlib
import sys

import numpy as np

from .. import _cabi

KERNEL_DTYPES = (np.dtype(np.float32), np.dtype(np.int16), np.dtype(np.float64))


def _smoothing_filter(n_grad_freq, n_grad_time):
    """The mask-smoothing filter of base.py:7-29 as an array: outer product of the two triangles
    (n + 1 - |k|) / (n + 1), |k| <= n, normalised to unit sum.  Kept as the `_smoothing_filter` attribute for
    callers that inspect it; the kernels apply the same taps as exact integers (n + 1 - |k|)."""
    def tri(n):
        k = np.arange(-n, n + 1, dtype=np.float64)
        return (n + 1 - np.abs(k)) / (n + 1)

    filt = np.outer(tri(n_grad_freq), tri(n_grad_time))
    return filt / np.sum(filt)


def samples_for_device(y2d):
    """float32 / int16 / float64 go to the library as they are; any other dtype takes the
    reference's own route -- promoted to float64 (base.py:140) -- and is cast back on return."""
    if y2d.dtype in (np.float32, np.int16, np.float64):
        return np.ascontiguousarray(y2d)
    return np.ascontiguousarray(y2d, dtype=np.float64)


# ---- the device route: torch CUDA tensors in, torch CUDA tensors out ------------------------------------------------
def is_device_tensor(y):
    """True when `y` takes the device route: a torch tensor on a CUDA device.  (Tests on the CPU simulator library, whose
    `simulated_device` is set, send CPU tensors this way too; the product library never does.)"""
    torch = sys.modules.get("torch")
    if torch is None or not isinstance(y, torch.Tensor):
        return False
    return y.is_cuda or _cabi.library().simulated_device


def numpy_dtype_of(t):
    """The numpy dtype `t.cpu().numpy()` would have; complex raises ValueError (as the numpy route), a dtype without a
    numpy counterpart (bfloat16, ...) raises TypeError."""
    torch = sys.modules["torch"]
    if t.is_complex():
        raise ValueError("Waveform must be real-valued")
    try:
        dt = torch.empty(0, dtype=t.dtype).numpy().dtype
    except TypeError as e:
        raise TypeError(f"sample dtype {t.dtype} has no numpy counterpart: {e}") from None
    _cabi.format_code(dt)                                   # (raises TypeError for anything the kernels cannot take)
    return dt


class DeviceSite:
    """Where a device-route call runs: the tensor's device, made current with torch.cuda.device(), on that device's
    current torch stream.  Outputs are allocated there with torch.  (On the simulator: host memory, no stream.)"""

    def __init__(self, t):
        self.torch = sys.modules["torch"]
        self.device = t.device
        self.cuda = t.device.type == "cuda"

    def active(self):
        return self.torch.cuda.device(self.device) if self.cuda else contextlib.nullcontext()

    @property
    def stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream if self.cuda else None

    def empty(self, shape, np_dtype):
        tdt = self.torch.from_numpy(np.empty(0, np_dtype)).dtype
        return self.torch.empty(shape, dtype=tdt, device=self.device)

    def check_same_device(self, t, what):
        if t.device != self.device:
            raise ValueError(f"{what} is on {t.device}, the samples are on {self.device}")

    def rows(self, t):
        """[C, N] -> (tensor, row stride) the kernels read in place: rows with a unit sample stride that do not overlap
        (e.g. y[:, a:b], y[::2]).  Any other layout is copied to contiguous rows first."""
        C, N = t.shape
        if (N <= 1 or t.stride(1) == 1) and (C == 1 or t.stride(0) >= N):
            return t, (t.stride(0) if C > 1 else N)
        return t.contiguous(), N

    def kernel_rows(self, t, np_dtype):
        """rows() in a dtype the gate runs: float32 / int16 / float64 as they are, any other dtype promoted to
        float64 by b200gate_convert (the reference's base.py:140)."""
        x, stride = self.rows(t)
        if np_dtype in KERNEL_DTYPES:
            return x, stride, np_dtype
        C, N = x.shape
        x64 = self.empty((C, N), np.float64)
        _cabi.convert(_cabi.library(), _cabi.CONVERT_CAST, x.data_ptr(), np_dtype, stride, x64.data_ptr(), np.float64,
                      N, C, N, self.stream)
        return x64, N, np.dtype(np.float64)

    def cast_back(self, out, np_dtype):
        """A float64 result [C, n] (unit sample stride) in `np_dtype` with ndarray.astype's rules (base.py:218-226);
        results already in `np_dtype` are returned as they are."""
        if out.dtype == self.torch.from_numpy(np.empty(0, np_dtype)).dtype:
            return out
        C, n = out.shape
        res = self.empty((C, n), np_dtype)
        _cabi.convert(_cabi.library(), _cabi.CONVERT_CAST, out.data_ptr(), np.float64, out.stride(0) if C > 1 else n,
                      res.data_ptr(), np_dtype, n, C, n, self.stream)
        return res


class SpectralGate:
    """``y`` is a numpy array (or anything np.asarray takes, CPU tensors included), or a torch CUDA tensor.

    A CUDA tensor takes the device route: the handles are created and run under ``torch.cuda.device(y.device)``, every
    step is enqueued on ``torch.cuda.current_stream(y.device)``, and get_traces() returns a tensor allocated there, with
    the numpy route's shape and dtype and the same bits as ``get_traces()`` on ``y.cpu().numpy()``.  Rows with a unit
    sample stride are read in place; other layouts are copied to contiguous rows.  float32 / int16 / float64 go to the
    kernels as they are; every other real dtype numpy knows is promoted to float64 on the device and the result cast
    back with ndarray.astype's rules (b200gate_convert); bfloat16 and other dtypes without a numpy counterpart raise
    TypeError.  The per-chunk plugin points (`_read_chunk`, `filter_chunk`, `_do_filter`) stay numpy-only.

    Where the host waits: get_traces() only enqueues its work (its first call may allocate the library's workspace,
    and device allocation can itself wait).  Three steps wait for the whole device, not just the current stream.  The
    stationary threshold computation reads the per-bin statistics back and frees its scratch buffers, as on the numpy
    route.  A noise clip shorter than the window is handled by a second handle, which is destroyed at once.  Destroying
    a handle, when the object is freed, synchronises the device before its buffers are released or cached.
    reduce_noise() builds the object, calls get_traces() and drops the object, so it returns only once the device is
    idle, including work on other streams.  A caller who wants the result still in flight keeps the object and calls
    get_traces().
    """

    def __init__(
        self,
        y,
        sr,
        prop_decrease,
        chunk_size,
        padding,
        n_fft,
        win_length,
        hop_length,
        time_constant_s,
        freq_mask_smooth_hz,
        time_mask_smooth_ms,
        tmp_folder,
        use_tqdm,
        n_jobs,
    ):
        self.sr = sr
        self.flat = False
        self._site = None
        if is_device_tensor(y):
            self._site = DeviceSite(y)
            self._dtype = numpy_dtype_of(y)
            empty = y.numel() == 0
        else:
            y = np.asarray(y)          # (the reference copies with np.array; nothing here writes to the caller's samples)
            if np.iscomplexobj(y):
                # the reference fails inside scipy / numpy broadcasting on complex samples (a ValueError); fail before the device
                raise ValueError("Waveform must be real-valued")
            self._dtype = y.dtype
            empty = y.size == 0
        if empty:
            raise ValueError("zero-size array to reduction operation maximum which has no identity")     # what the reference's _amp_to_db raises
        # reshape data to (#channels, #frames)                      (base.py:54-62)
        if len(y.shape) == 1:
            self.y = y[None, :]
            self.flat = True
        elif len(y.shape) > 2:
            raise ValueError("Waveform must be in shape (# frames, # channels)")
        else:
            self.y = y
        self.n_channels, self.n_frames = self.y.shape
        self._chunk_size = chunk_size
        self.padding = padding
        # accepted for signature compatibility; the GPU grid replaces joblib / tqdm / the temp memmap
        self.n_jobs = n_jobs
        self.use_tqdm = use_tqdm
        self._tmp_folder = tmp_folder

        self._n_fft = n_fft
        self._win_length = self._n_fft if win_length is None else win_length          # base.py:79-86
        self._hop_length = self._win_length // 4 if hop_length is None else hop_length
        self._time_constant_s = time_constant_s
        self._prop_decrease = prop_decrease

        self._n_grad_freq = 0
        self._n_grad_time = 0
        if (freq_mask_smooth_hz is None) & (time_mask_smooth_ms is None):               # base.py:92-97
            self.smooth_mask = False
        else:
            self._generate_mask_smoothing_filter(freq_mask_smooth_hz, time_mask_smooth_ms)
        self._gate = None
        self._unit_gate = None

    def _generate_mask_smoothing_filter(self, freq_mask_smooth_hz, time_mask_smooth_ms):
        """base.py:99-128 -- same integer arithmetic and the same ValueErrors.  Only the extents are
        kept: the taps are the rationals (n+1-|k|)/(n+1)^2 and the kernels apply them in integers."""
        if freq_mask_smooth_hz is None:
            n_grad_freq = 1
        else:
            n_grad_freq = int(freq_mask_smooth_hz / (self.sr / (self._n_fft / 2)))
            if n_grad_freq < 1:
                raise ValueError(
                    "freq_mask_smooth_hz needs to be at least {}Hz".format(int((self.sr / (self._n_fft / 2))))
                )
        if time_mask_smooth_ms is None:
            n_grad_time = 1
        else:
            n_grad_time = int(time_mask_smooth_ms / ((self._hop_length / self.sr) * 1000))
            if n_grad_time < 1:
                raise ValueError(
                    "time_mask_smooth_ms needs to be at least {}ms".format(int((self._hop_length / self.sr) * 1000))
                )
        if (n_grad_time == 1) & (n_grad_freq == 1):
            self.smooth_mask = False
        else:
            self.smooth_mask = True
            self._n_grad_freq, self._n_grad_time = n_grad_freq, n_grad_time
            self._smoothing_filter = _smoothing_filter(n_grad_freq, n_grad_time)

    # -- parameters handed to the C ABI ------------------------------------------------------------
    def _gate_params(self):
        return dict(
            surface=_cabi.SURFACE_NUMPY,
            n_fft=int(self._n_fft),
            win_length=int(self._win_length),
            hop_length=int(self._hop_length),
            n_grad_freq=int(self._n_grad_freq) if self.smooth_mask else 0,
            n_grad_time=int(self._n_grad_time) if self.smooth_mask else 0,
            chunk_size=int(self._chunk_size) if self._chunk_size is not None else 0,
            padding=int(self.padding),
            sr=float(self.sr),
            prop_decrease=float(self._prop_decrease),
            top_db=80.0,                     # spectralgate/utils.py:11
            std_ddof=0,
        )

    def _samples_for_device(self, y2d):
        return samples_for_device(y2d)

    def _run(self, y2d, lo=0, hi=None):
        """One library call; returns columns [lo, hi) of the (partially written) output rows."""
        x = self._samples_for_device(y2d)
        out = self._gate.run_host(x)[:, lo:hi]
        if out.dtype != self._dtype:
            with np.errstate(invalid="ignore"):
                out = out.astype(self._dtype)                  # base.py:218-226
        return out

    def _run_device(self, lo, hi, w_lo, w_hi):
        """The device route's library call: the run writes columns [w_lo, w_hi) (set_range's span) densely into a
        [C, w_hi - w_lo] slab addressed through the virtual base slab - w_lo; returns columns [lo, hi) of it."""
        site = self._site
        x, stride, kdt = site.kernel_rows(self.y, self._dtype)
        C, N = x.shape
        slab = site.empty((C, w_hi - w_lo), kdt)
        self._gate.run_device(x.data_ptr(), slab.data_ptr() - w_lo * kdt.itemsize, kdt, C, N, stride, w_hi - w_lo,
                              site.stream)
        return site.cast_back(slab[:, lo - w_lo: hi - w_lo], self._dtype)

    # -- the reference's per-chunk plugin point (base.py:130-160); numpy arrays only, also on the device route -------
    def _read_chunk(self, i1, i2):
        """base.py:130-142: the span [i1, i2) of every channel as float64, zeros outside the recording.  numpy only:
        not available when the samples are a CUDA tensor."""
        lo, hi = max(i1, 0), min(i2, self.n_frames)
        chunk = np.zeros((self.n_channels, i2 - i1))
        chunk[:, lo - i1: hi - i1] = self.y[:, lo:hi]
        return chunk

    def filter_chunk(self, start_frame, end_frame):
        """base.py:144-150: pad by `padding` on both sides, filter, return the centre.  numpy only (see _read_chunk)."""
        i1, i2 = start_frame - self.padding, end_frame + self.padding
        filtered = self._do_filter(self._read_chunk(i1, i2))
        return filtered[:, start_frame - i1: end_frame - i1]

    def _get_filtered_chunk(self, ind):
        """base.py:152-156."""
        return self.filter_chunk(start_frame=ind * self._chunk_size, end_frame=(ind + 1) * self._chunk_size)

    def _unit_gate_params(self):
        """Parameters of the gate that filters ONE already padded chunk (chunk_size <= 0 and padding = 0 make the
        library treat its whole input as the single unit of stationary.py:83-127 / nonstationary.py:47-97)."""
        raise NotImplementedError

    def _do_filter(self, chunk):
        """base.py:158-160 / stationary.py:129 / nonstationary.py:99: filter one padded chunk [C, Lp]; the result has
        the chunk's shape and dtype, its first (Lp // hop) * hop columns filled.  One library call on a second handle
        that shares this gate's statistics.  Takes and returns numpy arrays only, whichever route the recording took."""
        chunk = np.asarray(chunk)
        if self._unit_gate is None:
            self._unit_gate = _cabi.Gate(**self._unit_gate_params())
            self._prepare_unit_gate(self._unit_gate)
        x = self._samples_for_device(chunk)
        out = self._unit_gate.run_host(x)
        return out if out.dtype == chunk.dtype else out.astype(chunk.dtype)

    def _prepare_unit_gate(self, gate):
        pass

    def get_traces(self, start_frame=None, end_frame=None):
        """base.py:167-226.  With both bounds None this is the whole recording (what reduce_noise
        calls).  A sub-range runs only the units the reference would: the chunks
        int(start/cs)..int((end-1)/cs) of the grid anchored at sample 0 when the range is longer
        than chunk_size (base.py:175-217), else ONE padded chunk covering [0, end_frame) whose
        padding is read from the recording (base.py:222 -- start_frame is ignored there, as in
        the reference).  On the device route the result is a tensor on the samples' device."""
        if start_frame is None:
            start_frame = 0
        if end_frame is None:
            end_frame = self.n_frames
        if self._chunk_size is not None and end_frame - start_frame > self._chunk_size:
            # the reference's memmap has end-start columns; a range past the recording fails there too
            if start_frame < 0 or end_frame > self.n_frames:
                raise ValueError("start_frame / end_frame outside the recording")
            first, last = int(start_frame / self._chunk_size), int((end_frame - 1) / self._chunk_size)
            self._gate.set_range(1, first, last)
            lo = start_frame
            span = (first * self._chunk_size, min(self.n_frames, (last + 1) * self._chunk_size))
        else:
            if not 0 < end_frame <= self.n_frames:
                raise ValueError("end_frame outside the recording")
            self._gate.set_range(2, int(end_frame))
            lo = 0
            span = (0, int(end_frame))
        try:
            if self._site is None:
                res = self._run(self.y, lo, end_frame)
            else:
                with self._site.active():
                    res = self._run_device(lo, end_frame, *span)
        finally:
            self._gate.set_range(0)
        return res.flatten() if self.flat else res

    def _on_device(self):
        """Context of the handle calls: the samples' CUDA device on the device route, nothing otherwise."""
        return contextlib.nullcontext() if self._site is None else self._site.active()
