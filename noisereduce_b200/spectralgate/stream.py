"""NoiseReduceStream -- reduce_noise() on a recording that arrives block by block (a live capture, or a file larger than
host memory read piece by piece), on libb200gate's streaming entry points (include/b200gate.h, b200gate_stream_*).

The reference needs the whole [C, N] array and writes its result to a temp-file memmap (base.py:181-187).  Its chunk
loop is local, though: output chunk i (samples [i cs, (i + 1) cs)) depends only on input [i cs - pad, (i + 1) cs + pad),
zeros outside [0, N) (base.py:130-156), and the stationary thresholds come from y_noise or from the first chunk_size
samples (stationary.py:47-81).  So a stream can return chunk i as soon as sample (i + 1) cs + pad has arrived, and what
it returns, concatenated, is bit-identical to reduce_noise() on the concatenated input.
"""
import contextlib
import sys

import numpy as np

from .. import _cabi
from .base import KERNEL_DTYPES, DeviceSite, SpectralGate, is_device_tensor, numpy_dtype_of, samples_for_device
from .stationary import install_noise_thresholds


class NoiseReduceStream:
    """Denoise a recording block by block::

        s = NoiseReduceStream(sr=48000, n_channels=64, stationary=True)
        for block in blocks:            # [64, n], any n >= 0; one dtype for the whole stream
            out = s.push(block)         # [64, m]: the next m samples of the result, m a multiple of chunk_size
        out = s.finish()                # the rest; the stream is then closed

    The arguments are reduce_noise()'s gate arguments, with its defaults and its ValueErrors, plus ``n_channels``
    (None: 1-D blocks and outputs, like flat input to reduce_noise).  If y is the concatenation of every pushed block
    (N samples), the concatenation of every push() result and the finish() result equals ``reduce_noise(y, sr, ...)``
    with the same arguments: shape, dtype and every bit.

    Emission rule: once R samples have been pushed in total, exactly E(R) have been returned, where
    ``E(R) = chunk_size * max(0, (R - padding) // chunk_size)`` if R > chunk_size, else 0.  A chunk is returned as soon
    as its padded span has arrived, so the latency is at most chunk_size + padding - 1 samples.  A recording of
    N <= chunk_size samples is one padded chunk in reduce_noise(); that is only known at the end, so such a stream
    returns everything from finish().

    float32, int16 and float64 blocks go to the GPU as they are; any other real dtype is promoted to float64 per block
    and the result cast back, as reduce_noise() does.  The stationary gate without y_noise takes its thresholds from the
    first min(N, chunk_size) samples of the stream (clip_noise_stationary=True, reduce_noise()'s default).

    Blocks may be torch CUDA tensors; push() and finish() then return CUDA tensors on the same device, with the same
    bits.  Each push only enqueues work on the device's current torch stream (b200gate_stream_push with device pointers),
    except the one that completes the stationary noise clip, which is collected on the device and whose statistics are
    read back (the host waits for that stream).  Each returned tensor holds exactly its own samples; a push that returns
    nothing returns an empty tensor without storage.  The first block fixes the memory space and the device: a later
    block from the other memory space or another device raises ValueError.  y_noise may be a host array (its statistics
    are computed as reduce_noise() does) or a CUDA tensor on the blocks' device.  Host waits for the whole device: the
    handle's destruction (when the stream object is freed) synchronises the device before it releases its buffers, and
    so does the one-time remaking of the handle on the first CUDA block's device when it was made on another device,
    or before torch had initialised CUDA.

    The device holds a window of about 2 * padding + chunk_size samples per channel plus one slice of input, whatever
    the stream length or block sizes.  Not supported: chunk_size=None (the whole recording is one unit, so nothing could
    be returned early) and the stationary gate with clip_noise_stationary=False and no y_noise (its thresholds need the
    whole recording); both raise ValueError, as do blocks whose channel count or dtype differ from the first block and a
    push() after finish().  The torch route (use_torch), TorchGate and multi-GPU streaming are not covered.
    """

    def __init__(self, sr, n_channels=None, stationary=False, y_noise=None, prop_decrease=1.0, time_constant_s=2.0,
                 freq_mask_smooth_hz=500, time_mask_smooth_ms=50, thresh_n_mult_nonstationary=2,
                 sigmoid_slope_nonstationary=10, n_std_thresh_stationary=1.5, chunk_size=600000, padding=30000,
                 n_fft=1024, win_length=None, hop_length=None, clip_noise_stationary=True):
        if chunk_size is None:
            raise ValueError("NoiseReduceStream needs a chunk_size: with chunk_size=None the whole recording is one "
                             "unit and nothing can be returned before the end")
        if stationary and y_noise is None and not clip_noise_stationary:
            raise ValueError("NoiseReduceStream: the stationary gate with clip_noise_stationary=False takes its "
                             "thresholds from the whole recording; pass y_noise or clip_noise_stationary=True")
        if n_channels is not None and int(n_channels) < 1:
            raise ValueError("n_channels must be >= 1 (or None for 1-D blocks)")
        # reduce_noise()'s argument resolution (defaults, smoothing extents, errors), as the offline classes do it
        geo = SpectralGate(np.zeros(1, np.float32), sr, prop_decrease, chunk_size, padding, n_fft, win_length,
                           hop_length, time_constant_s, freq_mask_smooth_hz, time_mask_smooth_ms, None, False, 1)
        params = geo._gate_params()
        if stationary:
            params.update(stationary=1, n_std_thresh=float(n_std_thresh_stationary),
                          clip_noise=1 if clip_noise_stationary else 0)
        else:
            params.update(stationary=0, time_constant_s=float(time_constant_s),
                          thresh_n_mult=float(thresh_n_mult_nonstationary),
                          sigmoid_slope=float(sigmoid_slope_nonstationary))
        self.sr = sr
        self.n_channels = None if n_channels is None else int(n_channels)
        self.stationary = bool(stationary)
        self.chunk_size, self.padding = int(chunk_size), int(padding)
        self._params = params
        self._clip_to = self.chunk_size if clip_noise_stationary else None
        self._dtype = None                  # of the first block
        self._kdt = None                    # the dtype the gate runs: the first block's, or float64 (promoted)
        self._site = None                   # CUDA-tensor blocks: their device (fixed by the first block)
        self._received = 0
        self._returned = 0
        self._closed = False
        self._clip = None                   # stationary without y_noise: the first chunk_size samples, [C, chunk_size]
        self._need_thresholds = False
        self._thresh = None                 # thresholds from y_noise, kept for a handle remade on the blocks' device
        self._gate_device = None            # the CUDA device the handle was created on, where known
        noise = None
        if stationary and y_noise is None:
            self._need_thresholds = True
        elif stationary:                                            # stationary.py:51-59
            if is_device_tensor(y_noise):
                self._site = DeviceSite(y_noise)                    # the blocks must then be on y_noise's device
                noise = y_noise
            else:
                noise = np.array(y_noise)
            noise = noise[None, :] if noise.ndim == 1 else noise
        torch = sys.modules.get("torch")
        if self._site is not None:
            self._gate_device = self._site.device
        elif torch is not None and torch.cuda.is_initialized():
            self._gate_device = torch.device("cuda", torch.cuda.current_device())
        # The handle is made here, so that the library's argument checks and y_noise's errors (a clip too short for
        # the window) are raised by the constructor, as reduce_noise() raises them.
        with self._on_device():
            self._gate = _cabi.Gate(**params)
            if noise is not None:
                self._thresh = install_noise_thresholds(self._gate, params, noise, self._clip_to, self._stream())[2]

    def _on_device(self):
        return contextlib.nullcontext() if self._site is None else self._site.active()

    def _stream(self):
        return None if self._site is None else self._site.stream

    # -- emission rule --------------------------------------------------------------------------------------------
    def emitted(self, received=None):
        """E(R): how many samples have been returned once R (default: all pushed so far) have been received."""
        R = self._received if received is None else int(received)
        cs = self.chunk_size
        return cs * max(0, (R - self.padding) // cs) if R > cs else 0

    @property
    def samples_received(self):
        return self._received

    @property
    def samples_returned(self):
        return self._returned

    # -- blocks ------------------------------------------------------------------------------------------------------
    def _rows(self, block):
        if self._closed:
            raise ValueError("push() after finish(): the stream is closed")
        on_device = is_device_tensor(block)
        if self._dtype is not None and on_device != (self._site is not None):
            raise ValueError("a stream's blocks stay in the memory space of its first block (CUDA tensors or host arrays)")
        if on_device:
            x, dt = block, numpy_dtype_of(block)
            if self._site is not None:
                self._site.check_same_device(x, "this block")
        else:
            x = np.asarray(block)
            if np.iscomplexobj(x):
                raise ValueError("Waveform must be real-valued")
            dt = x.dtype
        if self.n_channels is None:
            if x.ndim != 1:
                raise ValueError(f"this stream takes 1-D blocks (n_channels=None), got shape {tuple(x.shape)}")
            x = x[None, :]
        elif x.ndim != 2 or x.shape[0] != self.n_channels:
            raise ValueError(f"expected a [{self.n_channels}, n] block, got shape {tuple(x.shape)}")
        if self._dtype is None:
            if on_device:
                self._bind_device(x)
            elif self._site is not None:
                raise ValueError("y_noise is a CUDA tensor: the stream's blocks must be CUDA tensors on its device")
            self._dtype = dt
            self._kdt = dt if dt in KERNEL_DTYPES else np.dtype(np.float64)
            with self._on_device():
                self._gate.stream_begin(self._kdt, x.shape[0])
        elif dt != self._dtype:
            raise ValueError(f"block dtype {dt} differs from the stream's dtype {self._dtype}")
        return x

    def _bind_device(self, x):
        """The first block is a CUDA tensor: the stream runs on its device.  A handle made on another device, or on one
        that is not known (torch had not initialised CUDA when the stream was constructed), is remade there once, with
        y_noise's thresholds copied over rather than recomputed; closing the old handle waits for the device."""
        if self._site is None:
            self._site = DeviceSite(x)
        if self._site.cuda and self._gate_device != self._site.device:
            self._gate.close()
            with self._site.active():
                self._gate = _cabi.Gate(**self._params)
                if self._thresh is not None:
                    self._gate.set_noise_threshold(self._thresh)
        self._gate_device = self._site.device

    def _collect_noise(self, x):
        """Keep the first chunk_size samples; once they are all here, set the thresholds from them.  CUDA-tensor blocks
        are collected on their device."""
        if self._clip is None:
            if self._site is None:
                self._clip = np.empty((x.shape[0], self.chunk_size), dtype=x.dtype)
            else:
                self._clip = self._site.empty((x.shape[0], self.chunk_size), self._dtype)
        r0 = self._received
        take = min(x.shape[1], self.chunk_size - r0)
        if take > 0:
            self._clip[:, r0:r0 + take] = x[:, :take]
        if r0 + take >= self.chunk_size:
            self._set_stream_thresholds(self.chunk_size)

    def _set_stream_thresholds(self, n):
        install_noise_thresholds(self._gate, self._params, self._clip[:, :n], self._clip_to, self._stream())
        self._need_thresholds = False
        self._clip = None

    def _result(self, out, m):
        if self._site is not None:
            # Device memory is committed when allocated: a result holds its own m columns only, never the push's whole
            # [C, n + chunk_size] output buffer (callers keep many results to concatenate them).
            if m == 0:
                out = self._site.empty((out.shape[0], 0), self._dtype)
            elif self._kdt == self._dtype:
                out = out[:, :m].clone(memory_format=self._site.torch.contiguous_format)
            else:
                out = self._site.cast_back(out[:, :m], self._dtype)     # (a new [C, m] tensor)
            return out[0] if self.n_channels is None else out
        out = out[:, :m] if m > 0 else np.empty((out.shape[0], 0), out.dtype)    # (an empty result holds no buffer)
        if out.dtype != self._dtype:
            with np.errstate(invalid="ignore"):
                out = out.astype(self._dtype)                  # base.py:218-226
        return out[0] if self.n_channels is None else out

    def push(self, block):
        """Append `block` ([n_channels, n], or [n] when n_channels is None) and return the next samples of the result
        ([n_channels, m] / [m]); m = E(R + n) - E(R) is a multiple of chunk_size and may be 0.  A CUDA tensor block
        returns a CUDA tensor; the call only enqueues work on the device's current torch stream, except when it
        completes the stationary noise clip (the thresholds are read back once)."""
        x = self._rows(block)
        if self._site is not None:
            with self._site.active():
                return self._push_device(x)
        if self._need_thresholds:
            self._collect_noise(x)
        C, n = x.shape
        es = x.dtype.itemsize
        if C > 1 and x.dtype in (np.float32, np.int16, np.float64) and x.strides[1] == es and x.strides[0] % es == 0 \
                and x.strides[0] >= n * es:
            xd, stride = x, x.strides[0] // es      # rows with contiguous samples (e.g. y[:, i:j]) are read in place
        else:
            xd, stride = samples_for_device(x), n
        cap = n + self.chunk_size
        out = np.empty((C, cap), dtype=xd.dtype)       # (pages past the returned columns are never touched)
        m = self._gate.stream_push(xd.ctypes.data, n, stride, False, out.ctypes.data, cap, cap)
        self._received += n
        self._returned += m
        return self._result(out, m)

    def _push_device(self, x):
        site = self._site
        if self._need_thresholds:
            self._collect_noise(x)
        C, n = x.shape
        ptr, stride = None, 0
        if n > 0:
            xd, stride, _ = site.kernel_rows(x, self._dtype)
            ptr = xd.data_ptr()
        cap = n + self.chunk_size
        out = site.empty((C, cap), self._kdt)
        m = self._gate.stream_push(ptr, n, stride, True, out.data_ptr(), cap, cap, site.stream)
        self._received += n
        self._returned += m
        return self._result(out, m)

    def finish(self):
        """The rest of the result (fewer than chunk_size + padding samples per channel, or the whole recording when it
        is at most chunk_size samples long); the stream is closed afterwards."""
        if self._closed:
            raise ValueError("finish() after finish(): the stream is closed")
        self._closed = True
        if self._received == 0:
            # what reduce_noise() raises on an empty recording (the reference's _amp_to_db)
            raise ValueError("zero-size array to reduction operation maximum which has no identity")
        C = 1 if self.n_channels is None else self.n_channels
        cap = self.chunk_size + self.padding
        with self._on_device():
            if self._need_thresholds:               # a recording shorter than chunk_size: thresholds from all of it
                self._set_stream_thresholds(self._received)
            if self._site is None:
                out = np.empty((C, cap), dtype=self._kdt)
                m = self._gate.stream_finish(out.ctypes.data, cap, cap)
            else:
                out = self._site.empty((C, cap), self._kdt)
                m = self._gate.stream_finish(out.data_ptr(), cap, cap, self._site.stream)
            self._returned += m
            return self._result(out, m)
