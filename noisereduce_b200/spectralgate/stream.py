"""NoiseReduceStream -- reduce_noise() on a recording that arrives block by block (a live capture, or a file larger than
host memory read piece by piece), on libb200gate's streaming entry points (include/b200gate.h, b200gate_stream_*).

The reference needs the whole [C, N] array and writes its result to a temp-file memmap (base.py:181-187).  Its chunk
loop is local, though: output chunk i (samples [i cs, (i + 1) cs)) depends only on input [i cs - pad, (i + 1) cs + pad),
zeros outside [0, N) (base.py:130-156), and the stationary thresholds come from y_noise or from the first chunk_size
samples (stationary.py:47-81).  So a stream can return chunk i as soon as sample (i + 1) cs + pad has arrived, and what
it returns, concatenated, is bit-identical to reduce_noise() on the concatenated input.
"""
import numpy as np

from .. import _cabi
from .base import SpectralGate, samples_for_device
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
        self._gate = _cabi.Gate(**params)
        self._dtype = None                  # of the first block
        self._received = 0
        self._returned = 0
        self._closed = False
        self._clip = None                   # stationary without y_noise: the first chunk_size samples, [C, chunk_size]
        self._need_thresholds = False
        if stationary:
            if y_noise is None:
                self._need_thresholds = True
            else:                                                   # stationary.py:51-59
                noise = np.array(y_noise)
                if noise.ndim == 1:
                    noise = np.expand_dims(noise, 0)
                install_noise_thresholds(self._gate, params, noise, self._clip_to)

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
        x = np.asarray(block)
        if np.iscomplexobj(x):
            raise ValueError("Waveform must be real-valued")
        if self.n_channels is None:
            if x.ndim != 1:
                raise ValueError(f"this stream takes 1-D blocks (n_channels=None), got shape {x.shape}")
            x = x[None, :]
        elif x.ndim != 2 or x.shape[0] != self.n_channels:
            raise ValueError(f"expected a [{self.n_channels}, n] block, got shape {x.shape}")
        if self._dtype is None:
            self._dtype = x.dtype
            dev = samples_for_device(x[:, :0]).dtype
            self._gate.stream_begin(dev, x.shape[0])
        elif x.dtype != self._dtype:
            raise ValueError(f"block dtype {x.dtype} differs from the stream's dtype {self._dtype}")
        return x

    def _collect_noise(self, x):
        """Keep the first chunk_size samples; once they are all here, set the thresholds from them."""
        if self._clip is None:
            self._clip = np.empty((x.shape[0], self.chunk_size), dtype=x.dtype)
        r0 = self._received
        take = min(x.shape[1], self.chunk_size - r0)
        if take > 0:
            self._clip[:, r0:r0 + take] = x[:, :take]
        if r0 + take >= self.chunk_size:
            self._set_stream_thresholds(self.chunk_size)

    def _set_stream_thresholds(self, n):
        install_noise_thresholds(self._gate, self._params, self._clip[:, :n], self._clip_to)
        self._need_thresholds = False
        self._clip = None

    def _result(self, out, m):
        out = out[:, :m] if m > 0 else np.empty((out.shape[0], 0), out.dtype)    # (an empty result holds no buffer)
        if out.dtype != self._dtype:
            with np.errstate(invalid="ignore"):
                out = out.astype(self._dtype)                  # base.py:218-226
        return out[0] if self.n_channels is None else out

    def push(self, block):
        """Append `block` ([n_channels, n], or [n] when n_channels is None) and return the next samples of the result
        ([n_channels, m] / [m]); m = E(R + n) - E(R) is a multiple of chunk_size and may be 0."""
        x = self._rows(block)
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

    def finish(self):
        """The rest of the result (fewer than chunk_size + padding samples per channel, or the whole recording when it
        is at most chunk_size samples long); the stream is closed afterwards."""
        if self._closed:
            raise ValueError("finish() after finish(): the stream is closed")
        self._closed = True
        if self._received == 0:
            # what reduce_noise() raises on an empty recording (the reference's _amp_to_db)
            raise ValueError("zero-size array to reduction operation maximum which has no identity")
        if self._need_thresholds:                   # a recording shorter than chunk_size: thresholds from all of it
            self._set_stream_thresholds(self._received)
        dev = samples_for_device(np.empty((1, 0), self._dtype)).dtype
        C = 1 if self.n_channels is None else self.n_channels
        cap = self.chunk_size + self.padding
        out = np.empty((C, cap), dtype=dev)
        m = self._gate.stream_finish(out.ctypes.data, cap, cap)
        self._returned += m
        return self._result(out, m)
