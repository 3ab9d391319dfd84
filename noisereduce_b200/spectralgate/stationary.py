"""Mirror of noisereduce/spectralgate/stationary.py:7 (SpectralGateStationary) on libb200gate."""
import numpy as np

from .. import _cabi
from .base import KERNEL_DTYPES, DeviceSite, SpectralGate, is_device_tensor, numpy_dtype_of, samples_for_device


class SpectralGateStationary(SpectralGate):
    def __init__(
        self,
        y,
        sr,
        y_noise,
        n_std_thresh_stationary,
        chunk_size,
        clip_noise_stationary,
        padding,
        n_fft,
        win_length,
        hop_length,
        time_constant_s,
        freq_mask_smooth_hz,
        time_mask_smooth_ms,
        tmp_folder,
        prop_decrease,
        use_tqdm,
        n_jobs,
    ):
        super().__init__(
            y=y, sr=sr, chunk_size=chunk_size, padding=padding, n_fft=n_fft, win_length=win_length,
            hop_length=hop_length, time_constant_s=time_constant_s, freq_mask_smooth_hz=freq_mask_smooth_hz,
            time_mask_smooth_ms=time_mask_smooth_ms, tmp_folder=tmp_folder, prop_decrease=prop_decrease,
            use_tqdm=use_tqdm, n_jobs=n_jobs,
        )
        self.n_std_thresh_stationary = n_std_thresh_stationary

        if y_noise is None:                                     # stationary.py:47-59
            noise = self.y
        else:
            if self._site is not None and is_device_tensor(y_noise):
                self._site.check_same_device(y_noise, "y_noise")     # a CUDA y_noise on y's device is read in place
            else:
                y_noise = np.array(y_noise)                          # host statistics, as on the numpy route
            if len(y_noise.shape) == 1:
                noise = y_noise[None, :]
            elif len(y.shape) > 2:
                raise ValueError("Waveform must be in shape (# frames, # channels)")
            else:
                noise = y_noise

        self._noise2d, self._clip_noise = noise, bool(clip_noise_stationary)
        params = self._gate_params()
        params.update(stationary=1, n_std_thresh=float(n_std_thresh_stationary),
                      clip_noise=1 if clip_noise_stationary else 0)
        self._params = params
        with self._on_device():
            self._gate = _cabi.Gate(**params)
            self.mean_freq_noise, self.std_freq_noise, self.noise_thresh = install_noise_thresholds(
                self._gate, params, noise, self._chunk_size if clip_noise_stationary else None,
                None if self._site is None else self._site.stream)

    def _unit_gate_params(self):
        p = dict(self._params)
        p.update(chunk_size=0, padding=0)
        return p

    def _prepare_unit_gate(self, gate):
        gate.set_noise_threshold(self.noise_thresh)          # the thresholds of the whole recording (stationary.py:79-81)

    @property
    def y_noise(self):
        """The collapsed noise clip the reference keeps as an attribute (stationary.py:61-64): channel mean in
        the input dtype, clipped to chunk_size.  Computed on demand -- the thresholds come from the device.  A CUDA
        tensor clip is copied to the host here, and its mean taken over the row-major copy (see
        install_noise_thresholds)."""
        n = self._noise2d[:, : self._chunk_size] if self._clip_noise else self._noise2d
        if not isinstance(n, np.ndarray):
            n = np.ascontiguousarray(n.cpu().numpy())
        return np.mean(n, axis=0)


def install_noise_thresholds(gate, params, noise, clip_to, stream=None):
    """stationary.py:61-81 on the device: channel mean in the input dtype, clip to `clip_to` samples (chunk_size when
    clip_noise_stationary, else None), STFT, dB with the 80 dB floor, per-bin mean / std over time, threshold.  `noise`
    is [C, n], a host array or a device tensor (read where it is, on `stream`); `gate` is a stationary handle created
    from `params`, which receives the thresholds.  Returns (mean, std, threshold) per bin, as host arrays.

    The channel mean of a float16, integer or bool clip follows np.mean's dtype rules (stationary.py:61).  For a host
    array numpy computes it; for a device tensor b200gate_convert does, summing in channel order.  numpy sums pairwise
    instead when the channels are adjacent in memory (a Fortran-order clip), which can differ from the channel-order
    sum once there are 8 or more channels: for such layouts the device route's result is that of the row-major copy of the
    clip.  The statistics are read back to the host and the library's scratch buffers freed, so the host waits for the
    device.  A clip shorter than the window is handled by a second handle, whose destruction also waits."""
    on_device = not isinstance(noise, np.ndarray)
    if on_device:
        site = DeviceSite(noise)
        dt = numpy_dtype_of(noise)
        noise, stride = site.rows(noise)
    clip = noise
    if not on_device and noise.dtype not in KERNEL_DTYPES:
        # the reference collapses the clip with np.mean in the clip's own dtype rules (stationary.py:61): float16 stays
        # float16 (float32 accumulation, rounded), integers / bool become float64 -- numpy decides, the device gets the result
        clip = np.mean(noise, axis=0)[None, :]
        if clip.dtype not in (np.float32, np.float64):
            clip = clip.astype(np.float32)
    n_eff = clip.shape[1]
    if clip_to is not None:
        n_eff = min(n_eff, int(clip_to))                                      # stationary.py:63-64
    if on_device and dt not in KERNEL_DTYPES:
        # the same collapse on the device: float64 [1, n_eff] (a float16 mean widens exactly)
        mean64 = site.empty((1, n_eff), np.float64)
        _cabi.convert(gate.lib, _cabi.CONVERT_CHANNEL_MEAN, clip.data_ptr(), dt, stride, mean64.data_ptr(), np.float64,
                      n_eff, clip.shape[0], n_eff, stream)
        clip, stride, dt = mean64, n_eff, np.dtype(np.float64)

    def stats(g, n):
        if on_device:
            g.noise_stats_device(clip.data_ptr(), dt, clip.shape[0], n, stride, stream)
        else:
            g.noise_stats_host(samples_for_device(clip[:, :n]), stream)

    win_length, hop_length = params["win_length"], params["hop_length"]
    noverlap = win_length - hop_length
    if n_eff < win_length:
        # scipy.signal.stft on a clip shorter than the window shrinks the window to the clip (nperseg = len(x), with a
        # warning) and then insists on noverlap < nperseg; the reference inherits both behaviours (stationary.py:67-73)
        if noverlap >= n_eff:
            raise ValueError("noverlap must be less than nperseg.")
        short = dict(params)
        short.update(win_length=int(n_eff), hop_length=int(n_eff - noverlap))
        stats_gate = _cabi.Gate(lib=gate.lib, **short)
        try:
            stats(stats_gate, n_eff)
            mean, std = stats_gate.noise_mean_std()
            thresh = stats_gate.noise_threshold()
        finally:
            stats_gate.close()
        gate.set_noise_threshold(thresh)
    else:
        stats(gate, clip.shape[1])
        mean, std = gate.noise_mean_std()
        thresh = gate.noise_threshold()
    return mean, std, thresh
