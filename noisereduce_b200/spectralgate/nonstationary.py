"""Mirror of noisereduce/spectralgate/nonstationary.py:7 (SpectralGateNonStationary) on libb200gate."""
from .. import _cabi
from .base import SpectralGate


class SpectralGateNonStationary(SpectralGate):
    def __init__(
        self,
        y,
        sr,
        chunk_size,
        padding,
        n_fft,
        win_length,
        hop_length,
        time_constant_s,
        freq_mask_smooth_hz,
        time_mask_smooth_ms,
        thresh_n_mult_nonstationary,
        sigmoid_slope_nonstationary,
        tmp_folder,
        prop_decrease,
        use_tqdm,
        n_jobs,
    ):
        self._thresh_n_mult_nonstationary = thresh_n_mult_nonstationary
        self._sigmoid_slope_nonstationary = sigmoid_slope_nonstationary
        super().__init__(
            y=y, sr=sr, chunk_size=chunk_size, padding=padding, n_fft=n_fft, win_length=win_length,
            hop_length=hop_length, time_constant_s=time_constant_s, freq_mask_smooth_hz=freq_mask_smooth_hz,
            time_mask_smooth_ms=time_mask_smooth_ms, tmp_folder=tmp_folder, prop_decrease=prop_decrease,
            use_tqdm=use_tqdm, n_jobs=n_jobs,
        )
        params = self._gate_params()
        params.update(stationary=0, time_constant_s=float(time_constant_s),
                      thresh_n_mult=float(thresh_n_mult_nonstationary),
                      sigmoid_slope=float(sigmoid_slope_nonstationary))
        self._params = params
        with self._on_device():
            self._gate = _cabi.Gate(**params)

    def _unit_gate_params(self):
        p = dict(self._params)
        p.update(chunk_size=0, padding=0)
        return p
