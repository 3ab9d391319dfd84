"""Mirror of noisereduce/spectralgate/streamed_torch_gate.py:7 (StreamedTorchGate): reduce_noise(use_torch=True).

The reference's torch route is NOT the numpy algorithm on a GPU: every padded chunk goes through TorchGate
(streamed_torch_gate.py:81-88), i.e. torch.stft(center=True) framing, per-chunk self statistics with top_db = 40 and an
unbiased std, the blend applied before the smoothing, and for the non-stationary gate a moving mean of
int(time_constant_s / hop * sr) frames instead of the filtfilt follower, with temp_coeff = 1 / sigmoid_slope and
n_thresh = thresh_n_mult_nonstationary (streamed_torch_gate.py:66-79).  The reference feeds TorchGate the float64 chunk
of base.py:140, so every chunk is computed in float64.

get_traces() runs the whole chunk grid of base.py:167-226 as ONE library call on the chunked torch surface
(B200GATE_SURFACE_TORCH_CHUNKED): every (chunk, channel) unit is a padded chunk filtered with TorchGate's arithmetic,
bit-identical to the reference's loop of one TorchGate call per chunk, which is kept as _get_traces_per_chunk().

Samples that are a torch CUDA tensor are read where they are and the result is a tensor on their device, as on the
numpy route (see SpectralGate).  There is no CPU path: `device` must be a CUDA device.
"""
import contextlib

import numpy as np
import torch

from .. import _cabi
from ..torchgate import TorchGate
from .base import SpectralGate, is_device_tensor


def torch_route_params(tg, stationary, chunk_size, padding):
    """Parameters of the chunked torch surface for TorchGate `tg` (the mapping of streamed_torch_gate.py:66-79)."""
    nf, nt = tg._extents if tg.smoothing_filter is not None else (0, 0)
    return dict(
        surface=_cabi.SURFACE_TORCH_CHUNKED, stationary=1 if stationary else 0, n_fft=int(tg.n_fft),
        win_length=int(tg.win_length), hop_length=int(tg.hop_length), n_grad_freq=int(nf), n_grad_time=int(nt),
        std_ddof=1, chunk_size=int(chunk_size) if chunk_size is not None else 0, padding=int(padding),
        sr=float(tg.sr), prop_decrease=float(tg.prop_decrease), n_std_thresh=float(tg.n_std_thresh_stationary),
        top_db=40.0,                                                   # torchgate/utils.py:6
        n_movemean=int(tg.n_movemean_nonstationary), thresh_n_mult=float(tg.n_thresh_nonstationary),
        sigmoid_slope=1.0 / float(tg.temp_coeff_nonstationary))


def make_torch_route_gate(params, lib=None):
    """A chunked-torch-surface handle with the reference's own window table (torchgate.py:231: torch.hann_window)."""
    gate = _cabi.Gate(lib=lib, **params)
    gate.set_window(torch.hann_window(params["win_length"]).numpy())
    return gate


def torch_noise_rows(y_noise):
    """y_noise as the route hands it to TorchGate (streamed_torch_gate.py:55-63): a tensor, 1-D made [1, Ln]."""
    if isinstance(y_noise, torch.Tensor):
        t = y_noise
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(y_noise)))
    return t.unsqueeze(0) if t.ndim == 1 else t


def check_torch_noise(xn, win_length):
    """TorchGate.forward's checks of xn (torchgate.py:214-220)."""
    assert xn.ndim == 1 or xn.ndim == 2
    if xn.shape[-1] < win_length * 2:
        raise Exception(f"xn must be bigger than {win_length * 2}")


def install_torch_noise(gate, xn, device, stream):
    """TorchGate.forward(x, xn)'s thresholds (torchgate.py:140-164) from the [Bn, Ln] clip, converted to float64 by torch
    as the reference converts it, on the handle `gate`, which lives on `device` (the host waits for the statistics)."""
    x64 = xn.detach().to(device=device, dtype=torch.float64).contiguous()
    gate.torch_set_noise(x64.data_ptr(), x64.shape[0], x64.shape[1], x64.stride(0), True, stream, dtype=np.float64)


def torch_len(L, n_fft, hop):
    """torch.istft(center=True) length of TorchGate's output for an L-sample input (torchgate.py:255-262)."""
    return (L // hop) * hop + (n_fft & 1)


class StreamedTorchGate(SpectralGate):
    def __init__(
        self,
        y,
        sr,
        stationary=False,
        y_noise=None,
        prop_decrease=1.0,
        time_constant_s=2.0,
        freq_mask_smooth_hz=500,
        time_mask_smooth_ms=50,
        thresh_n_mult_nonstationary=2,
        sigmoid_slope_nonstationary=10,
        n_std_thresh_stationary=1.5,
        tmp_folder=None,
        chunk_size=600000,
        padding=30000,
        n_fft=1024,
        win_length=None,
        hop_length=None,
        clip_noise_stationary=True,
        use_tqdm=False,
        n_jobs=1,
        device="cuda",
        _lib=None,
    ):
        super().__init__(
            y=y, sr=sr, chunk_size=chunk_size, padding=padding, n_fft=n_fft, win_length=win_length,
            hop_length=hop_length, time_constant_s=time_constant_s, freq_mask_smooth_hz=freq_mask_smooth_hz,
            time_mask_smooth_ms=time_mask_smooth_ms, tmp_folder=tmp_folder, prop_decrease=prop_decrease,
            use_tqdm=use_tqdm, n_jobs=n_jobs,
        )
        self._lib = _lib                                   # tests: the CPU simulator build of the library
        want = torch.device(device)
        if self._site is not None:                         # CUDA samples: the work runs on their device
            if not (want.type == "cuda" and want.index is None) and want != self._site.device:
                raise ValueError(f"device={device!r}, but the samples are on {self._site.device}")
            self.device = self._site.device
        elif _lib is None and not getattr(_cabi._LIB, "simulated_device", False):   # (tests: simulator, host memory)
            if not torch.cuda.is_available():
                raise RuntimeError("noisereduce_b200 has no CPU path: use_torch=True needs a CUDA device")
            self.device = want
            if self.device.type != "cuda":
                raise RuntimeError("noisereduce_b200 has no CPU path: device must be a CUDA device")
        else:
            self.device = torch.device("cpu")
        if y_noise is not None:                            # streamed_torch_gate.py:55-63
            if is_device_tensor(y_noise) and y_noise.device != self.device:
                raise ValueError(f"y_noise is on {y_noise.device}, the work runs on {self.device}")
            if not isinstance(y_noise, torch.Tensor):
                y_noise = np.asarray(y_noise)
            if y_noise.shape[-1] > self.n_frames and clip_noise_stationary:
                y_noise = y_noise[..., : self.n_frames]
            y_noise = torch_noise_rows(y_noise).to(self.device)
        self.y_noise = y_noise
        self._stationary = bool(stationary)
        self.tg = TorchGate(
            sr=sr,
            nonstationary=not stationary,
            n_std_thresh_stationary=n_std_thresh_stationary,
            n_thresh_nonstationary=thresh_n_mult_nonstationary,
            temp_coeff_nonstationary=1 / sigmoid_slope_nonstationary,
            n_movemean_nonstationary=int(time_constant_s / self._hop_length * sr),
            prop_decrease=prop_decrease,
            n_fft=self._n_fft,
            win_length=self._win_length,
            hop_length=self._hop_length,
            freq_mask_smooth_hz=freq_mask_smooth_hz,
            time_mask_smooth_ms=time_mask_smooth_ms,
        ).to(self.device)

    # -- the one library call over the chunk grid ----------------------------------------------------------------------
    def _gate_params(self):
        return torch_route_params(self.tg, self._stationary, self._chunk_size, self.padding)

    def _on_device(self):
        if self._site is not None:
            return self._site.active()
        return torch.cuda.device(self.device) if self.device.type == "cuda" else contextlib.nullcontext()

    def _check_unit(self, unit_len, chunked):
        """What the reference's loop raises for these padded chunks (unit_len samples each): TorchGate.forward's checks
        (torchgate.py:214-220), then -- on the chunk grid -- the slice assignment of a torch output shorter than
        padding + chunk_size (base.py:200-207)."""
        W = self.tg.win_length
        if unit_len < W * 2:
            raise Exception(f"x must be bigger than {W * 2}")
        if self.y_noise is not None:
            check_torch_noise(self.y_noise, W)
        have = torch_len(unit_len, self._n_fft, self._hop_length) - self.padding
        if chunked and have < self._chunk_size:
            raise ValueError(f"could not broadcast input array from shape ({self.n_channels},{max(have, 0)}) into shape "
                             f"({self.n_channels},{self._chunk_size})")
        return have

    def get_traces(self, start_frame=None, end_frame=None):
        """base.py:167-226 as the reference runs it for this back-end, as one library call: the chunks
        int(start/cs)..int((end-1)/cs) when the range is longer than chunk_size, else one padded chunk covering
        [0, end_frame).  Same result as _get_traces_per_chunk() in shape, dtype and every bit; on the device route a
        tensor on the samples' device."""
        start = 0 if start_frame is None else start_frame
        end = self.n_frames if end_frame is None else end_frame
        chunked = self._chunk_size is not None and end - start > self._chunk_size
        have = self._check_unit((self._chunk_size if chunked else end) + 2 * self.padding, chunked)
        with self._on_device():
            if self._gate is None:
                self._gate = make_torch_route_gate(self._gate_params(), self._lib)
                if self._stationary and self.y_noise is not None:
                    install_torch_noise(self._gate, self.y_noise, self.device,
                                        None if self._site is None else self._site.stream)
            out = super().get_traces(start_frame, end_frame)
        if not chunked and have < end:        # base.py:222: the slice of a torch output shorter than padding + end
            out = out[..., :have]
        return out

    # -- the reference's loop, kept as the bit-identity reference ---------------------------------------------------
    def _do_filter(self, chunk):
        """streamed_torch_gate.py:81-88: one padded chunk [C, Lp] through TorchGate; [C, (Lp // hop) * hop] back."""
        x = torch.from_numpy(np.ascontiguousarray(chunk)).to(self.device) if isinstance(chunk, np.ndarray) else chunk
        with torch.no_grad():
            out = self.tg(x=x, xn=self.y_noise, _lib=self._lib)
        return out.cpu().numpy()

    def _get_traces_per_chunk(self, start_frame=None, end_frame=None):
        """base.py:167-226 as the reference runs it: a loop over the chunk grid, each chunk padded, filtered by
        _do_filter (one TorchGate call) and its centre copied out.  numpy samples only."""
        if start_frame is None:
            start_frame = 0
        if end_frame is None:
            end_frame = self.n_frames
        if self._chunk_size is not None and end_frame - start_frame > self._chunk_size:
            ich1, ich2 = int(start_frame / self._chunk_size), int((end_frame - 1) / self._chunk_size)
            out = np.zeros((self.n_channels, int(end_frame - start_frame)), dtype=self._dtype)
            pos = 0
            for ich in range(ich1, ich2 + 1):
                start0 = start_frame - ich * self._chunk_size if ich == ich1 else 0
                end0 = end_frame - ich * self._chunk_size if ich == ich2 else self._chunk_size
                part = self._get_filtered_chunk(ich)
                with np.errstate(invalid="ignore"):
                    out[:, pos: pos + end0 - start0] = part[:, start0:end0]
                pos += end0 - start0
        else:
            with np.errstate(invalid="ignore"):
                out = self.filter_chunk(start_frame=0, end_frame=end_frame).astype(self._dtype)
        return out.flatten() if self.flat else out
