"""reduce_noise() -- drop-in for noisereduce/noisereduce.py:13 on the H100-native backend."""
from .spectralgate import SpectralGateNonStationary, SpectralGateStationary


def reduce_noise(
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
    use_torch=False,
    device="cuda",
):
    """Reduce noise via spectral gating (same arguments, defaults and return value as the reference).

    y : np.ndarray, shape (# frames,) or (# channels, # frames); the result has the same shape and
    dtype.  ``n_jobs``, ``tmp_folder`` and ``use_tqdm`` are accepted and ignored: the chunk loop they
    steer in the reference runs as one GPU grid here.  ``use_torch=True`` takes the reference's torch route
    (noisereduce.py:121-143 -> StreamedTorchGate): every padded chunk through TorchGate -- a different gate from
    the numpy one (torch.stft framing, per-chunk self statistics, top_db 40, moving-mean follower; see
    spectralgate/streamed_torch_gate.py) -- on ``device``, which must be a CUDA device.  There is no CPU path.

    y may also be a torch CUDA tensor (use_torch=False): the samples are read where they are and the result is a tensor
    on the same device, with the same shape and dtype and the same bits as
    ``torch.from_numpy(reduce_noise(y.cpu().numpy(), sr, ...))``.  The work runs on that device's current torch stream,
    but the call does not return with it in flight.  The stationary threshold computation waits for the device.  So
    does the destruction of the call's library handle on return, which waits for the whole device, including work on
    other streams (spectralgate/base.py has the details).  ``y_noise`` may
    then be a numpy array, a CPU tensor or a CUDA tensor on y's device (another device raises ValueError).  float16,
    integer and bool tensors are promoted to float64 and cast back on the device with numpy's rules; bfloat16 raises
    TypeError.  CPU tensors take the numpy route and return numpy arrays, as before.  See spectralgate/base.py.
    """
    if use_torch:
        if n_jobs != 1:                                         # noisereduce.py:115-118
            raise ValueError("n_jobs must be 1 when using torch version of spectral gating.")
        from .spectralgate.streamed_torch_gate import StreamedTorchGate
        sg = StreamedTorchGate(                                 # (n_std_thresh_stationary is not forwarded, as in the reference)
            y=y, sr=sr, stationary=stationary, y_noise=y_noise, prop_decrease=prop_decrease,
            time_constant_s=time_constant_s, freq_mask_smooth_hz=freq_mask_smooth_hz,
            time_mask_smooth_ms=time_mask_smooth_ms, thresh_n_mult_nonstationary=thresh_n_mult_nonstationary,
            sigmoid_slope_nonstationary=sigmoid_slope_nonstationary, tmp_folder=tmp_folder, chunk_size=chunk_size,
            padding=padding, n_fft=n_fft, win_length=win_length, hop_length=hop_length,
            clip_noise_stationary=clip_noise_stationary, use_tqdm=use_tqdm, n_jobs=n_jobs, device=device,
        )
        return sg.get_traces()
    if stationary:
        sg = SpectralGateStationary(
            y=y, sr=sr, y_noise=y_noise, prop_decrease=prop_decrease,
            n_std_thresh_stationary=n_std_thresh_stationary, chunk_size=chunk_size,
            clip_noise_stationary=clip_noise_stationary, padding=padding, n_fft=n_fft,
            win_length=win_length, hop_length=hop_length, time_constant_s=time_constant_s,
            freq_mask_smooth_hz=freq_mask_smooth_hz, time_mask_smooth_ms=time_mask_smooth_ms,
            tmp_folder=tmp_folder, use_tqdm=use_tqdm, n_jobs=n_jobs,
        )
    else:
        sg = SpectralGateNonStationary(
            y=y, sr=sr, chunk_size=chunk_size, padding=padding, prop_decrease=prop_decrease,
            n_fft=n_fft, win_length=win_length, hop_length=hop_length, time_constant_s=time_constant_s,
            freq_mask_smooth_hz=freq_mask_smooth_hz, time_mask_smooth_ms=time_mask_smooth_ms,
            thresh_n_mult_nonstationary=thresh_n_mult_nonstationary,
            sigmoid_slope_nonstationary=sigmoid_slope_nonstationary, tmp_folder=tmp_folder,
            use_tqdm=use_tqdm, n_jobs=n_jobs,
        )
    return sg.get_traces()
