"""reduce_noise_batch() -- many recordings of different lengths through ONE library handle and one b200gate_run_rows call.

Every item is cut into (chunk, channel) units exactly as reduce_noise() cuts it (a recording no longer than chunk_size is
one padded chunk of its own length), the units of all items form one table, and the kernels read each unit's geometry
from it (include/b200gate.h, b200gate_run_rows).  So ``outs[i]`` has the bits of ``reduce_noise(ys[i], sr, ...)`` while
the handle's life cycle -- construction, the stationary thresholds, the device-wide wait of its destruction -- is paid
once per call instead of once per item.
"""
import ctypes

import numpy as np

from . import _cabi
from .spectralgate.base import KERNEL_DTYPES, DeviceSite, SpectralGate, is_device_tensor, numpy_dtype_of
from .spectralgate.stationary import install_noise_thresholds

_ROW_ALIGN = 16          # host rows are packed at 16-byte offsets (the analysis kernel prefetches 16-byte aligned spans)
_FPAD = 544              # padded bin count of the n_fft = 1024 kernels (csrc/gate_kernels.cuh, kFPad)


def _refuse_smoothing(stationary, nf, nt):
    """The extents the batch kernels hold (b200gate_run_rows returns B200GATE_ERR_ARG for the rest)."""
    if stationary:
        # the in-synthesis smoothing's byte lanes (csrc/gate_host.cu, packed_smoothing_fits)
        if nt + 1 > 14:
            raise NotImplementedError(f"reduce_noise_batch: time_mask_smooth_ms gives {nt} frames; the stationary batch "
                                      "kernels smooth at most 13")
        if 2 * nf + 1 > 36:
            raise NotImplementedError(f"reduce_noise_batch: freq_mask_smooth_hz gives {nf} bins; the stationary batch "
                                      "kernels smooth at most 17")
    else:
        # the streaming float-mask smoothing keeps 2 nt + 1 mask rows in shared memory (smooths_smem_bytes)
        if ((2 * nt + 1) * _FPAD + _FPAD + 2 * nf + 8) * 4 > 200 * 1024:
            raise NotImplementedError(f"reduce_noise_batch: time_mask_smooth_ms / freq_mask_smooth_hz give ({nt}, {nf}) "
                                      "frames / bins, beyond the batch kernels' shared-memory ring")


def reduce_noise_batch(
    ys,
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
    y_noise_per_item=None,
):
    """Denoise a list of recordings in one GPU call; ``outs[i]`` is bit-identical to ``reduce_noise(ys[i], sr, ...)``.

    ys : non-empty list / tuple of recordings, each ``(n,)`` or ``(channels, n)``; all numpy arrays, or all torch CUDA
    tensors on one device; all of one dtype.  Lengths and channel counts may differ.  The other arguments are
    reduce_noise()'s, with the same defaults.  Returns a list with one result per item, of the item's type, shape, dtype
    and device.  An item reduce_noise() refuses raises the same exception type before any GPU work.

    CUDA tensors are read where they are (unit sample stride, any row stride; other layouts are copied) and each result
    is a new tensor, enqueued on the device's current torch stream.  Numpy items are staged through one pooled
    page-locked buffer, one copy to the device and one back.  One library handle serves the whole call; its destruction
    on return waits for the device, as in reduce_noise().

    Covered: the non-stationary gate, and the stationary gate with a ``y_noise`` (one noise clip for the whole batch:
    with a clip the thresholds do not depend on the item) or with ``y_noise_per_item``; n_fft = win_length = 1024,
    hop_length = 256; float32, int16 and float64 samples.  Everything else raises NotImplementedError naming the
    argument: ``use_torch=True``, ``stationary=True`` with neither, another geometry, another dtype, tensors that require
    grad, and smoothing extents beyond the batch kernels'.

    y_noise_per_item : with ``stationary=True``, a list or tuple with one entry per item: ``None`` makes ``outs[i]``
    ``reduce_noise(ys[i], sr, stationary=True, ...)`` (the item's first chunk_size samples are its noise clip), a clip
    (numpy array or tensor, ``(n,)`` or ``(C, n)``) makes it ``reduce_noise(ys[i], sr, stationary=True, y_noise=clip,
    ...)``.  Every item gets its own thresholds; the clips of one dtype and memory space take one batched statistics
    call (b200gate_noise_stats_rows), ``None`` entries reading the item's rows where the batch reads them.  A clip of a
    dtype other than float32 / int16 / float64, or one with fewer than win_length samples after clipping, takes
    reduce_noise()'s one-clip path and pays a library handle's life cycle of its own.  ``ValueError`` when it is given
    together with ``y_noise``, with ``stationary=False``, or with a length other than ``len(ys)``; a clip reduce_noise()
    refuses raises what reduce_noise() raises.
    """
    if not isinstance(ys, (list, tuple)):
        raise TypeError("reduce_noise_batch: ys must be a list or tuple of recordings")
    if len(ys) == 0:
        raise ValueError("reduce_noise_batch: ys is empty")
    on_device = [is_device_tensor(y) for y in ys]
    if any(on_device) and not all(on_device):
        raise TypeError("reduce_noise_batch: ys mixes device tensors with host arrays")
    on_device = on_device[0]
    if not on_device:
        ys = [np.asarray(y) for y in ys]
    dtypes = {numpy_dtype_of(y) if on_device else y.dtype for y in ys}
    if len(dtypes) > 1:
        raise TypeError(f"reduce_noise_batch: ys mixes sample dtypes {sorted(str(d) for d in dtypes)}")
    if on_device and len({y.device for y in ys}) > 1:
        raise ValueError("reduce_noise_batch: ys are on different devices")

    if y_noise_per_item is not None:
        if not isinstance(y_noise_per_item, (list, tuple)):
            raise TypeError("reduce_noise_batch: y_noise_per_item must be a list or tuple with one entry per item")
        if y_noise is not None:
            raise ValueError("reduce_noise_batch: give y_noise (one clip for the batch) or y_noise_per_item, not both")
        if not stationary:
            raise ValueError("reduce_noise_batch: y_noise_per_item is for the stationary gate (stationary=True)")
        if len(y_noise_per_item) != len(ys):
            raise ValueError(f"reduce_noise_batch: y_noise_per_item has {len(y_noise_per_item)} entries for {len(ys)} items")

    # ---- scope of this version ------------------------------------------------------------------------------------
    if use_torch:
        raise NotImplementedError("reduce_noise_batch: use_torch=True is not supported")
    if stationary and y_noise is None and y_noise_per_item is None:
        raise NotImplementedError("reduce_noise_batch: stationary=True needs a y_noise, or y_noise_per_item (every item "
                                  "then has its own thresholds)")
    win = n_fft if win_length is None else win_length
    hop = win // 4 if hop_length is None else hop_length
    if (n_fft, win, hop) != (1024, 1024, 256):
        raise NotImplementedError(f"reduce_noise_batch: n_fft / win_length / hop_length = {n_fft} / {win} / {hop}; only "
                                  "1024 / 1024 / 256 is supported")
    dtype = np.dtype(next(iter(dtypes)))
    if dtype not in KERNEL_DTYPES and not np.issubdtype(dtype, np.complexfloating):
        raise NotImplementedError(f"reduce_noise_batch: sample dtype {dtype}; only float32, int16 and float64 are supported")
    if on_device and any(y.requires_grad for y in ys) and DeviceSite(ys[0]).torch.is_grad_enabled():
        raise NotImplementedError("reduce_noise_batch: tensors that require grad are not supported")

    # ---- every item through reduce_noise()'s own checks (SpectralGate.__init__ touches no device) -------------------
    common = dict(sr=sr, prop_decrease=prop_decrease, chunk_size=chunk_size, padding=padding, n_fft=n_fft,
                  win_length=win_length, hop_length=hop_length, time_constant_s=time_constant_s,
                  freq_mask_smooth_hz=freq_mask_smooth_hz, time_mask_smooth_ms=time_mask_smooth_ms, tmp_folder=tmp_folder,
                  use_tqdm=use_tqdm, n_jobs=n_jobs)
    items = [SpectralGate(y=y, **common) for y in ys]
    params = items[0]._gate_params()
    _refuse_smoothing(stationary, params["n_grad_freq"], params["n_grad_time"])
    if stationary:
        params.update(stationary=1, n_std_thresh=float(n_std_thresh_stationary), clip_noise=1 if clip_noise_stationary else 0)
    else:
        params.update(stationary=0, time_constant_s=float(time_constant_s), thresh_n_mult=float(thresh_n_mult_nonstationary),
                      sigmoid_slope=float(sigmoid_slope_nonstationary))
    site = items[0]._site
    noise = None
    clip_to = chunk_size if clip_noise_stationary else None
    if stationary and y_noise_per_item is None:                  # the clip's layout checks of SpectralGateStationary
        if site is not None and is_device_tensor(y_noise):
            site.check_same_device(y_noise, "y_noise")
        else:
            y_noise = np.array(y_noise)
        if len(y_noise.shape) > 2:
            raise ValueError("Waveform must be in shape (# frames, # channels)")
        noise = y_noise[None, :] if len(y_noise.shape) == 1 else y_noise
    clips = None
    if y_noise_per_item is not None:
        # an item that is its own clip stays None (read where the batch reads it) unless it is shorter than the window
        clips = [None if c is None and _effective_length(it.n_frames, clip_to) >= params["win_length"] else
                 _NoiseClip(it.y if c is None else c, site, clip_to, params["win_length"], params["hop_length"], i)
                 for i, (it, c) in enumerate(zip(items, y_noise_per_item))]

    # ---- one handle, one call ---------------------------------------------------------------------------------------
    with items[0]._on_device():
        gate = _cabi.Gate(**params)
        try:
            stream = None if site is None else site.stream
            install = None
            if clips is not None:
                def install(own_rows):
                    _install_per_item(gate, params, clips, own_rows, dtype, on_device, clip_to, stream)
            elif stationary:
                install_noise_thresholds(gate, params, noise, clip_to, stream)
            outs = _run_tensors(gate, items, dtype, stream, install) if on_device else \
                _run_arrays(gate, items, dtype, install)
        finally:
            gate.close()
    return [o.flatten() if it.flat else o for o, it in zip(outs, items)]


def _effective_length(n, clip_to):
    """Samples of a noise clip the statistics read (stationary.py:63-64)."""
    return n if clip_to is None else min(n, int(clip_to))


class _NoiseClip:
    """One explicit entry of y_noise_per_item, checked as SpectralGateStationary checks its y_noise.  ``batched``: the
    clip takes b200gate_noise_stats_rows (a [C, n] clip of a kernel dtype with at least win_length samples after
    clipping); otherwise install_noise_thresholds() on a handle of its own, reduce_noise()'s path."""

    def __init__(self, clip, site, clip_to, win_length, hop_length, i):
        if site is not None and is_device_tensor(clip):
            site.check_same_device(clip, f"y_noise_per_item[{i}]")       # a CUDA clip is read in place
            self.is_device, self.dtype = True, numpy_dtype_of(clip)
        else:
            clip = np.array(clip)                                        # host statistics, as reduce_noise()
            self.is_device, self.dtype = False, clip.dtype
        self.noise = clip[None, :] if len(clip.shape) == 1 else clip
        self.batched = len(self.noise.shape) == 2 and self.dtype in KERNEL_DTYPES
        if len(self.noise.shape) == 2:
            n_eff = _effective_length(self.noise.shape[1], clip_to)
            if n_eff <= win_length - hop_length:                         # what scipy.signal.stft raises (stationary.py)
                raise ValueError("noverlap must be less than nperseg.")
            self.batched = self.batched and n_eff >= win_length

    def rows(self, clip_to):
        """(pointer, C, n, row stride) for b200gate_noise_stats_rows; keeps any copy it makes alive on self."""
        if self.is_device:
            self._rows, stride = DeviceSite(self.noise).rows(self.noise)
            C, n = self._rows.shape
            return self._rows.data_ptr(), C, n, stride
        x, es = self.noise, self.dtype.itemsize
        C, n = x.shape
        if not (x.strides[1] == es and x.strides[0] % es == 0 and (C == 1 or x.strides[0] >= n * es)):
            x = np.ascontiguousarray(x[:, :_effective_length(n, clip_to)])     # (the statistics read no further)
            C, n = x.shape
        self._rows = x
        return x.ctypes.data, C, n, x.strides[0] // es if C > 1 else n


def _install_per_item(gate, params, clips, own_rows, dtype, on_device, clip_to, stream):
    """Per-item thresholds on `gate`: one b200gate_noise_stats_rows call per (dtype, memory space) of the clips -- an item
    without a clip is read at own_rows[i], where the batch reads its samples -- and the one-clip path for the rest."""
    thr = np.empty((len(clips), gate.n_bins), np.float64)
    groups = {}
    for i, c in enumerate(clips):
        if c is None:
            groups.setdefault((dtype, on_device), []).append((i, own_rows[i]))
        elif c.batched:
            groups.setdefault((c.dtype, c.is_device), []).append((i, c.rows(clip_to)))
        else:
            single = _cabi.Gate(lib=gate.lib, **params)
            try:
                thr[i] = install_noise_thresholds(single, params, c.noise, clip_to, stream)[2]
            finally:
                single.close()
    for (dt, is_device), members in groups.items():
        thr[[i for i, _ in members]] = gate.noise_stats_rows([r for _, r in members], dt, is_device,
                                                             stream if is_device else None)
    gate.set_noise_threshold_rows(thr)


def _run_tensors(gate, items, dtype, stream, install=None):
    site, es = items[0]._site, dtype.itemsize
    rows, outs, keep, own = [], [], [], []
    for it in items:
        x, stride = site.rows(it.y)
        keep.append(x)
        C, n = x.shape
        out = site.empty((C, n), dtype)
        outs.append(out)
        xp, op = x.data_ptr(), out.data_ptr()
        own.append((xp, C, n, stride))
        rows.extend((xp + c * stride * es, op + c * n * es, n, C) for c in range(C))
    if install is not None:
        install(own)
    gate.run_rows(rows, dtype, True, stream)
    return outs


def _run_arrays(gate, items, dtype, install=None):
    es = dtype.itemsize
    offs, total = [], 0
    for it in items:
        for _ in range(it.n_channels):
            offs.append(total)
            total += (it.n_frames * es + _ROW_ALIGN - 1) // _ROW_ALIGN * _ROW_ALIGN
    # input rows in the first half of one page-locked buffer, results in the second (ordinary memory if it cannot be pinned)
    dll = gate.lib.dll
    pinned = dll.b200gate_host_alloc(2 * total)
    store = None if pinned else np.empty(2 * total + _ROW_ALIGN, np.uint8)
    base = pinned or -(-store.ctypes.data // _ROW_ALIGN) * _ROW_ALIGN
    try:
        rows, own, k = [], [], 0
        for it in items:
            # an item's rows are evenly spaced: its own noise clip is (first row, C, n, row pitch)
            pitch = (offs[k + 1] - offs[k]) // es if it.n_channels > 1 else it.n_frames
            own.append((base + offs[k], it.n_channels, it.n_frames, pitch))
            for c in range(it.n_channels):
                row = np.frombuffer((ctypes.c_char * (it.n_frames * es)).from_address(base + offs[k]), dtype=dtype)
                row[:] = it.y[c]
                rows.append((base + offs[k], base + total + offs[k], it.n_frames, it.n_channels))
                k += 1
        if install is not None:
            install(own)
        gate.run_rows(rows, dtype, False)
        outs, k = [], 0
        for it in items:
            out = np.empty((it.n_channels, it.n_frames), dtype)
            for c in range(it.n_channels):
                out[c] = np.frombuffer((ctypes.c_char * (it.n_frames * es)).from_address(base + total + offs[k]), dtype=dtype)
                k += 1
            outs.append(out)
    finally:
        if pinned:
            dll.b200gate_host_free(pinned)
    return outs
