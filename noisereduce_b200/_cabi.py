"""ctypes binding of libb200gate.so (include/b200gate.h).

There is deliberately no fallback here: if the CUDA library has not been built, or no CUDA device
is present, the calls raise.  (tests/ load a CPU *simulator* build of the same sources through
``GateLibrary(path)`` to debug kernel logic without a GPU; the package itself never does.)
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libb200gate.so")

ABI_VERSION = 1
OK, ERR_ARG, ERR_CUDA, ERR_STATE, ERR_NOMEM = 0, -1, -2, -3, -4
F32, I16, F64 = 0, 1, 2
SURFACE_NUMPY, SURFACE_TORCH, SURFACE_TORCH_CHUNKED = 0, 1, 2
_DTYPES = {np.dtype(np.float32): F32, np.dtype(np.int16): I16, np.dtype(np.float64): F64}
# b200gate_convert's further formats (include/b200gate.h)
BOOL, I8, U8, U16, I32, U32, I64, U64, F16 = 3, 4, 5, 6, 7, 8, 9, 10, 11
CONVERT_CAST, CONVERT_CHANNEL_MEAN = 0, 1
_FORMATS = {**_DTYPES, **{np.dtype(t): c for t, c in (
    (np.bool_, BOOL), (np.int8, I8), (np.uint8, U8), (np.uint16, U16), (np.int32, I32), (np.uint32, U32),
    (np.int64, I64), (np.uint64, U64), (np.float16, F16))}}

EXPORTS = [
    "b200gate_create", "b200gate_destroy", "b200gate_last_error", "b200gate_noise_stats",
    "b200gate_noise_stats_collapsed", "b200gate_channel_sum", "b200gate_set_noise_threshold",
    "b200gate_get_noise_threshold", "b200gate_get_noise_mean_std", "b200gate_set_window",
    "b200gate_torch_set_noise",
    "b200gate_run", "b200gate_set_range", "b200gate_get_stats", "b200gate_debug_select_unit", "b200gate_debug_dims",
    "b200gate_debug_read_bits", "b200gate_debug_read_mask", "b200gate_debug_read_spec",
    "b200gate_run_sharded", "b200gate_peer_push", "b200gate_peer_barrier", "b200gate_torch_apply_masks",
    "b200gate_host_alloc", "b200gate_host_free",
    "b200gate_stream_begin", "b200gate_stream_push", "b200gate_stream_finish", "b200gate_convert",
    "b200gate_mask_store_bytes", "b200gate_set_mask_store", "b200gate_adjoint", "b200gate_run_rows",
    "b200gate_torch_apply_masks_rows", "b200gate_noise_stats_rows", "b200gate_set_noise_threshold_rows",
    "b200gate_tstream_begin", "b200gate_tstream_push", "b200gate_tstream_finish",
    "b200gate_tstream_push_rows", "b200gate_tstream_end_rows", "b200gate_tstream_reset_rows",
]


class Params(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32), ("surface", C.c_int32), ("stationary", C.c_int32),
        ("n_fft", C.c_int32), ("win_length", C.c_int32), ("hop_length", C.c_int32),
        ("n_grad_freq", C.c_int32), ("n_grad_time", C.c_int32), ("std_ddof", C.c_int32),
        ("clip_noise", C.c_int32), ("n_movemean", C.c_int32), ("debug_guard_scale", C.c_int32),
        ("reserve_sms", C.c_int32), ("path_flags", C.c_int32),
        ("chunk_size", C.c_int64), ("padding", C.c_int64),
        ("sr", C.c_double), ("prop_decrease", C.c_double), ("n_std_thresh", C.c_double),
        ("top_db", C.c_double), ("time_constant_s", C.c_double), ("thresh_n_mult", C.c_double),
        ("sigmoid_slope", C.c_double), ("workspace_limit_bytes", C.c_double),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("units", C.c_int64), ("frames", C.c_int64), ("kernel_launches", C.c_int64),
        ("bins_rechecked_fp64", C.c_int64), ("bins_unresolved", C.c_int64),
        ("rowfloor_flags", C.c_int64), ("rowfloor_ambiguous", C.c_int64),
        ("last_run_ms", C.c_double), ("last_h2d_ms", C.c_double), ("last_d2h_ms", C.c_double),
        ("k1_ms", C.c_double), ("smooth_ms", C.c_double), ("k2_ms", C.c_double),
        ("fused_ms", C.c_double), ("fused_path", C.c_int64), ("fused_fallbacks", C.c_int64),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class Row(C.Structure):
    """b200gate_row: one channel of one recording (b200gate_run_rows)."""
    _fields_ = [("in_", C.c_void_p), ("out", C.c_void_p), ("n", C.c_int64), ("channels", C.c_int64)]


class NoiseClip(C.Structure):
    """b200gate_noise_clip: one noise clip of b200gate_noise_stats_rows, [C][n] with row stride `stride` elements."""
    _fields_ = [("x", C.c_void_p), ("C", C.c_int64), ("n", C.c_int64), ("stride", C.c_int64)]


class GateError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200gate error {code}: {msg}")
        self.code = code


class GateLibrary:
    """A loaded libb200gate with typed prototypes.

    ``simulated_device`` (tests only, default False): the library is the CPU simulator build, whose "device" pointers
    are host pointers, and CPU torch tensors take the CUDA-tensor route of reduce_noise() / NoiseReduceStream."""

    simulated_device = False

    def __init__(self, path: str = DEFAULT_LIB):
        if not os.path.exists(path):
            raise RuntimeError(
                f"{path} not found: build the CUDA library first "
                "(python -m noisereduce_b200.csrc.build, or __graft_entry__.build()). "
                "noisereduce_b200 has no CPU fallback."
            )
        self.path = path
        self.dll = C.CDLL(path)
        d = self.dll
        vp, i64, i32, dbl = C.c_void_p, C.c_int64, C.c_int32, C.c_double
        d.b200gate_create.argtypes = [C.POINTER(Params), C.POINTER(vp)]
        d.b200gate_destroy.argtypes = [vp]
        d.b200gate_destroy.restype = None
        d.b200gate_last_error.argtypes = [vp]
        d.b200gate_last_error.restype = C.c_char_p
        d.b200gate_noise_stats.argtypes = [vp, vp, C.c_int, i64, i64, i64, C.c_int, vp]
        d.b200gate_noise_stats_collapsed.argtypes = [vp, vp, C.c_int, i64, C.c_int, vp]
        d.b200gate_channel_sum.argtypes = [vp, vp, C.c_int, i64, i64, i64, C.c_int, vp, C.c_int, vp]
        d.b200gate_set_noise_threshold.argtypes = [vp, C.POINTER(dbl), i32]
        d.b200gate_get_noise_threshold.argtypes = [vp, C.POINTER(dbl), i32]
        d.b200gate_get_noise_mean_std.argtypes = [vp, C.POINTER(dbl), C.POINTER(dbl), i32]
        d.b200gate_set_window.argtypes = [vp, C.POINTER(C.c_float), i32]
        d.b200gate_torch_set_noise.argtypes = [vp, vp, C.c_int, i64, i64, i64, C.c_int, vp]
        d.b200gate_run.argtypes = [vp, vp, vp, C.c_int, i64, i64, i64, i64, C.c_int, vp]
        d.b200gate_torch_apply_masks.argtypes = [vp, vp, vp, C.c_int, i64, i64, i64, i64, C.c_int, vp]
        d.b200gate_set_range.argtypes = [vp, i32, i64, i64]
        d.b200gate_get_stats.argtypes = [vp, C.POINTER(Stats)]
        d.b200gate_debug_select_unit.argtypes = [vp, i64, i64]
        d.b200gate_debug_dims.argtypes = [vp, C.POINTER(i64), C.POINTER(i32), C.POINTER(i32)]
        d.b200gate_debug_read_bits.argtypes = [vp, vp]
        d.b200gate_debug_read_mask.argtypes = [vp, vp]
        d.b200gate_debug_read_spec.argtypes = [vp, vp]
        pvp = C.POINTER(vp)
        d.b200gate_run_sharded.argtypes = [vp, vp, C.c_int, i64, i64, i64, vp, pvp, vp, pvp, C.c_uint32, i32, i32, i32, i32, vp, vp]
        d.b200gate_peer_push.argtypes = [vp, pvp, i32, i64, i64, i64, i64, i32, vp]
        d.b200gate_peer_barrier.argtypes = [vp, pvp, i32, i32, C.c_uint32, vp]
        d.b200gate_host_alloc.argtypes = [C.c_size_t]
        d.b200gate_host_alloc.restype = vp
        d.b200gate_host_free.argtypes = [vp]
        d.b200gate_host_free.restype = None
        d.b200gate_stream_begin.argtypes = [vp, C.c_int, i64]
        d.b200gate_stream_push.argtypes = [vp, vp, i64, i64, C.c_int, vp, i64, i64, C.POINTER(i64), vp]
        d.b200gate_stream_finish.argtypes = [vp, vp, i64, i64, C.POINTER(i64), vp]
        d.b200gate_convert.argtypes = [C.c_int, vp, C.c_int, i64, vp, C.c_int, i64, i64, i64, vp]
        d.b200gate_mask_store_bytes.argtypes = [vp, i64, i64, C.POINTER(i64)]
        d.b200gate_set_mask_store.argtypes = [vp, vp, i64]
        d.b200gate_adjoint.argtypes = [vp, vp, vp, vp, C.c_int, i64, i64, i64, i64, C.c_int, vp]
        d.b200gate_run_rows.argtypes = [vp, C.POINTER(Row), i64, C.c_int, C.c_int, vp]
        d.b200gate_torch_apply_masks_rows.argtypes = [vp, C.POINTER(Row), i64, C.c_int, C.c_int, vp]
        d.b200gate_noise_stats_rows.argtypes = [vp, C.POINTER(NoiseClip), i64, C.c_int, C.c_int, C.POINTER(dbl), vp]
        d.b200gate_set_noise_threshold_rows.argtypes = [vp, C.POINTER(dbl), i64, i32]
        d.b200gate_tstream_begin.argtypes = [vp, i64]
        d.b200gate_tstream_push.argtypes = [vp, vp, i64, i64, vp, i64, i64, C.POINTER(i64), vp]
        d.b200gate_tstream_finish.argtypes = [vp, vp, i64, i64, C.POINTER(i64), vp]
        d.b200gate_tstream_push_rows.argtypes = [vp, vp, C.POINTER(i64), i64, vp, i64, i64, C.POINTER(i64), vp]
        d.b200gate_tstream_end_rows.argtypes = [vp, C.POINTER(i64), i64, vp, i64, i64, C.POINTER(i64), vp]
        d.b200gate_tstream_reset_rows.argtypes = [vp, C.POINTER(i64), i64]


def _i64p(a: np.ndarray):
    """A C int64_t* to the data of a contiguous int64 numpy array."""
    assert a.dtype == np.int64 and a.flags.c_contiguous
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def format_code(dt) -> int:
    """b200gate_convert's code for a numpy dtype (every real dtype numpy and torch share)."""
    dt = np.dtype(dt)
    if dt not in _FORMATS:
        raise TypeError(f"unsupported sample dtype {dt}")
    return _FORMATS[dt]


def convert(lib, op, src_ptr, src_dtype, src_stride, dst_ptr, dst_dtype, dst_stride, C_, N, stream=None):
    """b200gate_convert on device pointers (include/b200gate.h): op CONVERT_CAST or CONVERT_CHANNEL_MEAN."""
    rc = lib.dll.b200gate_convert(op, src_ptr, format_code(src_dtype), src_stride, dst_ptr, format_code(dst_dtype),
                                  dst_stride, C_, N, stream)
    if rc != 0:
        raise GateError(rc, lib.dll.b200gate_last_error(None).decode())


def peer_push(lib, src_ptr, peer_ptrs, rows, row_bytes, src_stride_bytes, dst_stride_bytes, n_ctas, stream):
    arr = (C.c_void_p * len(peer_ptrs))(*[int(p) for p in peer_ptrs])
    rc = lib.dll.b200gate_peer_push(src_ptr, arr, len(peer_ptrs), rows, row_bytes, src_stride_bytes, dst_stride_bytes, n_ctas, stream)
    if rc != 0:
        raise GateError(rc, "b200gate_peer_push")


def peer_barrier(lib, flags_local, flags_peers, rank, world, epoch, stream):
    arr = (C.c_void_p * world)(*[int(p) if p else None for p in flags_peers])
    rc = lib.dll.b200gate_peer_barrier(flags_local, arr, rank, world, epoch, stream)
    if rc != 0:
        raise GateError(rc, "b200gate_peer_barrier")


# ---- result arrays in page-locked memory ---------------------------------------------------------------------------
# A fresh np.empty() result of several GB is written through page faults and a staging copy; a buffer leased from the
# library's pinned pool (b200gate_host_alloc) takes the device -> host copy directly and is reused by the next call once
# the caller has dropped the previous result.  Small results and anything beyond the budget stay ordinary arrays.
PINNED_RESULT_MIN_BYTES = 32 << 20
_pinned_leased_bytes = 0


def _pinned_budget_bytes() -> int:
    env = os.environ.get("B200GATE_PINNED_RESULT_LIMIT")
    if env is not None:
        return int(float(env))
    try:
        return int(os.sysconf("SC_PHYS_PAGES") * os.sysconf("SC_PAGE_SIZE") * 0.25)
    except (ValueError, OSError):
        return 8 << 30


class _PinnedLease:
    """Owns one b200gate_host_alloc buffer; the ndarray built on it keeps this object alive through its base chain."""

    def __init__(self, lib: "GateLibrary", nbytes: int):
        global _pinned_leased_bytes
        self.lib, self.nbytes = lib, nbytes
        self.ptr = lib.dll.b200gate_host_alloc(nbytes)
        if not self.ptr:
            raise MemoryError("b200gate_host_alloc")
        _pinned_leased_bytes += nbytes

    def __del__(self):
        global _pinned_leased_bytes
        if getattr(self, "ptr", None):
            self.lib.dll.b200gate_host_free(self.ptr)
            _pinned_leased_bytes -= self.nbytes
            self.ptr = None


def result_empty(lib: "GateLibrary", shape, dtype) -> np.ndarray:
    """np.empty(shape, dtype) -- in pooled page-locked memory when the array is large and the budget allows."""
    dtype = np.dtype(dtype)
    nbytes = int(np.prod(shape)) * dtype.itemsize
    if nbytes >= PINNED_RESULT_MIN_BYTES and _pinned_leased_bytes + nbytes <= _pinned_budget_bytes():
        try:
            lease = _PinnedLease(lib, nbytes)
        except MemoryError:
            return np.empty(shape, dtype)
        buf = (C.c_char * nbytes).from_address(lease.ptr)
        buf._b200_lease = lease              # frombuffer keeps `buf` alive, `buf` keeps the lease: freed with the last view
        return np.frombuffer(buf, dtype=dtype).reshape(shape)
    return np.empty(shape, dtype)


_LIB: Optional[GateLibrary] = None


def library() -> GateLibrary:
    """The product library (lazy, cached).  Raises if it has not been built."""
    global _LIB
    if _LIB is None:
        _LIB = GateLibrary(DEFAULT_LIB)
    return _LIB


def dtype_code(dt) -> int:
    dt = np.dtype(dt)
    if dt not in _DTYPES:
        raise TypeError(f"unsupported sample dtype {dt}")
    return _DTYPES[dt]


class Gate:
    """One b200gate handle (RAII)."""

    def __init__(self, lib: Optional[GateLibrary] = None, **kw):
        self.lib = lib or library()
        p = Params()
        p.abi_version = ABI_VERSION
        for k, v in kw.items():
            if not hasattr(p, k):
                raise TypeError(f"unknown b200gate parameter {k}")
            setattr(p, k, v)
        self.params = p
        self._h = C.c_void_p()
        rc = self.lib.dll.b200gate_create(C.byref(p), C.byref(self._h))
        if rc != 0:
            raise GateError(rc, self.lib.dll.b200gate_last_error(None).decode())
        self.n_bins = p.n_fft // 2 + 1

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.dll.b200gate_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise GateError(rc, self.lib.dll.b200gate_last_error(self._h).decode())

    # -- noise statistics ------------------------------------------------------------------------
    def noise_stats_host(self, y2d: np.ndarray, stream=None):
        y2d = np.ascontiguousarray(y2d)
        self._check(self.lib.dll.b200gate_noise_stats(
            self._h, y2d.ctypes.data, dtype_code(y2d.dtype), y2d.shape[0], y2d.shape[1], y2d.shape[1], 0, stream))

    def noise_stats_device(self, ptr, dtype, C_, N, stride, stream=None):
        self._check(self.lib.dll.b200gate_noise_stats(self._h, ptr, dtype_code(dtype), C_, N, stride, 1, stream))

    def channel_sum_device(self, ptr, dtype, C_, n, stride, acc_ptr, init, stream=None):
        self._check(self.lib.dll.b200gate_channel_sum(
            self._h, ptr, dtype_code(dtype), C_, n, stride, 1, acc_ptr, 1 if init else 0, stream))

    def noise_stats_collapsed_device(self, ptr, dtype, n, stream=None):
        self._check(self.lib.dll.b200gate_noise_stats_collapsed(self._h, ptr, dtype_code(dtype), n, 1, stream))

    def set_window(self, window_f32):
        w = np.ascontiguousarray(window_f32, dtype=np.float32)
        self._check(self.lib.dll.b200gate_set_window(self._h, w.ctypes.data_as(C.POINTER(C.c_float)), w.shape[0]))

    def torch_set_noise(self, ptr, Bn, Ln, stride, is_device=True, stream=None, dtype=np.float32):
        self._check(self.lib.dll.b200gate_torch_set_noise(self._h, ptr, dtype_code(dtype), Bn, Ln, stride, 1 if is_device else 0, stream))

    def set_noise_threshold(self, thresh_db):
        t = np.ascontiguousarray(thresh_db, dtype=np.float64)
        self._check(self.lib.dll.b200gate_set_noise_threshold(
            self._h, t.ctypes.data_as(C.POINTER(C.c_double)), t.shape[0]))

    def noise_stats_rows(self, clips, dtype, is_device, stream=None) -> np.ndarray:
        """b200gate_noise_stats_rows on (ptr, C, n, stride) tuples of one dtype; returns the thresholds [len(clips)][n_bins]."""
        arr = (NoiseClip * len(clips))(*clips)
        out = np.empty((len(clips), self.n_bins), dtype=np.float64)
        self._check(self.lib.dll.b200gate_noise_stats_rows(self._h, arr, len(clips), dtype_code(dtype), 1 if is_device else 0,
                                                           out.ctypes.data_as(C.POINTER(C.c_double)), stream))
        return out

    def set_noise_threshold_rows(self, thresh_db):
        """b200gate_set_noise_threshold_rows: one threshold row per recording of the next run_rows calls."""
        t = np.ascontiguousarray(thresh_db, dtype=np.float64)
        self._check(self.lib.dll.b200gate_set_noise_threshold_rows(
            self._h, t.ctypes.data_as(C.POINTER(C.c_double)), t.shape[0], t.shape[1]))

    def noise_threshold(self) -> np.ndarray:
        out = np.empty(self.n_bins, dtype=np.float64)
        self._check(self.lib.dll.b200gate_get_noise_threshold(
            self._h, out.ctypes.data_as(C.POINTER(C.c_double)), self.n_bins))
        return out

    def noise_mean_std(self):
        m = np.empty(self.n_bins, dtype=np.float64)
        s = np.empty(self.n_bins, dtype=np.float64)
        self._check(self.lib.dll.b200gate_get_noise_mean_std(
            self._h, m.ctypes.data_as(C.POINTER(C.c_double)), s.ctypes.data_as(C.POINTER(C.c_double)), self.n_bins))
        return m, s

    # -- the operator ------------------------------------------------------------------------------
    def run_host(self, y2d: np.ndarray, out: Optional[np.ndarray] = None, stream=None) -> np.ndarray:
        y2d = np.ascontiguousarray(y2d)
        if out is None:
            out = result_empty(self.lib, y2d.shape, y2d.dtype)
        self._check(self.lib.dll.b200gate_run(
            self._h, y2d.ctypes.data, out.ctypes.data, dtype_code(y2d.dtype), y2d.shape[0], y2d.shape[1],
            y2d.shape[1], out.shape[1], 0, stream))
        return out

    def run_device(self, in_ptr, out_ptr, dtype, C_, N, in_stride, out_stride, stream=None):
        self._check(self.lib.dll.b200gate_run(
            self._h, in_ptr, out_ptr, dtype_code(dtype), C_, N, in_stride, out_stride, 1, stream))

    def run_rows(self, rows, dtype, is_device, stream=None):
        """b200gate_run_rows on (in_ptr, out_ptr, n, channels of the recording) tuples: one recording channel each (include/b200gate.h)."""
        arr = (Row * len(rows))(*rows)
        self._check(self.lib.dll.b200gate_run_rows(self._h, arr, len(rows), dtype_code(dtype), 1 if is_device else 0, stream))

    def run_sharded(self, in_ptr, dtype, C_local, N, in_stride, gathered_local, gathered_peers, flags_local, flags_peers,
                    epoch, rank, world, groups, push_ctas, compute_stream, comm_stream):
        """b200gate_run_sharded: channel groups into this rank's slice of the gathered buffer + kernel-issued NVLink
        pushes into every peer's copy + device-side epoch barrier (include/b200gate.h)."""
        gp = (C.c_void_p * world)(*[int(p) if p else None for p in gathered_peers])
        fp = (C.c_void_p * world)(*[int(p) if p else None for p in flags_peers])
        self._check(self.lib.dll.b200gate_run_sharded(
            self._h, in_ptr, dtype_code(dtype), C_local, N, in_stride, gathered_local, gp, flags_local, fp, epoch, rank, world,
            groups, push_ctas, compute_stream, comm_stream))

    def torch_apply_masks_device(self, in_ptr, out_ptr, dtype, C_, N, in_stride, out_stride, stream=None):
        self._check(self.lib.dll.b200gate_torch_apply_masks(
            self._h, in_ptr, out_ptr, dtype_code(dtype), C_, N, in_stride, out_stride, 1, stream))

    def torch_apply_masks_rows(self, rows, dtype, is_device, stream=None):
        """b200gate_torch_apply_masks_rows on (in_ptr, out_ptr, n, channels) tuples: the masks of the last run_rows."""
        arr = (Row * len(rows))(*rows)
        self._check(self.lib.dll.b200gate_torch_apply_masks_rows(self._h, arr, len(rows), dtype_code(dtype),
                                                                 1 if is_device else 0, stream))

    # -- kept masks and the adjoint (numpy surface) ---------------------------------------------------------------------
    def mask_store_bytes(self, C_, N) -> int:
        n = C.c_int64()
        self._check(self.lib.dll.b200gate_mask_store_bytes(self._h, C_, N, C.byref(n)))
        return n.value

    def set_mask_store(self, ptr, nbytes=0):
        self._check(self.lib.dll.b200gate_set_mask_store(self._h, ptr, nbytes))

    def adjoint_device(self, store_ptr, g_ptr, grad_ptr, dtype, C_, N, g_stride, grad_stride, stream=None):
        self._check(self.lib.dll.b200gate_adjoint(self._h, store_ptr, g_ptr, grad_ptr, dtype_code(dtype), C_, N, g_stride,
                                                  grad_stride, 1, stream))

    # -- streaming (b200gate_stream_*): pointers and sizes as in the header; the push / finish return n_out --------------
    def stream_begin(self, dtype, C_):
        self._check(self.lib.dll.b200gate_stream_begin(self._h, dtype_code(dtype), C_))

    def stream_push(self, in_ptr, n, in_stride, is_device, out_ptr, out_stride, out_capacity, stream=None) -> int:
        n_out = C.c_int64()
        self._check(self.lib.dll.b200gate_stream_push(self._h, in_ptr, n, in_stride, 1 if is_device else 0, out_ptr,
                                                      out_stride, out_capacity, C.byref(n_out), stream))
        return n_out.value

    def stream_finish(self, out_ptr, out_stride, out_capacity, stream=None) -> int:
        n_out = C.c_int64()
        self._check(self.lib.dll.b200gate_stream_finish(self._h, out_ptr, out_stride, out_capacity, C.byref(n_out), stream))
        return n_out.value

    # -- torch streams (b200gate_tstream_*): device float32 rows; the push / finish return n_out -------------------------
    def tstream_begin(self, n_rows):
        self._check(self.lib.dll.b200gate_tstream_begin(self._h, n_rows))

    def tstream_push(self, in_ptr, n, in_stride, out_ptr, out_stride, out_capacity, stream=None) -> int:
        n_out = C.c_int64()
        self._check(self.lib.dll.b200gate_tstream_push(self._h, in_ptr, n, in_stride, out_ptr, out_stride, out_capacity,
                                                       C.byref(n_out), stream))
        return n_out.value

    def tstream_finish(self, out_ptr, out_stride, out_capacity, stream=None) -> int:
        n_out = C.c_int64()
        self._check(self.lib.dll.b200gate_tstream_finish(self._h, out_ptr, out_stride, out_capacity, C.byref(n_out), stream))
        return n_out.value

    # per-row torch streams: n and rows are int64 numpy arrays; the push / end return n_out as one
    def tstream_push_rows(self, in_ptr, n, in_stride, out_ptr, out_stride, out_capacity, stream=None) -> np.ndarray:
        n_out = np.empty_like(n)
        self._check(self.lib.dll.b200gate_tstream_push_rows(self._h, in_ptr, _i64p(n), in_stride, out_ptr, out_stride,
                                                            out_capacity, _i64p(n_out), stream))
        return n_out

    def tstream_end_rows(self, rows, out_ptr, out_stride, out_capacity, stream=None) -> np.ndarray:
        n_out = np.empty_like(rows)
        self._check(self.lib.dll.b200gate_tstream_end_rows(self._h, _i64p(rows), len(rows), out_ptr, out_stride,
                                                           out_capacity, _i64p(n_out), stream))
        return n_out

    def tstream_reset_rows(self, rows):
        self._check(self.lib.dll.b200gate_tstream_reset_rows(self._h, _i64p(rows), len(rows)))

    def set_range(self, mode: int, a: int = 0, b: int = 0):
        self._check(self.lib.dll.b200gate_set_range(self._h, mode, a, b))

    def stats(self) -> dict:
        s = Stats()
        self._check(self.lib.dll.b200gate_get_stats(self._h, C.byref(s)))
        return s.as_dict()

    # -- parity taps (tests) -----------------------------------------------------------------------
    def debug_select_unit(self, chunk: int, channel: int):
        self._check(self.lib.dll.b200gate_debug_select_unit(self._h, chunk, channel))

    def debug_read(self):
        T, F, W = C.c_int64(), C.c_int32(), C.c_int32()
        self._check(self.lib.dll.b200gate_debug_dims(self._h, C.byref(T), C.byref(F), C.byref(W)))
        T, F, W = T.value, F.value, W.value
        bits = np.zeros((T, W), dtype=np.uint32)
        mask = np.zeros((T, F), dtype=np.float32)
        spec = np.zeros((T, F, 2), dtype=np.float32)
        self._check(self.lib.dll.b200gate_debug_read_bits(self._h, bits.ctypes.data))
        self._check(self.lib.dll.b200gate_debug_read_mask(self._h, mask.ctypes.data))
        self._check(self.lib.dll.b200gate_debug_read_spec(self._h, spec.ctypes.data))
        # unpack to bool [F, T] like the oracle's taps
        b = ((bits[:, :, None] >> np.arange(32, dtype=np.uint32)[None, None, :]) & 1).astype(bool)
        b = b.reshape(T, W * 32)[:, :F]
        return dict(mask0=b.T.copy(), mask=mask.T.copy(), X=(spec[..., 0] + 1j * spec[..., 1]).T.copy())
