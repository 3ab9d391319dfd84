/* b200gate.h -- C ABI of libb200gate.so, the H100-native spectral-gating operator.
 *
 * Drop-in boundary (SURVEY.md section 8b).  Each entry point replaces one piece of the reference
 * (timsainb/noisereduce @ 51c8534, paths relative to the reference checkout):
 *
 *   b200gate_create            <- SpectralGate.__init__ geometry + smoothing-filter extents
 *                                 (noisereduce/spectralgate/base.py:33-128) and the TorchGate
 *                                 constructor (noisereduce/torchgate/torchgate.py:32-71)
 *   b200gate_noise_stats       <- the one-time noise statistics of SpectralGateStationary.__init__
 *                                 (noisereduce/spectralgate/stationary.py:47-81)
 *   b200gate_run               <- SpectralGate.get_traces() -> filter_chunk -> _do_filter over all
 *                                 chunks and channels (base.py:130-226; stationary.py:83-131;
 *                                 nonstationary.py:47-115), i.e. the body of reduce_noise()
 *                                 (noisereduce/noisereduce.py:185), and TorchGate.forward
 *                                 (torchgate.py:200-264) when params.surface == B200GATE_SURFACE_TORCH
 *   b200gate_stream_*          <- the same chunk loop on a recording that arrives block by block, in place of
 *                                 the temp-file memmap the result is written to (base.py:181-187)
 *
 * Conventions: plain pointers and sizes, no torch / numpy types.  All buffers are caller-owned; the
 * library owns only its handle and device workspace.  Every function returns B200GATE_OK (0) or a
 * negative error code; b200gate_last_error() gives the message.  A handle serialises its work on the
 * CUDA stream passed in (0 = legacy default stream); handles are independent, so one per thread /
 * per rank is the threading model.  There is no CPU fallback: without a CUDA device
 * b200gate_create fails with B200GATE_ERR_CUDA.
 */
#ifndef B200GATE_H
#define B200GATE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200GATE_ABI_VERSION 1

enum {
    B200GATE_OK = 0,
    B200GATE_ERR_ARG = -1,          /* bad argument / unsupported geometry                       */
    B200GATE_ERR_CUDA = -2,         /* CUDA runtime error (message has the CUDA error string)    */
    B200GATE_ERR_STATE = -3,        /* call order (e.g. stationary run before noise statistics)  */
    B200GATE_ERR_NOMEM = -4
};

enum { B200GATE_F32 = 0, B200GATE_I16 = 1, B200GATE_F64 = 2 };     /* sample dtypes */
/* further sample formats, taken by b200gate_convert only (the gate itself runs F32 / I16 / F64); BOOL is one byte 0/1 */
enum { B200GATE_BOOL = 3, B200GATE_I8 = 4, B200GATE_U8 = 5, B200GATE_U16 = 6, B200GATE_I32 = 7, B200GATE_U32 = 8,
       B200GATE_I64 = 9, B200GATE_U64 = 10, B200GATE_F16 = 11 };
enum { B200GATE_CONVERT_CAST = 0, B200GATE_CONVERT_CHANNEL_MEAN = 1 };   /* b200gate_convert operations */
/* which reference semantics.  NUMPY: SpectralGate's chunk loop (reduce_noise()).  TORCH: TorchGate.forward on whole rows.
 * TORCH_CHUNKED: reduce_noise(use_torch=True), i.e. the chunk loop of base.py:167-226 around TorchGate
 * (streamed_torch_gate.py:81-88).  Each (chunk, channel) unit is the padded chunk [i cs - pad, (i + 1) cs + pad), zeros
 * outside [0, N), filtered with TorchGate's arithmetic (torch.stft(center=True) framing with the window of
 * b200gate_set_window, per-unit self statistics or the thresholds of b200gate_torch_set_noise, the blend before the
 * smoothing, the moving-mean follower), always in float64 like the reference's float64 chunks; the run writes columns
 * [pad, pad + cs) of each unit's torch-length output ((Lp / hop) * hop + (n_fft & 1) samples, Lp = cs + 2 pad).
 * chunk_size <= 0 (or N <= chunk_size) makes the whole recording one padded chunk [-pad, N + pad).  Ranges and streams
 * work as on the numpy surface.  Refused with B200GATE_ERR_ARG: a padded chunk shorter than 2 win_length ("x must be
 * bigger than ..."), and a chunked run whose torch output is shorter than pad + chunk_size.  A single padded chunk whose
 * torch output is shorter than pad + N writes only its first (torch length - pad) columns, as the reference's slice does. */
enum { B200GATE_SURFACE_NUMPY = 0, B200GATE_SURFACE_TORCH = 1, B200GATE_SURFACE_TORCH_CHUNKED = 2 };

/* Resolved operator parameters.  The Python shims resolve defaults exactly as the reference does
 * (win_length = n_fft, hop_length = win_length // 4, n_grad_* from Hz / ms) and raise the
 * reference's own exceptions; the library re-validates and rejects what this build cannot run. */
typedef struct b200gate_params {
    int32_t abi_version;        /* B200GATE_ABI_VERSION                                          */
    int32_t surface;            /* B200GATE_SURFACE_*                                            */
    int32_t stationary;         /* 1: stationary gate, 0: non-stationary gate                    */
    int32_t n_fft;              /* [8, 8192] if a power of two, else [8, 4096] (Bluestein)         */
    int32_t win_length;         /* 1 <= win_length <= n_fft                                      */
    int32_t hop_length;         /* 1 <= hop_length <= win_length.  n_fft=1024/win=1024/hop=256 (both gates, both
                                 * surfaces) and 2048/2048/512 (numpy surface, non-stationary) run the tuned FP32 kernels; every other
                                 * geometry runs the float64 general family (gate_generic.cuh)    */
    int32_t n_grad_freq;        /* smoothing half-widths; 0,0 = mask smoothing disabled          */
    int32_t n_grad_time;
    int32_t std_ddof;           /* 0 numpy surface (np.std), 1 torch surface (std_mean)          */
    int32_t clip_noise;         /* clip_noise_stationary                                         */
    int32_t n_movemean;         /* torch surface, non-stationary                                 */
    int32_t debug_guard_scale;  /* tests only: multiplies the FP32 guard band (0 = 1x), forcing more
                                 * bins through the FP64 re-decision path                          */
    int32_t reserve_sms;        /* SMs the persistent grids leave free (for a concurrent NCCL collective) */
    int32_t path_flags;         /* kept cross-check variants of the same arithmetic (default 0).  bit 1: do not cache
                                 * spectra between analysis and synthesis (re-transform instead; saves 8 KB of workspace per
                                 * frame pair); bit 2: run the float64 general-geometry family even for a tuned geometry;
                                 * bit 4: two units per warp in the n_fft 1024 FFT kernels
                                 * (the dual forms) instead of one; bit 5: tile-based float-mask smoothing;
                                 * bit 6: the non-stationary follower stores its forward sweep instead of regenerating
                                 * it; bit 7: tap-loop float-mask smoothing instead of the box-sum form; bit 8: stationary
                                 * gate, smooth the binary mask in a separate kernel that stores 16-bit numerators for the
                                 * synthesis kernel to read, instead of inside the synthesis kernel (same integers, more
                                 * workspace and HBM traffic); bit 9: stationary gate, n_fft 1024, one unit per warp: the
                                 * analysis kernel that tracks the top_db row maxima of every bin and loads its samples
                                 * directly does the whole analysis, instead of the kernel that prefetches sample windows
                                 * by bulk copy and leaves the maxima to that kernel only when a frame could reach the
                                 * floor (same arithmetic).  (bit 0 selected a single-pass experiment and bit 3 a
                                 * cp.async staging of k1's sample rows; both were removed and are ignored)           */
    int64_t chunk_size;         /* <= 0: never chunk (torch surface / chunk_size=None)           */
    int64_t padding;
    double sr;
    double prop_decrease;
    double n_std_thresh;        /* n_std_thresh_stationary                                       */
    double top_db;              /* 80 numpy surface, 40 torch surface                            */
    double time_constant_s;     /* numpy surface, non-stationary                                 */
    double thresh_n_mult;       /* thresh_n_mult_nonstationary / n_thresh_nonstationary          */
    double sigmoid_slope;       /* sigmoid_slope_nonstationary / 1 / temp_coeff_nonstationary    */
    double workspace_limit_bytes; /* 0: library default; bounds the per-batch device workspace   */
} b200gate_params;

typedef struct b200gate_handle b200gate_handle;

/* Counters of the last b200gate_run (device-side exactness bookkeeping and launch counts). */
typedef struct b200gate_stats {
    int64_t units;                  /* (chunk, channel) units processed                           */
    int64_t frames;                 /* STFT frames analysed                                       */
    int64_t kernel_launches;        /* kernels launched by the last run                           */
    int64_t bins_rechecked_fp64;    /* mask decisions inside the FP32 guard band, redone in FP64  */
    int64_t bins_unresolved;        /* ... still inside 1e-12 relative after FP64 (expected 0)    */
    int64_t rowfloor_flags;         /* (unit, bin) rows lifted by the top_db floor                */
    int64_t rowfloor_ambiguous;     /* ... whose FP32 decision was inside the guard band (exp. 0) */
    double last_run_ms;             /* device time of the last run, CUDA events on its stream     */
    double last_h2d_ms, last_d2h_ms;
    double k1_ms, smooth_ms, k2_ms; /* per-kernel device time summed over the run's batches       */
    double fused_ms;                /* single-pass kernel (k1/smooth/k2 are 0 when it ran)        */
    int64_t fused_path;             /* 1: the single-pass kernel produced the result              */
    int64_t fused_fallbacks;        /* 1: top_db floor could trigger -> redone on the two-pass path */
} b200gate_stats;

int b200gate_create(const b200gate_params* params, b200gate_handle** out);
void b200gate_destroy(b200gate_handle* h);
const char* b200gate_last_error(const b200gate_handle* h);   /* h == NULL: last create() error */

/* Stationary noise statistics (stationary.py:47-81): channel mean in the input dtype, clip to
 * chunk_size, STFT, dB with top_db floor, per-bin mean/std over time, thresh = mean + n_std*std.
 * y_noise: [C][N] samples, row stride `stride` elements, host or device memory. */
int b200gate_noise_stats(b200gate_handle* h, const void* y_noise, int dtype, int64_t C, int64_t N,
                         int64_t stride, int is_device, void* cuda_stream);
/* Same, from an already collapsed (channel-mean) noise clip of n samples in float64 or float32:
 * used by multi-GPU callers that build the channel mean across ranks themselves. */
int b200gate_noise_stats_collapsed(b200gate_handle* h, const void* noise_mean, int dtype, int64_t n,
                                   int is_device, void* cuda_stream);
/* Channel-order partial sum of the first `n` samples of `C` channels, continuing from *acc_inout
 * (device buffer of n elements: float32 for F32 input, float64 otherwise; ignored if init != 0).
 * Lets ranks chain the reference's sequential float32 channel sum exactly. */
int b200gate_channel_sum(b200gate_handle* h, const void* y, int dtype, int64_t C, int64_t n,
                         int64_t stride, int is_device, void* acc_inout_device, int init,
                         void* cuda_stream);
int b200gate_set_noise_threshold(b200gate_handle* h, const double* thresh_db, int32_t n_bins);
int b200gate_get_noise_threshold(const b200gate_handle* h, double* thresh_db, int32_t n_bins);

/* Per-recording stationary thresholds (reduce_noise_batch with a noise clip per item).
 * b200gate_noise_stats_rows: the thresholds of n_clips noise clips, row r of thresh_out [n_clips][513] (host memory) in
 * every bit what b200gate_noise_stats + b200gate_get_noise_threshold give for clip r on this handle.  Clip r is
 * [C][n] samples of `dtype` with row stride `stride` elements, clipped to chunk_size when clip_noise is set, as
 * b200gate_noise_stats does.  Device clips (is_device = 1) are read in place on cuda_stream; host clips may lie anywhere:
 * their channel sums are taken on the host, in channel order as b200gate_noise_stats does, and only the sums are copied
 * to the device, in one copy.  The clips run in groups whose float64 spectrograms fit the workspace limit
 * (workspace_limit_bytes, or 70 % of the free device memory), one launch per kernel and group; the thresholds are read
 * back once, and the call returns after that synchronise.  The handle's installed thresholds are not touched.
 * B200GATE_ERR_ARG: a geometry other than n_fft = win_length = 1024, hop_length = 256 (or the general family), a clip
 * with a null pointer, no channels or samples, a row stride below n for C > 1, or fewer than win_length samples after
 * clipping (scipy shortens the window for such a clip: b200gate_noise_stats on a handle with win_length = n takes it). */
typedef struct b200gate_noise_clip { const void* x; int64_t C; int64_t n; int64_t stride; } b200gate_noise_clip;
int b200gate_noise_stats_rows(b200gate_handle* h, const b200gate_noise_clip* clips, int64_t n_clips, int dtype,
                              int is_device, double* thresh_out, void* cuda_stream);
/* b200gate_set_noise_threshold_rows: install one threshold row per recording, thresh_db [n_recordings][n_bins = 513],
 * for the next b200gate_run_rows calls (see there).  The tables are built on the host with the arithmetic of
 * b200gate_set_noise_threshold, so a recording's tables equal the ones its row would give as a single set, and go to the
 * device in one copy.  While they are installed b200gate_run, a stationary stream, b200gate_get_noise_threshold and
 * b200gate_get_noise_mean_std return B200GATE_ERR_STATE; b200gate_set_noise_threshold and b200gate_noise_stats return
 * the handle to one set.  B200GATE_ERR_ARG: a handle other than a stationary numpy-surface gate at n_fft 1024, or
 * n_bins != 513. */
int b200gate_set_noise_threshold_rows(b200gate_handle* h, const double* thresh_db, int64_t n_recordings, int32_t n_bins);
int b200gate_get_noise_mean_std(const b200gate_handle* h, double* mean_db, double* std_db, int32_t n_bins);

/* Torch surfaces only: install the analysis/synthesis window the caller built with
 * torch.hann_window (float32, win_length values), so tables match the reference bit for bit. */
int b200gate_set_window(b200gate_handle* h, const float* window, int32_t win_length);
/* Torch surfaces only: thresholds from a noise clip xn [Bn][Ln] (float32; float64 on the general family; Bn == 1 or
 * Bn == C, the rows of a run), as TorchGate.forward(x, xn) (torchgate.py:140-164).  On TORCH_CHUNKED unit
 * (chunk, channel) uses row `channel`.  xn == NULL returns to self-statistics. */
int b200gate_torch_set_noise(b200gate_handle* h, const void* xn, int dtype, int64_t Bn, int64_t Ln,
                             int64_t stride, int is_device, void* cuda_stream);

/* Torch surface only: apply the MASKS OF THE LAST b200gate_run (same [C][N]) to another signal: analysis of `in`, the
 * stored masks, synthesis.  The gate is linear in its input once the masks are fixed and its operator is
 * out = OLA(w B_mask(w frame(in))) / env with a symmetric B_mask, so this call on g / env, times env, is the adjoint:
 * the backward pass of TorchGate.forward (torchgate.py:223-262 builds the masks under no_grad and lets the gradient flow
 * through stft -> * mask -> istft).  Needs the tuned n_fft = 1024 geometry and a forward that fitted one workspace batch. */
int b200gate_torch_apply_masks(b200gate_handle* h, const void* in, void* out, int dtype, int64_t C, int64_t N,
                               int64_t in_stride, int64_t out_stride, int is_device, void* cuda_stream);

/* The operator.  in/out: [C][N] samples of `dtype` with row strides in elements; host or device
 * pointers (is_device).  out may not alias in.  For the torch surface out holds [C][(N/hop)*hop].
 * Returns after the work is enqueued for device pointers; for host pointers it returns after the
 * result is in `out`. */
int b200gate_run(b200gate_handle* h, const void* in, void* out, int dtype, int64_t C, int64_t N,
                 int64_t in_stride, int64_t out_stride, int is_device, void* cuda_stream);

/* Rows of different lengths in one call.  Numpy surface: every row is a recording of its own, one channel of `n`
 * samples, and out[0, n) of row r holds exactly what b200gate_run writes for that channel of its [channels][n] recording -- the chunk
 * grid, the padded span, the frame count and everything derived from them (smoothing edges, overlap-add edge norm,
 * top_db row maxima, the non-stationary follower's sweeps and its choice between regenerating and storing the forward
 * sweep) are taken per row.  The channels of a multi-channel recording are simply consecutive rows: with the thresholds
 * fixed (b200gate_noise_stats / b200gate_set_noise_threshold, once for all rows) a channel's result depends on no other
 * channel in either gate.  With per-recording thresholds installed (b200gate_set_noise_threshold_rows, stationary gate)
 * the rows group into recordings in order: row 0 starts recording 0, and a recording is `channels` consecutive rows
 * of equal n and channels; every unit of recording i compares against row i of the thresholds.  The number of
 * recordings must equal the rows installed (B200GATE_ERR_ARG otherwise, as for a recording whose rows differ in n or
 * channels or that runs past the last row).  With one set installed nothing of this applies.
 * The units of all rows share the workspace at the pitch of the call's longest unit.
 * Device pointers (is_device = 1) are read and written where they are and the call only enqueues on cuda_stream, without
 * waiting for the device.  Host rows must lie in one buffer each way: they travel as the span that covers them, one copy
 * in and one copy out (bytes of the output span between rows are overwritten), and the call returns with the result in
 * place.  b200gate_get_stats counts the units of all rows and their own frames.
 * Torch surface (B200GATE_SURFACE_TORCH): every row is one TorchGate row of n >= 2 win_length float32 samples, filtered
 * as b200gate_run filters a [1][n] input -- one unit with origin 0 and no chunk padding, zeros outside [0, n), T = n / hop
 * + 1 frames, statistics over the row's own frames (or the thresholds of b200gate_torch_set_noise: one row for every row
 * of the call, or row r for row r) -- and out[0, (n / hop) * hop + (n_fft & 1)) of row r holds the result.  Device rows
 * are written there and nowhere else.  Host rows travel as the output span that covers them, zeroed on the device first:
 * every byte of that span outside the rows' results (samples [(n / hop) * hop, n) of a row, gaps between rows) is
 * overwritten with zeros.  `channels` keeps its meaning (TorchGate passes 1).  Stationary smoothing extents beyond the
 * in-synthesis smoothing run through a separate numerator kernel, up to the 16-bit numerator limit below.  The masks of a call that fits one workspace batch stay on the handle for
 * b200gate_torch_apply_masks_rows.
 * B200GATE_ERR_STATE: the TORCH_CHUNKED surface, an open stream, a mask store set, a range mode other than 0, a
 * numpy-surface stationary gate without thresholds.  B200GATE_ERR_ARG: a geometry other than n_fft = win_length = 1024,
 * hop_length = 256; a smoothing filter that b200gate_create sent to the general family ((n_grad_freq + 1)^2
 * (n_grad_time + 1)^2 > 65535, or either extent > 64); non-zero path_flags; smoothing extents beyond the in-synthesis smoothing (numpy surface, stationary:
 * n_grad_time > 13 or n_grad_freq > 17) or beyond the streaming float-mask smoothing; n <= 0, channels <= 0, a null
 * pointer, out overlapping in; scattered host rows; on the torch surface a dtype other than B200GATE_F32, a row shorter
 * than 2 win_length ("x must be bigger than ..."), xn thresholds of more than one row that are not one per row.  A
 * refused call changes nothing on the handle. */
typedef struct b200gate_row {
    const void* in; void* out; int64_t n;
    int64_t channels;   /* rows of the recording this row is a channel of (>= 1).  Sizes the synthesis work items as
                         * b200gate_run does for a [channels][n] recording that fits one workspace batch: the last bit
                         * of the hops at work-item seams depends on that length, everything else does not */
} b200gate_row;
int b200gate_run_rows(b200gate_handle* h, const b200gate_row* rows, int64_t n_rows, int dtype, int is_device,
                      void* cuda_stream);
/* Torch surface: the rows form of b200gate_torch_apply_masks -- apply the masks of the last b200gate_run_rows on this
 * handle to another set of rows with the same n, row by row (analysis of `in`, the stored masks, synthesis), i.e. the
 * backward pass of TorchGate.forward(x, lengths=...).  B200GATE_ERR_STATE when the last run was not a rows run, its
 * masks did not fit one workspace batch, or the row count or an n differs. */
int b200gate_torch_apply_masks_rows(b200gate_handle* h, const b200gate_row* rows, int64_t n_rows, int dtype, int is_device,
                                    void* cuda_stream);

/* Sub-range processing for the next b200gate_run calls (SpectralGate.get_traces(start_frame, end_frame),
 * base.py:167-226).  mode 0: the whole recording (default).  mode 1: only chunks [a, b] of the chunk grid
 * anchored at sample 0 (the reference's chunked branch); samples outside those chunks are not written.
 * mode 2: one padded chunk covering [0, a) whose padding is read from the recording itself (the reference's
 * `filter_chunk(0, end_frame)` branch, base.py:222); only out[:, 0:a] is written.
 * In modes 1 and 2 `out` is still the address of (row 0, sample 0), but only the range is addressed: a caller
 * may pass `slab - first_sample` with out_stride = the slab's row pitch (>= the range length) to have the range
 * written densely into a [C][range] slab (noisereduce_b200/parallel.py gathers such slabs across GPUs). */
int b200gate_set_range(b200gate_handle* h, int32_t mode, int64_t a, int64_t b);

/* ---- the adjoint: backpropagation through b200gate_run (numpy surface) ---------------------------------------------
 * With its masks held fixed (the thresholds, decisions, top_db row flags and the non-stationary noise floor are
 * constants, as in TorchGate's backward, torchgate.py:223-262), unit u = (chunk i, channel c) of a run is a linear map of
 * its padded span: y_u = crop(D^-1 OLA(w P w frame(pad_u y))), P = irfft diag(M) rfft cut to the frame (a symmetric
 * matrix), D = sum of w^2 (1 where <= 1e-10).  b200gate_adjoint computes grad = A^T g, the sum over units of the same
 * re-transforming synthesis run on g / D over the unit's centre (zero elsewhere, including centre samples the forward
 * leaves at zero), with an un-normalised overlap-add over the whole padded span [i cs - pad, (i + 1) cs + pad) clipped to
 * [0, N).  Spans of overlapping units are added in increasing unit order without atomics: the result is the same in every
 * bit from run to run and for any workspace limit.
 *
 * b200gate_mask_store_bytes: the size of the masks a run of [C][N] keeps, in the handle's current range mode.
 * b200gate_set_mask_store: a caller-owned device buffer of `bytes` bytes (NULL: keep nothing, the default).  While it is
 *   set, each b200gate_run writes its final masks there instead of to the workspace -- the same kernels and the same
 *   bits, no extra traffic: stationary n_fft 1024, the decision words and top_db row flags (68 B per frame and unit); the
 *   non-stationary gate (n_fft 1024 and 2048), the float masks; the general family, the float64 masks.  A run whose masks do not
 *   fit returns B200GATE_ERR_ARG.  Streams never keep masks.
 * b200gate_adjoint: grad [C][N] (row stride grad_stride, every sample written) = A^T g for the run whose masks are in
 *   `store` (same C, N and range mode as that run; B200GATE_ERR_STATE otherwise).  g is read on the samples the run
 *   wrote only, so in range modes 1 and 2 it may be a virtual base like `out` (g_stride >= the range length).  dtype
 *   B200GATE_F32 or B200GATE_F64 for both g and grad (the n_fft 2048 kernels read float32 rows: a float64 g is converted
 *   through the handle's staging buffer); device pointers only (is_device = 1); enqueued on cuda_stream.
 *   The adjoint grows the handle's workspace as a run does (the per-unit span and numerators, within the workspace
 *   limit); it stays allocated until the handle is destroyed.
 * All three refuse the torch surfaces (B200GATE_ERR_STATE; their backward is b200gate_torch_apply_masks). */
int b200gate_mask_store_bytes(b200gate_handle* h, int64_t C, int64_t N, int64_t* bytes);
int b200gate_set_mask_store(b200gate_handle* h, void* store, int64_t bytes);
int b200gate_adjoint(b200gate_handle* h, const void* store, const void* g, void* grad, int dtype, int64_t C, int64_t N,
                     int64_t g_stride, int64_t grad_stride, int is_device, void* cuda_stream);

/* ---- streaming: a recording that arrives block by block (numpy or TORCH_CHUNKED surface, chunk_size > 0) ----------
 * The reference holds the whole [C][N] input and writes the result to a temp-file memmap (base.py:181-187).  A stream
 * returns each chunk as soon as its padded span has arrived, and the concatenation of everything it returns is
 * bit-identical to b200gate_run on the concatenated input.  Output chunk i (samples [i cs, (i + 1) cs)) reads only input
 * [i cs - pad, (i + 1) cs + pad), zero outside [0, N) (base.py:130-156); a recording of N <= cs samples is one padded
 * chunk (base.py:222), which is only known at the end.  So after R samples have been received, exactly
 *     E(R) = cs * max(0, floor((R - pad) / cs))  if R > cs,   E(R) = 0 otherwise
 * have been returned: the latency is at most cs + pad - 1 samples.
 *
 * b200gate_stream_begin starts (or restarts) a stream of C channels of `dtype` on the handle.  The handle then keeps a
 * device window of samples [max(0, E - pad), R) of every channel; its size depends on chunk_size, padding and C only,
 * not on the stream length or the block sizes (a long push is consumed in slices of whole chunks).
 * b200gate_stream_push appends samples [0, n) of each row of `in` (row stride in_stride) and writes the next *n_out
 * samples of the result to out[c][0, *n_out).  in and out are host pointers, or device pointers with is_device = 1
 * (then the call only enqueues on cuda_stream; *n_out is known at once).  Every push of a stream uses the same memory
 * space; b200gate_stream_finish writes the rest of the result (< chunk_size + padding samples) into that space and
 * closes the stream.  Errors: out_capacity < n + chunk_size (push) or < chunk_size + padding (finish): B200GATE_ERR_ARG
 * before anything is written; a stationary gate without noise thresholds (b200gate_noise_stats /
 * b200gate_set_noise_threshold, which may be called while the stream is open) when a chunk would be returned:
 * B200GATE_ERR_STATE.  While a stream is open b200gate_run on the handle returns B200GATE_ERR_STATE.  After any other
 * error the stream is closed.  On TORCH_CHUNKED every unit can take its own statistics, so no thresholds are needed;
 * the single padded chunk of a recording of R <= chunk_size samples may return fewer than R samples (see the surface). */
int b200gate_stream_begin(b200gate_handle* h, int dtype, int64_t C);
int b200gate_stream_push(b200gate_handle* h, const void* in, int64_t n, int64_t in_stride, int is_device,
                         void* out, int64_t out_stride, int64_t out_capacity, int64_t* n_out, void* cuda_stream);
int b200gate_stream_finish(b200gate_handle* h, void* out, int64_t out_stride, int64_t out_capacity,
                           int64_t* n_out, void* cuda_stream);

/* ---- TorchGate.stream(): the non-stationary TorchGate on rows that arrive block by block ---------------------------
 * For a B200GATE_SURFACE_TORCH handle with stationary = 0 at n_fft = win_length = 1024, hop_length = 256 (any other
 * handle: B200GATE_ERR_STATE).  Every stage of that gate looks ahead a bounded distance, so after R samples per row
 *     hb(R) = 2 floor(nS / 2),  nS = 2 floor(c / 2) - 1 - right - n_grad_time,  c = floor((R - 512) / 256) + 1
 * (right = n_movemean - 1 - (n_movemean - 1) / 2) and the samples [0, 256 max(0, hb(R) - 2)) of every row are final.
 * The concatenation of everything a stream returns is bit-identical to b200gate_run on the concatenated rows.
 * b200gate_tstream_begin starts (or restarts) a stream of n_rows rows; its device state depends on n_rows and the
 * parameters only.  b200gate_tstream_push appends samples [0, n) of each row of `in` (device float32 rows, stride
 * in_stride) and writes the *n_out samples that became final to out[b][0, *n_out) (stride out_stride); it only enqueues
 * on cuda_stream.  b200gate_tstream_finish writes the rest of the (R / 256) 256 samples and closes the stream (it frees the
 * stream's device state, which waits for the device).  Errors: out_capacity below what the call returns: B200GATE_ERR_ARG,
 * the stream unchanged; finish with R < 2 win_length: B200GATE_ERR_ARG ("x must be bigger than 2048"), the stream stays
 * open.  While a torch stream is open b200gate_run, b200gate_run_rows, b200gate_torch_apply_masks(_rows) and
 * b200gate_stream_* return B200GATE_ERR_STATE. */
int b200gate_tstream_begin(b200gate_handle* h, int64_t n_rows);
int b200gate_tstream_push(b200gate_handle* h, const float* in, int64_t n, int64_t in_stride, float* out, int64_t out_stride,
                          int64_t out_capacity, int64_t* n_out, void* cuda_stream);
int b200gate_tstream_finish(b200gate_handle* h, float* out, int64_t out_stride, int64_t out_capacity, int64_t* n_out,
                            void* cuda_stream);

/* ---- TorchGate.sessions(): one torch stream whose rows each hold their own session ----------------------------------
 * The per-row form of a stream opened by b200gate_tstream_begin.  A row's session is the samples it receives between
 * the stream's start, or the b200gate_tstream_end_rows / _reset_rows that last emptied the row, and its end; everything
 * returned for it is bit-identical to b200gate_run on the session's samples alone, and after R samples of a session
 * exactly 256 max(0, hb(R) - 2) of its output samples have been returned (hb as above).  A stream takes either the
 * lockstep calls (b200gate_tstream_push / _finish) or these; the other kind returns B200GATE_ERR_STATE.
 * b200gate_tstream_push_rows appends samples [0, n[b]) of row b of `in` (device float32 rows, stride in_stride) to row
 * b's session for every row b, and writes the n_out[b] samples of row b that became final to out[b][0, n_out[b])
 * (stride out_stride).  b200gate_tstream_end_rows ends the sessions of rows[0, k): the rest of row rows[i]'s output,
 * n_out[i] samples, goes to out[i][0, n_out[i]), and the row is empty again.  Both only enqueue on cuda_stream; the row
 * tables travel through a ring of 16 pinned slots, and a call waits only when the device is 16 slices behind (a push
 * is one slice per 4096 samples of its longest row, an end one slice).  b200gate_tstream_reset_rows drops the sessions
 * of rows[0, k) without output.  Errors, all before any change to the stream: B200GATE_ERR_ARG for a negative n[b],
 * in_stride below the largest n[b], rows out of [0, n_rows) or listed twice, out_capacity below what the call returns,
 * and an end of a row holding fewer than 2 win_length samples ("x must be bigger than 2048").  The stream's device
 * state is fixed by b200gate_tstream_begin and released by b200gate_destroy. */
int b200gate_tstream_push_rows(b200gate_handle* h, const float* in, const int64_t* n, int64_t in_stride, float* out,
                               int64_t out_stride, int64_t out_capacity, int64_t* n_out, void* cuda_stream);
int b200gate_tstream_end_rows(b200gate_handle* h, const int64_t* rows, int64_t k, float* out, int64_t out_stride,
                              int64_t out_capacity, int64_t* n_out, void* cuda_stream);
int b200gate_tstream_reset_rows(b200gate_handle* h, const int64_t* rows, int64_t k);

int b200gate_get_stats(const b200gate_handle* h, b200gate_stats* out);

/* ---- sample formats of device-resident callers ----------------------------------------------------------------------
 * The reference runs any dtype other than float32 / int16 / float64 through float64 (base.py:140) and casts the result
 * back with ndarray.astype (base.py:218-226); its stationary thresholds start from np.mean(noise, axis=0) in the clip's
 * own dtype rules (stationary.py:61).  For samples already on the device these steps are kernels, bit-identical to
 * numpy on x86-64 (noisereduce_b200/csrc/gate_convert.cuh has the rules):
 *   B200GATE_CONVERT_CAST: dst[c][j] = src[c][j] for c < C, j < N, converted; one of src_dtype / dst_dtype is
 *     B200GATE_F64.  To float64 the cast is exact except for 64-bit integers beyond 2^53 (round to nearest even); from
 *     float64 it is ndarray.astype on unit-stride rows: float16 rounds once, bool is v != 0, integers truncate, and
 *     NaN, +-inf and out-of-range values map as x86-64's cvttsd2si does.
 *   B200GATE_CONVERT_CHANNEL_MEAN: dst[j] = mean over c of src[c][j], j < N, as float64 (dst_dtype B200GATE_F64,
 *     dst_stride ignored): float16 / float32 sum in float32 in channel order and float16 rounds the mean to half; every
 *     other format sums in float64 in channel order.  (numpy sums pairwise over a contiguous axis: for channel-adjacent
 *     layouts this equals np.mean of the row-major copy.)
 * src / dst are device pointers (may be NULL when there is nothing to convert) with row strides in elements (>= N
 * when C > 1).  No handle: the work is enqueued on
 * cuda_stream on the current device, and the call returns without waiting.  Errors are read with
 * b200gate_last_error(NULL). */
int b200gate_convert(int op, const void* src, int src_dtype, int64_t src_stride, void* dst, int dst_dtype,
                     int64_t dst_stride, int64_t C, int64_t N, void* cuda_stream);

/* Page-locked host buffers from the library's process-wide pool (the same pool the slab pipeline stages pageable
 * caller memory through).  A result array the reference would np.empty() (base.py:181-187 uses a temp-file memmap)
 * can be leased here instead: b200gate_run then copies device -> host straight into it at PCIe speed, with no page
 * faults and no staging copy, and a freed buffer is handed to the next call of the same size without paying
 * cudaMallocHost (~0.1 s per GB) again.  b200gate_host_alloc returns NULL when the memory cannot be pinned (callers fall
 * back to ordinary memory); b200gate_host_free(NULL) is a no-op.  Thread-safe. */
void* b200gate_host_alloc(size_t bytes);
void b200gate_host_free(void* p);

/* ---- multi-GPU (one process per GPU; SURVEY.md section 8e) ---------------------------------------------------
 * The path's one collective -- the all-gather of the final waveform -- is done with NVLink stores issued by a kernel
 * into buffers every peer has mapped (cudaIpc / CUDA VMM / torch symmetric memory), not with a library collective:
 * the interface therefore takes plain device pointers (this rank's buffer and its mappings of the peers' buffers)
 * instead of the ncclComm_t the survey sketched; NCCL / torch.distributed stays the caller's business (rendezvous,
 * the chained channel mean of the stationary threshold -- b200gate_channel_sum).
 *
 * b200gate_run_sharded: denoise this rank's [C_local][N] channels (device pointers) group by group into rows
 * [rank*C_local, (rank+1)*C_local) of `gathered_local` ([world*C_local][N], this rank's copy of the result) on
 * `compute_stream`, and push every finished group into the same rows of each peer's copy on `comm_stream` while
 * the next group is computed; a device-side barrier over the flag arrays (world uint32 each, zero-initialised,
 * `epoch` strictly increasing per call) ends the step.  On return everything is enqueued; after `compute_stream`
 * reaches this point `gathered_local` holds every rank's rows.  gathered_peers[r] / flags_peers[r] are this rank's
 * mappings of rank r's buffers (entry [rank] is ignored / the local array).  push_ctas = the number of SMs the copy kernel
 * occupies (each of its CTAs fills one SM; create the handle with reserve_sms >= push_ctas); <= 0 picks 12. */
int b200gate_run_sharded(b200gate_handle* h, const void* in_local, int dtype, int64_t C_local, int64_t N,
                         int64_t in_stride, void* gathered_local, void* const* gathered_peers, void* flags_local,
                         void* const* flags_peers, uint32_t epoch, int32_t rank, int32_t world, int32_t groups,
                         int32_t push_ctas, void* compute_stream, void* comm_stream);
/* The two building blocks, for callers with their own schedule (e.g. the slab ring of config 5): copy `rows` rows of
 * `row_bytes` bytes (16-byte multiples, 16-byte aligned) from local memory into n_peers mapped buffers; and the
 * epoch barrier described above. */
int b200gate_peer_push(const void* src, void* const* peer_dst, int32_t n_peers, int64_t rows, int64_t row_bytes,
                       int64_t src_stride_bytes, int64_t dst_stride_bytes, int32_t n_ctas, void* cuda_stream);
int b200gate_peer_barrier(void* local_flags, void* const* peer_flags, int32_t rank, int32_t world, uint32_t epoch,
                          void* cuda_stream);

/* ---- parity-test taps (tests/ only; read back stage outputs of the last run) ---------------- */
/* Select the (chunk, channel) unit whose stages the next run keeps.  chunk < 0 disables. */
int b200gate_debug_select_unit(b200gate_handle* h, int64_t chunk, int64_t channel);
/* Frames of the tapped unit; bits: [T][words] packed mask decisions (bit f%32 of word f/32),
 * with the top_db row floor already folded in.  mask: [T][F] smoothed multiplicative mask.
 * spec: [T][F][2] float, the FP32 STFT (re, im) as the analysis kernel saw it. */
int b200gate_debug_dims(const b200gate_handle* h, int64_t* T, int32_t* F, int32_t* words);
int b200gate_debug_read_bits(b200gate_handle* h, uint32_t* bits);
int b200gate_debug_read_mask(b200gate_handle* h, float* mask);
int b200gate_debug_read_spec(b200gate_handle* h, float* spec);

#ifdef __cplusplus
}
#endif
#endif /* B200GATE_H */
