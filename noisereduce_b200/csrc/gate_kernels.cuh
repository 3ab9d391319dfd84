// gate_kernels.cuh -- sm_100a kernels of the spectral-gating hot path (n_fft = 1024 family).
//
// Reference semantics restated by these kernels (paths relative to the reference checkout):
//   framing / STFT          scipy.signal.stft as called at noisereduce/spectralgate/stationary.py:87-93
//   dB floor + threshold    spectralgate/utils.py:11-16, stationary.py:96-110
//   mask smoothing          base.py:7-29 filter, fftconvolve(..., "same") at stationary.py:114
//   apply + iSTFT           stationary.py:117-126 (scipy.signal.istft)
//   chunk geometry          base.py:130-156, :167-226
//
// Work decomposition.  A *unit* is one (chunk, channel) pair -- the reference's _do_filter runs them
// independently (stationary.py:86), so they are the grid.  Inside a unit every warp is an autonomous
// worker that owns a run of consecutive STFT frames; it transforms TWO real frames per 1024-point
// complex FFT (frame a in the real part, frame b = next frame in the imaginary part) held entirely in
// its registers (warp_fft.cuh).  No warp ever waits for another warp.
//
//   k1_analyze    frames -> FFT -> |X|^2 against per-bin power thresholds -> 1 bit/bin mask words
//                 (+ per-(unit,bin) running max for the top_db floor, + FP64 re-decision of bins
//                 whose FP32 margin is inside a proven guard band, so decisions equal the float64
//                 reference's)
//   k_rowfloor    top_db floor:  max_t dB - top_db > thresh  <=>  lift the whole row
//   k_smooth      separable triangular smoothing of the binary mask in exact integer arithmetic
//                 (the reference's FFT convolution approximates exactly these rationals)
//   k2_synthesize frames -> FFT -> mask apply on the packed spectrum -> inverse FFT -> window ->
//                 overlap-add in registers -> normalise -> store the chunk centre
#pragma once
#include "warp_fft.cuh"

namespace b200 {

constexpr int kN = 1024;            // n_fft handled by this kernel family
constexpr int kF = kN / 2 + 1;      // 513 bins
constexpr int kFW = (kF + 31) / 32; // 17 mask words per frame
constexpr int kFPad = kFW * 32;     // 544: padded bin count (tables, mask row pitch)
constexpr int kWarps = 4;           // warps per CTA for k1/k2 (each warp is independent)
constexpr int kThreads = kWarps * 32;
#ifndef B200_K1_MINBLOCKS
#define B200_K1_MINBLOCKS 4          // k1 fits 128 registers: 16 warps per SM
#endif

struct Geom {
    int H;                  // hop
    int C;                  // channels
    int T;                  // frames per padded chunk: Lp / H + 1
    int n_chunks;
    long long n_total;      // samples per channel
    long long step;         // chunk_size (or n_total when there is a single chunk)
    long long pad;          // padding
    long long Lp;           // padded chunk length: step + 2 pad
    long long in_stride, out_stride;   // elements between channel rows
    int u0, n_units;        // this batch: units [u0, u0 + n_units); u = chunk * C + channel
};

// b200gate_run_rows: every unit of a call carries its own geometry and row pointers (kernels templated with ROWS read
// them from units[g.u0 + ul]; Geom then holds what the units share -- H, pad, u0, n_units -- and T = the longest unit's
// frame count, the pitch of every per-unit buffer).
struct UnitDesc {
    const void* x;          // sample 0 of the unit's input row
    void* y;                // sample 0 of its output row
    long long n_total;      // samples of the row
    long long i1;           // first sample of the padded span (may be < 0)
    long long Lp;           // padded span length
    long long o_lo, o_hi;   // samples of the row this unit writes
    int T;                  // frames: Lp / H + 1
    int tf_hi;              // masks are needed for frames [tf_lo, tf_hi) (tf_lo is the same for every unit)
    union {
        int regen;          // non-stationary gate, k_iir_sigmoid: iir_regen_ok of this unit's T
        int rec;            // stationary gate with per-recording thresholds (k1_analyze<.., PERREC>, k_rowfloor_rec):
                            // the unit's recording, its row of the threshold tables
    };
    int run;                // k2c_synthesize: output hops per work item, as run_core sizes them for this unit's recording
};

// TorchGate.stream() (b200gate_tstream_*): the kernels templated with STREAM address global frame t of a row in slot
// t & (ring - 1) of the row's frame rings (|X|, masks: ring rows of FPad floats; spectra: ring / 2 frame pairs), and
// k1n_magnitude / k_tgate_movmean start at global frame f0.  ring is a power of two, so pairs (2j, 2j+1) are adjacent.
struct StreamWin {
    int f0;
    int ring;
};

// TorchGate.sessions() (b200gate_tstream_push_rows / _end_rows): every row of a stream holds its own session, so the
// kernels templated with SESS (always with STREAM) read the row's window and frame ranges from this table, one entry per
// row, rewritten for every slice of a push.  An empty range is a row with nothing to do in that stage.
struct SessRow {
    long long R;            // samples of the row's session, this slice's included
    long long lo;           // the window holds samples [lo, R): sample j at win[row][j - lo]
    long long y;            // output sample j of the session goes to y[this + j] (K2Args::y)
    long long keep, shift;  // k_sess_copy_in: keep samples move from win[row][shift] to win[row][0] (shift > 0 only);
                            // then n samples of in[row][off, off + n) are appended at win[row][keep]
    int n;
    int a0, a1;             // analysis frames [a0, a1), a0 even
    int m0, m1;             // moving-mean frames
    int s0, s1;             // smoothing frames
    int ha, hb;             // synthesis hops [ha, hb), ha even
    int T;                  // the frame bound: INT_MAX while the session is live, R / H + 1 in the end() that finishes it
};

struct SessCopyArgs {
    const float* in;        // [rows][in_stride]; this slice starts at column off
    long long in_stride, off;
    float* win;             // [rows][cap]
    long long cap;
    const SessRow* rows;
};

// One CTA per row.  keep < 2 H + n_fft <= shift (the window pitch leaves that much room behind the kept span), so the
// move reads and writes disjoint spans; the append, which may overwrite the span moved from, follows a barrier.
__global__ void __launch_bounds__(256) k_sess_copy_in(const SessCopyArgs a) {
    const int b = blockIdx.x;
    const SessRow& r = a.rows[b];
    if (r.n == 0) return;
    float* w = a.win + (long long)b * a.cap;
    if (r.shift > 0)
        for (long long i = threadIdx.x; i < r.keep; i += blockDim.x) w[i] = w[r.shift + i];
    __syncthreads();
    const float* src = a.in + (long long)b * a.in_stride + a.off;
    for (long long i = threadIdx.x; i < r.n; i += blockDim.x) w[r.keep + i] = __ldg(src + i);
}

struct Tables {              // device pointers, built once per handle
    const float* wa;         // [N] analysis window / sum(w)
    const float* ws;         // [N] synthesis window * sum(w) / N
    const float2* tw;        // [32*32] radix-32 inter-pass twiddles
    const float* invn;       // [H] 1 / sum_i w^2[i H + r]  (interior overlap-add norm)
    const float* thr4;       // [FPad] 4 * T_amp^2, T_amp = 10^(thresh/20) - eps
    const float* gco;        // [FPad] guard-band coefficient: 4 * T_amp * kappa * eps32
    const float* floor4;     // [FPad] 4 * (10^((thresh + top_db)/20) - eps)^2
    const float* ef;         // [FPad] frequency edge factor of the smoothing filter
    const double* thr2_64;   // [F]  T_amp^2 in float64
    // (per-recording thresholds, b200gate_set_noise_threshold_rows: thr4 / gco / floor4 are [R][FPad] and thr2_64 is
    //  [R][F], one row per recording; slot FPad - 1 of a floor4 row holds the recording's min_floor4, see K1Args)
    const double* wa64;      // [N]  analysis window / sum(w), float64
    const double2* cs64;     // [N]  (cos, sin)(2 pi m / N), float64
    float ws_to_w;           // raw window = ws * ws_to_w
};

struct Counters {
    unsigned long long rechecked, unresolved, floor_flags, floor_ambiguous;
};

struct DebugTap {
    int ul;                  // local unit index to tap, -1 = off
    float* spec;             // [T][F][2]
    float* mask;             // [T][F]
};

// Mask numerators are stored as uint16 pairs, element [pair j][bin k][frame 2j + {0, 1}], so that the synthesis
// kernel fetches both frames of a pair with one 32-bit access; a unit owns ceil(T/2) pair rows of 2*FPad values.
__host__ __device__ __forceinline__ long long num_index(int t, int k) {
    return (((long long)(t >> 1) * kFPad + k) << 1) + (t & 1);
}
__host__ __device__ __forceinline__ long long num_unit_stride(int T) { return (long long)((T + 1) / 2) * (2 * kFPad); }

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One sample of the zero-extended padded chunk (base.py:130-142 zeros outside [0, n_total);
// scipy boundary='zeros' outside [0, Lp)).  j: chunk-local index, i1: global index of j = 0.
// The kernels read the caller's samples in their own dtype (float32 / int16 / float64) and convert on
// load -- the device-side form of base.py:140's promotion -- and k2 casts on store (base.py:218-226).
// u16 halves of a packed word -> float without the (quarter-rate) I2F unit: 2^23 + n as a float bit pattern, minus 2^23
// (exact for n < 2^23): integer-pipe bit operations and one FADD instead.
__device__ __forceinline__ float u16lo_to_float(unsigned pk) {
    return __uint_as_float((pk & 0xFFFFu) | 0x4B000000u) - 8388608.0f;
}
__device__ __forceinline__ float u16hi_to_float(unsigned pk) {
    return __uint_as_float((pk >> 16) | 0x4B000000u) - 8388608.0f;      // (the compiler emits one PRMT / LOP3)
}

template <typename T>
__device__ __forceinline__ float ld_sample(const T* p) { return (float)__ldg(p); }
template <typename T>
__device__ __forceinline__ double ld_sample_f64(const T* p) { return (double)__ldg(p); }
template <typename T>
__device__ __forceinline__ T st_cast(float v);
template <> __device__ __forceinline__ float st_cast<float>(float v) { return v; }
template <> __device__ __forceinline__ double st_cast<double>(float v) { return (double)v; }
template <> __device__ __forceinline__ short st_cast<short>(float v) { return (short)(int)v; }   // numpy astype: truncate, wrap

template <typename T>
__device__ __forceinline__ float chunk_sample(const T* __restrict__ xrow, long long j, long long i1,
                                              long long Lp, long long n_total) {
    const long long g = i1 + j;
    return (j >= 0 && j < Lp && g >= 0 && g < n_total) ? ld_sample(xrow + g) : 0.0f;
}
template <typename T>
__device__ __forceinline__ double chunk_sample_f64(const T* __restrict__ xrow, long long j, long long i1,
                                                   long long Lp, long long n_total) {
    const long long g = i1 + j;
    return (j >= 0 && j < Lp && g >= 0 && g < n_total) ? ld_sample_f64(xrow + g) : 0.0;
}

// Rows of a frame pair: frame t is rows 0..31, frame t+1 rows HR..31+HR of the same 32+HR row window
// (row = 32 consecutive samples = one coalesced 128-byte access of the warp).
template <int HR>
__device__ __forceinline__ bool pair_window_interior(long long base, long long i1, long long Lp, long long n_total) {
    const long long g0 = i1 + base;
    const int span = 32 * (32 + HR);
    return base >= 0 && base + span <= Lp && g0 >= 0 && g0 + span <= n_total;
}

// Load the raw samples of the pair (coalesced 128-byte rows straight into FFT order), window them and pack
// the two frames as one complex signal.  Returns this lane's contribution to ||frame pair||^2.
// (Measured and dropped: prefetch.global.L1 of the next pair's rows -- no effect -- and a register pre-load
//  of them -- more bookkeeping than hidden latency.)
template <int HR>
__device__ __forceinline__ float pack_frame_pair(float (&re)[32], float (&im)[32], const float (&xr)[32 + HR],
                                                 const float* __restrict__ s_wa, int lane, bool vb) {
    float e = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) {
        const float w = s_wa[lane + 32 * r];
        re[r] = xr[r] * w;
        im[r] = xr[r + HR] * w;
        e = fmaf(re[r], re[r], e);
    }
    if (vb) {
#pragma unroll
        for (int r = 0; r < 32; ++r) e = fmaf(im[r], im[r], e);
    } else {                                         // odd frame count: the pair's second frame does not exist
#pragma unroll
        for (int r = 0; r < 32; ++r) im[r] = 0.f;
    }
    return e;
}

template <int HR, typename T>
__device__ __forceinline__ void load_pair_rows(float (&xr)[32 + HR], const T* __restrict__ xrow, long long base,
                                               long long i1, long long Lp, long long n_total, int lane) {
    if (pair_window_interior<HR>(base, i1, Lp, n_total)) {
        const T* p = xrow + i1 + base + lane;
#pragma unroll
        for (int r = 0; r < 32 + HR; ++r) xr[r] = ld_sample(p + 32 * r);
    } else {                                         // chunk / recording edges: zero-extended samples
#pragma unroll
        for (int r = 0; r < 32 + HR; ++r) xr[r] = chunk_sample(xrow, base + lane + 32 * r, i1, Lp, n_total);
    }
}

template <int HR, typename T>
__device__ __forceinline__ float load_frame_pair(float (&re)[32], float (&im)[32], const T* __restrict__ xrow,
                                                 long long base, long long i1, long long Lp, long long n_total,
                                                 const float* __restrict__ s_wa, int lane, bool vb) {
    float xr[32 + HR];
    load_pair_rows<HR>(xr, xrow, base, i1, Lp, n_total, lane);
    return pack_frame_pair<HR>(re, im, xr, s_wa, lane, vb);
}

// Asynchronous global -> shared copies (LDGSTS): the next frame pair's cached spectrum is requested one whole
// iteration before it is needed and costs no registers while in flight.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
#ifdef B200_CUSIM_BUILD
    memcpy(smem_dst, gmem_src, 16);
#else
    const unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem_src));
#endif
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
#ifndef B200_CUSIM_BUILD
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
#endif
}
__device__ __forceinline__ void cp_async_commit() {
#ifndef B200_CUSIM_BUILD
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void cp_async_wait_all() {
#ifndef B200_CUSIM_BUILD
    asm volatile("cp.async.wait_group 0;" ::: "memory");
#endif
}

// ---- mbarrier + bulk asynchronous copy (global -> shared through the TMA engine) ------------------------------
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
#ifdef B200_CUSIM_BUILD
    *bar = 0; (void)count;
#else
    const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
#endif
}
__device__ __forceinline__ void mbar_init_fence() {
#ifndef B200_CUSIM_BUILD
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
#ifdef B200_CUSIM_BUILD
    (void)bar; (void)bytes;
#else
    const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(a), "r"(bytes) : "memory");
#endif
}
// dst, src 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
#ifdef B200_CUSIM_BUILD
    memcpy(smem_dst, gmem_src, bytes); (void)bar;
#else
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(d), "l"(gmem_src), "r"(bytes), "r"(b) : "memory");
#endif
}
// The spectrum cache is written once by the analysis kernel and read once by the synthesis kernel, ~30 GB each way per
// config-2 step.  Its stores stream (st.global.cs) and its bulk loads carry an L2 evict-first policy, so that it does not
// push the lines that ARE re-read out of L2 -- the sample windows of successive frame pairs overlap by 60 %, and each
// frame's decision words are read three times by the smoothing recurrence.  Measured on config 2: k1 16.3 -> 15.6 ms,
// k2 15.9 -> 15.6 ms, same outputs.
// bulk_g2s with an L2 evict-first policy: for data read exactly once (the cached spectra)
__device__ __forceinline__ void bulk_g2s_once(void* smem_dst, const void* gmem_src, unsigned bytes, unsigned long long* bar) {
#ifdef B200_CUSIM_BUILD
    bulk_g2s(smem_dst, gmem_src, bytes, bar);
#else
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    const unsigned b = (unsigned)__cvta_generic_to_shared(bar);
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(d), "l"(gmem_src), "r"(bytes), "r"(b), "l"(pol) : "memory");
#endif
}
// streaming (evict-first) global store of data no kernel re-reads soon (the spectrum cache)
template <typename V>
__device__ __forceinline__ void st_stream(V* p, V v) {
#ifdef B200_CUSIM_BUILD
    *p = v;
#else
    __stcs(p, v);
#endif
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
#ifdef B200_CUSIM_BUILD
    (void)bar; (void)parity;
    __syncwarp();                  // simulator: the issuing lane's (synchronous) copy precedes its own wait
#else
    const unsigned a = (unsigned)__cvta_generic_to_shared(bar);
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra D_%=;\n\t"
        "bra W_%=;\n\t"
        "D_%=:\n\t}"
        ::"r"(a), "r"(parity) : "memory");
#endif
}
// order this thread's earlier generic-proxy accesses of shared memory before later async-proxy (bulk copy) writes
__device__ __forceinline__ void fence_proxy_async_smem() {
#ifndef B200_CUSIM_BUILD
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
// shared -> global bulk copy (TMA store engine) of `bytes` (16-byte multiple, both sides 16-byte aligned); completion is
// tracked by bulk groups: commit, then wait_group.read before the shared source is overwritten
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, unsigned bytes) {
#ifdef B200_CUSIM_BUILD
    memcpy(gmem_dst, smem_src, bytes);
#else
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem_src);
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(s), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void bulk_wait_read_all() {
#ifndef B200_CUSIM_BUILD
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
#endif
}

#ifdef B200_CUSIM_BUILD
#define B200_NOINLINE __attribute__((noinline))
#else
#define B200_NOINLINE __noinline__
#endif

// Exact (float64) re-decision of one bin of one frame: direct DFT of the windowed samples.
// Warp-cooperative; every lane returns the same value.  2 = above threshold, 1 = not above,
// 0 = unresolved even in float64 (|P - T^2| <= 1e-12 T^2).  The tables come as pointers, not as `const Tables&`: a
// reference into the kernel's parameters would make the caller copy them all to local memory.
template <typename T>
__device__ B200_NOINLINE int recheck_bin_fp64(const T* __restrict__ xrow, long long base, long long i1,
                                              long long Lp, long long n_total, int k, const double* __restrict__ wa64,
                                              const double2* __restrict__ cs64, const double* __restrict__ thr2_64,
                                              int lane) {
    double sr = 0.0, si = 0.0;
    for (int n = lane; n < kN; n += 32) {
        const double x = chunk_sample_f64(xrow, base + n, i1, Lp, n_total) * wa64[n];   // the caller's exact samples
        const double2 cs = cs64[(k * n) & (kN - 1)];
        sr = fma(x, cs.x, sr);
        si = fma(-x, cs.y, si);
    }
    sr = warp_sum(sr);
    si = warp_sum(si);
    const double P = sr * sr + si * si;
    const double T2 = thr2_64[k];
    if (fabs(P - T2) <= 1e-12 * T2) return 0;
    return P > T2 ? 2 : 1;
}

// =============================================================================================
// k1: analysis.  bits[(ul*T + t)*FW + w] bit b  <=>  raw |X[32w+b, t]| above the bin threshold.
// =============================================================================================
struct K1Args {
    Geom g;
    Tables tb;
    const void* x;             // [C][in_stride] samples in the caller's dtype (kernel template T)
    unsigned* bits;            // [n_units][T][FW]
    unsigned* rowmax;          // [n_units][FPad]  max_t 4|X|^2 as float bits (>= 0 so uint order works); written only by
                               // the row-maximum instantiation k1_analyze<.., true>
    Counters* cnt;
    DebugTap dbg;
    int run;                   // frames per work item (even)
    int n_runs;                // ceil(T / run)
    float2* zcache;            // optional [n_units][ceil(T/2)][32 slots][32 lanes]: the packed spectrum of every
                               // frame pair, kept so that k2 need not transform the frames a second time
    int zpairs;                // ceil(T/2)
    int z_lo, z_hi;            // only frames [z_lo, z_hi) are read back by k2 (chunk centre + halo): the rest is not stored
    const unsigned* guard;     // optional device flag: when given and zero the kernel returns at once (it is then the
                               // row-maximum fallback behind k1_analyze<.., false> or k1d_analyze, gate_dual.cuh)
    unsigned* need_rowmax;     // k1_analyze<.., false>: device flag raised when a frame could reach its top_db floor
    float min_floor4;          // min over bins of 4 * (10^((thresh + top_db)/20) - eps)^2 (PERREC: per recording, in
                               // slot FPad - 1 of its floor4 row)
    const UnitDesc* units;     // ROWS instantiations: the call's unit table
};

// One pair's sample window (32 + 8 rows of 32 samples) as the 16-byte-aligned span that covers it: up to 16 bytes more.
constexpr int kK1WinBytes = 32 * (32 + 8) * 4 + 16;
constexpr int k1_smem_floats() {
    return kN + 2 * kN + 2 * kFPad + kWarps * kExchFloats + kWarps * 2 * kFW + 8 + kWarps * (kK1WinBytes / 4) + 2 * kWarps;
}

// ROWMAX = false (default): the window of the warp's next frame pair streams into a per-warp shared buffer by one bulk
// copy (TMA engine) while the current pair is transformed, and the top_db row maxima are not tracked: the kernel only
// raises need_rowmax when a pair's energy could reach the lowest floor (|X_k|^2 <= N ||frame||^2), and the host then runs
// the ROWMAX = true instantiation behind it (guarded by that flag) for the maxima.  That instantiation loads the samples
// directly and tracks the maxima of every bin; run alone it is the whole analysis.
// PERREC (with ROWS; b200gate_set_noise_threshold_rows): every unit compares against its recording's row of the
// threshold tables (UnitDesc::rec), read through the read-only data path instead of the block's shared copy -- a
// block's warps work on units of different recordings, and four per-warp copies would not fit next to the FFT tiles.
template <int HR, typename T, bool ROWMAX = false, bool ROWS = false, bool PERREC = false>
__global__ void __launch_bounds__(kThreads, B200_K1_MINBLOCKS) k1_analyze(const K1Args a) {
    static_assert(32 * (32 + HR) * 4 + 16 <= kK1WinBytes, "sample window must fit the buffer");
    static_assert(ROWS || !PERREC, "per-recording thresholds need the unit table");
    constexpr bool kBulk = !ROWMAX && sizeof(T) <= 4;   // float32 / int16 windows (float64: direct loads)
    if (a.guard && *a.guard == 0u) return;
    B200_DYN_SMEM(float, smem);
    float* s_wa = smem;
    float2* s_tw = reinterpret_cast<float2*>(smem + kN);
    float* s_thr4 = smem + 3 * kN;
    float* s_gco = s_thr4 + kFPad;
    float* s_tiles = s_gco + kFPad;
    unsigned* s_amb_all = reinterpret_cast<unsigned*>(s_tiles + kWarps * kExchFloats);
    unsigned char* s_win_all = reinterpret_cast<unsigned char*>(s_amb_all + kWarps * 2 * kFW + 8);   // 16-byte aligned
    unsigned long long* s_bar_all = reinterpret_cast<unsigned long long*>(s_win_all + kWarps * kK1WinBytes);
    for (int i = threadIdx.x; i < kN; i += kThreads) {
        s_wa[i] = a.tb.wa[i];
        s_tw[i] = a.tb.tw[i];
    }
    if (!PERREC) {
        for (int i = threadIdx.x; i < kFPad; i += kThreads) {
            s_thr4[i] = a.tb.thr4[i];
            s_gco[i] = a.tb.gco[i];
        }
    }
    const Geom& g = a.g;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* win = s_win_all + warp * kK1WinBytes;
    unsigned long long* bar = s_bar_all + warp;
    if (kBulk) {
        if (lane == 0) mbar_init(bar, 1);
        mbar_init_fence();
    }
    __syncthreads();
    unsigned phase = 0;

    float* tile = s_tiles + warp * kExchFloats;
    unsigned* s_amb = s_amb_all + warp * 2 * kFW;
    const int H = g.H;
    const int pl = (32 - lane) & 31;                 // partner lane holding the mirrored bins
    const long long n_items = (long long)g.n_units * a.n_runs;
    const long long item_stride = (long long)gridDim.x * kWarps;
    // work item = (local unit, run); the warp's items advance by item_stride = (step_ul, step_run) without dividing
    const int step_ul = (int)(item_stride / a.n_runs), step_run = (int)(item_stride - (long long)step_ul * a.n_runs);
    auto next_item = [&](int& ul_, int& run_) {
        ul_ += step_ul;
        run_ += step_run;
        if (run_ >= a.n_runs) { run_ -= a.n_runs; ++ul_; }
    };
    // sample row and chunk origin (global index of chunk sample 0) of a local unit; ROWS: also its span, row length and frames
    auto unit_row = [&](int ul_, const T*& xrow, long long& i1) {
        const int u = g.u0 + ul_;
        if (ROWS) {
            xrow = static_cast<const T*>(a.units[u].x);
            i1 = a.units[u].i1;
            return;
        }
        const int ic = u / g.C, c = u - ic * g.C;
        i1 = (long long)ic * g.step - g.pad;
        xrow = static_cast<const T*>(a.x) + (long long)c * g.in_stride;
    };
    auto unit_Lp = [&](int ul_) -> long long { return ROWS ? a.units[g.u0 + ul_].Lp : g.Lp; };
    auto unit_n = [&](int ul_) -> long long { return ROWS ? a.units[g.u0 + ul_].n_total : g.n_total; };
    // Request the window of pair (tt, tt + 1) of a unit into this warp's buffer when it lies inside the chunk and the
    // recording and the 16-byte-aligned span covering it lies inside the samples the chunk reads,
    // [max(0, i1), min(n_total, i1 + Lp)).  (Bounding it by the row instead let the aligned span reach past the rows a
    // caller staged or streamed -- [w_lo, w_hi) of b200gate_run -- by up to 15 bytes at either end.)  Returns the
    // window's element offset in the buffer, or -1: the pair is then loaded directly.  Warp-uniform; every lane has
    // finished reading the buffer.
    auto request = [&](const T* xr_, long long i1_, long long Lp_, long long n_, int tt) -> int {
        if (!kBulk) return -1;
        const long long bb = (long long)tt * H - kN / 2;
        if (!pair_window_interior<HR>(bb, i1_, Lp_, n_)) return -1;
        const unsigned long long src = reinterpret_cast<unsigned long long>(xr_ + i1_ + bb);
        const unsigned long long lo = src & ~15ull;
        const unsigned long long hi = (src + 32 * (32 + HR) * sizeof(T) + 15) & ~15ull;
        const long long r_lo = i1_ > 0 ? i1_ : 0, r_hi = i1_ + Lp_ < n_ ? i1_ + Lp_ : n_;
        if (lo < reinterpret_cast<unsigned long long>(xr_ + r_lo) || hi > reinterpret_cast<unsigned long long>(xr_ + r_hi))
            return -1;
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
            mbar_expect_tx(bar, (unsigned)(hi - lo));
            bulk_g2s(win, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), bar);
        }
        return (int)((src - lo) / sizeof(T));
    };
    long long item = (long long)blockIdx.x * kWarps + warp;
    int ul = (int)(item / a.n_runs), run = (int)(item - (long long)ul * a.n_runs);
    int woff = -1;                                   // element offset of the pending window in `win`, -1: none
    if (kBulk && item < n_items) {
        const T* xr_;
        long long i1_;
        unit_row(ul, xr_, i1_);
        woff = request(xr_, i1_, unit_Lp(ul), unit_n(ul), run * a.run);
    }

    for (; item < n_items; item += item_stride, next_item(ul, run)) {
        const T* xrow;
        long long i1;
        unit_row(ul, xrow, i1);
        const long long Lp_u = unit_Lp(ul), n_u = unit_n(ul);
        const int rec = PERREC ? a.units[g.u0 + ul].rec : 0;          // (PERREC) the unit's row of the threshold tables
        const int t0 = run * a.run;
        const int t1 = min(t0 + a.run, ROWS ? a.units[g.u0 + ul].T : g.T);
        float mx[ROWMAX ? kFW : 1];
        if (ROWMAX) {
#pragma unroll
            for (int q = 0; q < kFW; ++q) mx[q] = 0.f;
        }
        float emax = 0.f;                            // largest pair energy of the item (row floor test)

        for (int t = t0; t < t1; t += 2) {
            const bool vb = (t + 1 < t1);
            const long long base = (long long)t * H - kN / 2;
            float xr[32 + HR];
            if (kBulk && woff >= 0) {                        // warp-uniform
                mbar_wait(bar, phase);
                phase ^= 1u;
                const T* wp = reinterpret_cast<const T*>(win) + woff + lane;
#pragma unroll
                for (int r = 0; r < 32 + HR; ++r) xr[r] = (float)wp[32 * r];
            } else {
                load_pair_rows<HR>(xr, xrow, base, i1, Lp_u, n_u, lane);
            }
            if (kBulk) {                                     // the next window streams in behind this pair's transform
                if (t + 2 < t1) {
                    woff = request(xrow, i1, Lp_u, n_u, t + 2);
                } else if (item + item_stride < n_items) {   // the first window of the warp's next work item
                    int uln = ul, runn = run;
                    next_item(uln, runn);
                    const T* xr_;
                    long long i1_;
                    unit_row(uln, xr_, i1_);
                    woff = request(xr_, i1_, unit_Lp(uln), unit_n(uln), runn * a.run);
                } else {
                    woff = -1;
                }
            }
            float re[32], im[32];
            const float E = warp_sum(pack_frame_pair<HR>(re, im, xr, s_wa, lane, vb));
            if (!ROWMAX) emax = fmaxf(emax, E);
            const float S = sqrtf(E);
            warp_fft1024(re, im, tile, s_tw, lane);
            if (a.zcache && t >= a.z_lo && t < a.z_hi) {      // warp-uniform
                float2* zp = a.zcache + ((long long)ul * a.zpairs + (t >> 1)) * 1024 + lane;
#pragma unroll
                for (int q = 0; q < 32; ++q) st_stream(zp + 32 * q, make_float2(re[brev5(q)], im[brev5(q)]));
            }

            unsigned wordA = 0u, wordB = 0u;
            unsigned anyamb = 0u;
#pragma unroll
            for (int q = 0; q < kFW; ++q) {
                const int sA = brev5(q), sP = brev5(31 - q), s0 = brev5((32 - q) & 31);
                const float zr = re[sA], zi = im[sA];
                float pr = __shfl_sync(0xffffffffu, re[sP], pl);
                float pi = __shfl_sync(0xffffffffu, im[sP], pl);
                if (lane == 0) { pr = re[s0]; pi = im[s0]; }
                // 2 X_a = Z + conj(Zp),  2 X_b = (Z - conj(Zp)) / i
                const float ar = zr + pr, ai = zi - pi;
                const float br = zi + pi, bi = pr - zr;
                const float PA = fmaf(ar, ar, ai * ai);
                const float PB = fmaf(br, br, bi * bi);
                const int k = lane + 32 * q;
                const bool valid = (q < 16) || (lane == 0);
                const float th = PERREC ? __ldg(a.tb.thr4 + rec * kFPad + k) : s_thr4[k];
                const float gg = fmaf(PERREC ? __ldg(a.tb.gco + rec * kFPad + k) : s_gco[k], S, th * 8.0e-7f);
                const float dA = PA - th, dB = PB - th;
                const unsigned wA = __ballot_sync(0xffffffffu, valid && (dA > 0.f));
                const unsigned wB = __ballot_sync(0xffffffffu, valid && vb && (dB > 0.f));
                const bool amA = valid && fabsf(dA) <= gg, amB = valid && vb && fabsf(dB) <= gg;
                if (lane == q) { wordA = wA; wordB = wB; }
                if (__any_sync(0xffffffffu, amA || amB)) {   // rare: remember the bins inside the guard band
                    const unsigned mA = __ballot_sync(0xffffffffu, amA);
                    const unsigned mB = __ballot_sync(0xffffffffu, amB);
                    anyamb |= 1u << q;
                    if (lane == 0) { s_amb[2 * q] = mA; s_amb[2 * q + 1] = mB; }
                }
                if (ROWMAX && valid) mx[q] = fmaxf(mx[q], vb ? fmaxf(PA, PB) : PA);
            }
            if (a.dbg.ul == ul) {                            // parity tap (tests): the FP32 STFT itself
#pragma unroll 1
                for (int q = 0; q < kFW; ++q) {
                    float zr = 0.f, zi = 0.f, pr = 0.f, pi = 0.f;
#pragma unroll
                    for (int qq = 0; qq < kFW; ++qq)
                        if (qq == q) {
                            zr = re[brev5(qq)]; zi = im[brev5(qq)];
                            pr = __shfl_sync(0xffffffffu, re[brev5(31 - qq)], pl);
                            pi = __shfl_sync(0xffffffffu, im[brev5(31 - qq)], pl);
                            if (lane == 0) { pr = re[brev5((32 - qq) & 31)]; pi = im[brev5((32 - qq) & 31)]; }
                        }
                    const int k = lane + 32 * q;
                    if (((q < 16) || lane == 0) && k < kF) {
                        float* sp = a.dbg.spec + ((long long)t * kF + k) * 2;
                        sp[0] = 0.5f * (zr + pr); sp[1] = 0.5f * (zi - pi);
                        if (vb) { sp[2 * kF] = 0.5f * (zi + pi); sp[2 * kF + 1] = 0.5f * (pr - zr); }
                    }
                }
            }
            if (anyamb) {                             // warp-uniform, rare: redo those bins in float64
                __syncwarp();
                unsigned nre = 0, nun = 0;
                for (int q = 0; q < kFW; ++q) {
                    if (!((anyamb >> q) & 1u)) continue;
                    for (int fr = 0; fr < 2; ++fr) {
                        unsigned m = s_amb[2 * q + fr];
                        while (m) {
                            const int src = __ffs((int)m) - 1;
                            m &= m - 1;
                            const int r = recheck_bin_fp64(xrow, base + (long long)fr * H, i1, Lp_u, n_u,
                                                           src + 32 * q, a.tb.wa64, a.tb.cs64,
                                                           PERREC ? a.tb.thr2_64 + rec * kF : a.tb.thr2_64, lane);
                            ++nre;
                            if (r == 0) { ++nun; continue; }
                            if (lane == q) {
                                unsigned& wd = fr ? wordB : wordA;
                                wd = (r == 2) ? (wd | (1u << src)) : (wd & ~(1u << src));
                            }
                        }
                    }
                }
                __syncwarp();
                if (lane == 0 && !a.guard) {          // (a guarded fallback re-derives bins the kernel before it counted)
                    atomicAdd(&a.cnt->rechecked, (unsigned long long)nre);
                    if (nun) atomicAdd(&a.cnt->unresolved, (unsigned long long)nun);
                }
            }
            if (lane < kFW) {
                unsigned* dst = a.bits + ((long long)ul * g.T + t) * kFW + lane;
                dst[0] = wordA;
                if (vb) dst[kFW] = wordB;
            }
        }
        if (ROWMAX) {
#pragma unroll
            for (int q = 0; q < kFW; ++q)
                if ((q < 16) || (lane == 0))
                    atomicMax(a.rowmax + (long long)ul * kFPad + lane + 32 * q, __float_as_uint(mx[q]));
        } else if (4.0f * (float)kN * emax >=
                       0.999f * (PERREC ? __ldg(a.tb.floor4 + rec * kFPad + kFPad - 1) : a.min_floor4) && lane == 0) {
            atomicOr(a.need_rowmax, 1u);             // |X|^2 <= N * (frame energy): a bin could reach its top_db floor
        }
    }
}

// =============================================================================================
// top_db floor (spectralgate/utils.py:16): clamped dB > thresh  <=>  raw > thresh  OR
// (row max over the chunk's frames - top_db > thresh).  One thread per (unit, mask word).
// =============================================================================================
__device__ __forceinline__ void rowfloor_word(int i, int ul, int w, const unsigned* __restrict__ rowmax,
                                              const float* __restrict__ floor4, unsigned* __restrict__ rowflag,
                                              Counters* cnt) {
    unsigned word = 0u, nflag = 0u, namb = 0u;
    for (int b = 0; b < 32; ++b) {
        const int f = w * 32 + b;
        if (f >= kF) break;
        const float v = __uint_as_float(rowmax[(long long)ul * kFPad + f]);
        const float tf = floor4[f];
        if (v > tf) { word |= 1u << b; ++nflag; }
        if (fabsf(v - tf) <= tf * 1.0e-5f) ++namb;
    }
    rowflag[i] = word;
    if (nflag) atomicAdd(&cnt->floor_flags, (unsigned long long)nflag);
    if (namb) atomicAdd(&cnt->floor_ambiguous, (unsigned long long)namb);
}
__global__ void k_rowfloor(int n_units, const unsigned* __restrict__ rowmax, const float* __restrict__ floor4,
                           unsigned* __restrict__ rowflag, Counters* cnt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_units * kFW) return;
    const int ul = i / kFW, w = i - ul * kFW;
    rowfloor_word(i, ul, w, rowmax, floor4, rowflag, cnt);
}
// per-recording thresholds: unit ul (units = the batch's first entry of the unit table) reads its recording's floor4 row
__global__ void k_rowfloor_rec(int n_units, const UnitDesc* __restrict__ units, const unsigned* __restrict__ rowmax,
                               const float* __restrict__ floor4, unsigned* __restrict__ rowflag, Counters* cnt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_units * kFW) return;
    const int ul = i / kFW, w = i - ul * kFW;
    rowfloor_word(i, ul, w, rowmax, floor4 + (long long)units[ul].rec * kFPad, rowflag, cnt);
}

// =============================================================================================
// Mask smoothing in integers.  K = tri_f (x) tri_t / ((nf+1)^2 (nt+1)^2) with tri_n[k] = n+1-|k|
// (base.py:14-28), so  smoothed = p * num / D + (1-p) * edge,  num = sum tri_f tri_t bit.
// Output: num as uint16 [n_units][T][FPad] for frames [tf_lo, tf_hi).
// Time direction: per-bin streaming second-difference recurrence (tri = box * box);
// frequency direction: direct taps from the shared-memory tile.
// =============================================================================================
struct SmoothArgs {
    int n_units, T;
    int nf, nt;
    int tf_lo, tf_hi;          // frames that need masks
    int TT;                    // output frames per tile
    const unsigned* bits;      // [n_units][T][FW]
    const unsigned* rowflag;   // [n_units][FW]
    unsigned short* num;       // [n_units][ceil(T/2)][FPad][2]  (num_index)
    const UnitDesc* units;     // ROWS instantiations: units + (first unit of the batch); T is then the pitch only and
                               // tf_hi the largest of the batch
};

__host__ __device__ inline int smooth_rows(int TT, int nt) { return TT + 2 * nt + 2 * (nt + 1); }
__host__ __device__ inline int smooth_cpitch(int nf) { return (kFPad + 2 * nf + 2) | 1; }   // odd #shorts/2 not needed; keep simple
inline size_t smooth_smem_bytes(int TT, int nf, int nt) {
    return (size_t)smooth_rows(TT, nt) * kFW * 4 + (size_t)TT * smooth_cpitch(nf) * 2 + 16;
}

template <bool ROWS = false>
__global__ void __launch_bounds__(256) k_smooth_generic(const SmoothArgs a) {
    B200_DYN_SMEM(unsigned, smem);
    const int nt = a.nt, nf = a.nf, aa = nt + 1;
    const int rows = smooth_rows(a.TT, nt);
    const int cp = smooth_cpitch(nf);
    unsigned* s_bits = smem;                                                   // [rows][FW]
    unsigned short* s_c = reinterpret_cast<unsigned short*>(smem + rows * kFW);  // [TT][cp]
    const int ul = blockIdx.y;
    const int T = ROWS ? a.units[ul].T : a.T, tf_hi = ROWS ? a.units[ul].tf_hi : a.tf_hi;
    const int t0 = a.tf_lo + blockIdx.x * a.TT;
    if (t0 >= tf_hi) return;
    const int tt_n = min(a.TT, tf_hi - t0);
    // row rho <-> frame tau = t0 - nt - 2aa + rho ; the first 2aa rows are "before the stream" = 0
    const int tau0 = t0 - nt - 2 * aa;
    for (int i = threadIdx.x; i < rows * kFW; i += blockDim.x) {
        const int rho = i / kFW, w = i - rho * kFW;
        const int tau = tau0 + rho;
        unsigned v = 0u;
        if (rho >= 2 * aa && tau >= 0 && tau < T)
            v = a.bits[((long long)ul * a.T + tau) * kFW + w] | a.rowflag[ul * kFW + w];
        s_bits[i] = v;
    }
    for (int i = threadIdx.x; i < a.TT * cp; i += blockDim.x) s_c[i] = 0;
    __syncthreads();
    // time direction: c[f, t] = sum_b tri_t[b] m[f, t-b];  s2[tau] = c[., tau - nt]
    for (int f = threadIdx.x; f < kF; f += blockDim.x) {
        const int w = f >> 5, sh = f & 31;
        int d1 = 0, s2 = 0;
        const int steps = tt_n + 2 * nt;
        for (int s = 0; s < steps; ++s) {
            const int rho = 2 * aa + s;
            const int e = (int)((s_bits[rho * kFW + w] >> sh) & 1u)
                        - 2 * (int)((s_bits[(rho - aa) * kFW + w] >> sh) & 1u)
                        + (int)((s_bits[(rho - 2 * aa) * kFW + w] >> sh) & 1u);
            d1 += e;
            s2 += d1;
            const int tt = s - 2 * nt;
            if (tt >= 0) s_c[tt * cp + nf + f] = (unsigned short)s2;
        }
    }
    __syncthreads();
    // frequency direction
    for (int i = threadIdx.x; i < tt_n * kFPad; i += blockDim.x) {
        const int tt = i / kFPad, f = i - tt * kFPad;
        int acc = 0;
        if (f < kF) {
            const unsigned short* cr = s_c + tt * cp + f;      // cr[nf + d] = c[f + d]
            for (int d = -nf; d <= nf; ++d) acc += (nf + 1 - (d < 0 ? -d : d)) * (int)cr[nf + d];
        }
        a.num[(long long)ul * num_unit_stride(a.T) + num_index(t0 + tt, f)] = (unsigned short)acc;
    }
}

// ---------------------------------------------------------------------------------------------
// Packed variant (the one that normally runs).  A thread owns 4 consecutive bins as byte lanes of
// one register and streams over time: the time-direction recurrence costs ~4 ops/bin, and the
// frequency-direction triangle is NTW dp4a dot products per output against byte windows of the
// shared row.  Requirements: nt + 1 <= 14 (byte lanes: counts <= 196, biased first difference
// <= 31) and 2 nf + 1 <= 4 NTW; otherwise the host falls back to k_smooth_generic.
// CTA = 544 threads = 4 units x 136 bin-groups; one __syncthreads per frame.
// ---------------------------------------------------------------------------------------------
struct SmoothPArgs {
    int n_units, T;
    int nf, nt;
    int tf_lo, tf_hi;
    int strip;                 // output frames per CTA
    const unsigned* bits;
    const unsigned* rowflag;
    unsigned short* num;
    unsigned taps[9];          // triangle taps nf+1-|d|, d = -nf..nf, as packed bytes (zero padded)
};
constexpr int kSmoothGroups = kFPad / 4;          // 136 threads per unit
constexpr int kSmoothUnits = 4;
constexpr int kSmoothThreads = kSmoothGroups * kSmoothUnits;   // 544
constexpr int kSmoothBatch = 4;                    // frames per barrier
template <int NTW> __host__ __device__ constexpr int smoothp_rowbytes() { return kFPad + 4 * (NTW + 2) + 64; }
template <int NTW> __host__ __device__ constexpr int smoothp_smem_bytes() {
    return 2 * kSmoothBatch * kSmoothUnits * smoothp_rowbytes<NTW>();
}

__device__ __forceinline__ unsigned dp4a_u(unsigned a, unsigned b, unsigned c) {
#ifdef B200_CUSIM_BUILD
    for (int i = 0; i < 4; ++i) c += ((a >> (8 * i)) & 0xFFu) * ((b >> (8 * i)) & 0xFFu);
    return c;
#else
    return __dp4a(a, b, c);
#endif
}

template <int NTW>
__global__ void __launch_bounds__(kSmoothThreads, 3) k_smooth_packed(const SmoothPArgs a) {
    constexpr int RB = smoothp_rowbytes<NTW>();
    constexpr int NB = kSmoothBatch;
    B200_DYN_SMEM(unsigned char, s_raw);                      // [2][NB][4 units][RB]
    const int tid = threadIdx.x;
    const int ug = tid / kSmoothGroups, i = tid - ug * kSmoothGroups;
    const int ul = blockIdx.y * kSmoothUnits + ug;
    const bool active = ul < a.n_units;
    const int t_begin = a.tf_lo + blockIdx.x * a.strip;
    if (t_begin >= a.tf_hi) return;
    const int t_end = min(t_begin + a.strip, a.tf_hi);
    const int nt = a.nt, nf = a.nf, aa = nt + 1;
    for (int k = tid; k < 2 * NB * kSmoothUnits * RB / 4; k += kSmoothThreads) reinterpret_cast<unsigned*>(s_raw)[k] = 0u;
    __syncthreads();

    const int w = i >> 3, sh = (i & 7) * 4;
    const unsigned fl = active ? ((a.rowflag[ul * kFW + w] >> sh) & 0xFu) : 0u;
    const unsigned* bp = a.bits + (long long)(active ? ul : 0) * a.T * kFW + w;
    unsigned short* outp = a.num + (long long)(active ? ul : 0) * num_unit_stride(a.T) + 8 * i;
    unsigned taps[NTW];
#pragma unroll
    for (int m = 0; m < NTW; ++m) taps[m] = a.taps[m];

    const int tau_s = t_begin - nt;                 // first frame fed into the recurrence
    const int tau_e = t_end - 1 + nt;               // last one
    unsigned d1b = 0x10101010u, s2 = 0u;
    int par = 0;
    // warm-up: the first 2 nt frames only feed the recurrence (no output yet)
    auto nib = [&](int t) -> unsigned {
        return (active && t >= tau_s && t >= 0 && t < a.T) ? (((__ldg(bp + (long long)t * kFW) >> sh) & 0xFu) | fl) : 0u;
    };
    auto advance = [&](unsigned na, unsigned nb, unsigned nc) {
        const unsigned ea = (na * 0x00204081u) & 0x01010101u;
        const unsigned eb = (nb * 0x00204081u) & 0x01010101u;
        const unsigned ec = (nc * 0x00204081u) & 0x01010101u;
        d1b = d1b + ea + ec - 2u * eb;
        s2 = s2 + d1b - 0x10101010u;
    };
    int tau = tau_s;
    for (; tau < t_begin + nt; ++tau) advance(nib(tau), nib(tau - aa), nib(tau - 2 * aa));
    // steady state: NB output frames per barrier.  Of the three rows a frame needs, the two old ones (tau - aa,
    // tau - 2 aa) were read by this thread a few iterations ago and hit L1; the NEW row comes from L2 / HBM, and its
    // first use was where the kernel stalled.  The new rows
    // of the NEXT batch are therefore requested one whole batch -- two barriers -- before they are needed.
    auto in_range = [&](int t) -> bool { return active && t >= tau_s && t >= 0 && t < a.T; };
    unsigned pre[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) pre[j] = (tau + j <= tau_e && in_range(tau + j)) ? __ldg(bp + (long long)(tau + j) * kFW) : 0u;
    for (; tau <= tau_e; tau += NB) {
        unsigned na[NB], nb[NB], nc[NB];
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            const int tj = tau + j;
            const bool live = tj <= tau_e;
            na[j] = (live && in_range(tj)) ? (((pre[j] >> sh) & 0xFu) | fl) : 0u;
            pre[j] = (tj + NB <= tau_e && in_range(tj + NB)) ? __ldg(bp + (long long)(tj + NB) * kFW) : 0u;
            nb[j] = live ? nib(tj - aa) : 0u;
            nc[j] = live ? nib(tj - 2 * aa) : 0u;
        }
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            advance(na[j], nb[j], nc[j]);
            unsigned char* row = s_raw + ((par * NB + j) * kSmoothUnits + ug) * RB;
            row[nf + 4 * i + 0] = (unsigned char)(s2 & 0xFFu);
            row[nf + 4 * i + 1] = (unsigned char)((s2 >> 8) & 0xFFu);
            row[nf + 4 * i + 2] = (unsigned char)((s2 >> 16) & 0xFFu);
            row[nf + 4 * i + 3] = (unsigned char)(s2 >> 24);
        }
        __syncthreads();
        // frequency direction; frames (t, t+1) of a pair leave together as one 16-byte store (num_index layout)
        auto freq_taps = [&](int j, unsigned (&o)[4]) {
            const unsigned char* row = s_raw + ((par * NB + j) * kSmoothUnits + ug) * RB;
            const unsigned* rw = reinterpret_cast<const unsigned*>(row) + i;
            unsigned wv[NTW + 1];
#pragma unroll
            for (int m = 0; m <= NTW; ++m) wv[m] = rw[m];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                unsigned acc = 0u;
#pragma unroll
                for (int m = 0; m < NTW; ++m) {
                    const unsigned win = (jj == 0) ? wv[m] : __funnelshift_r(wv[m], wv[m + 1], 8 * jj);
                    acc = dp4a_u(win, taps[m], acc);
                }
                o[jj] = acc;
            }
        };
#pragma unroll
        for (int j = 0; j < NB; j += 2) {
            const int t_out = tau + j - nt;                   // even: strips start on even frames, NB is even
            if (tau + j > tau_e) break;
            unsigned oa[4], ob[4] = {0u, 0u, 0u, 0u};
            freq_taps(j, oa);
            if (tau + j + 1 <= tau_e) freq_taps(j + 1, ob);
            if (active) {
                uint4 pk;
                pk.x = oa[0] | (ob[0] << 16);
                pk.y = oa[1] | (ob[1] << 16);
                pk.z = oa[2] | (ob[2] << 16);
                pk.w = oa[3] | (ob[3] << 16);
                *reinterpret_cast<uint4*>(outp + (long long)(t_out >> 1) * (2 * kFPad)) = pk;
            }
        }
        par ^= 1;
    }
}

// =============================================================================================
// k2: synthesis.
// =============================================================================================
struct K2Args {
    Geom g;
    Tables tb;
    const void* x;                 // caller dtype (kernel template T)
    void* y;                       // [C][out_stride], caller dtype
    const unsigned short* num;     // [n_units][T][FPad] integer mask numerators (stationary)
    const float* fmask;            // [n_units][T][FPad] final float masks (non-stationary)
    float pD;                      // prop_decrease / D
    float one_minus_p;             // 1 - prop_decrease
    int nt;                        // time half-width (edge factor of the first/last frames)
    int run;                       // output hops per work item
    int n_runs;
    DebugTap dbg;
    const float2* zcache;          // optional: spectra stored by k1 / k1n (frames then are not re-transformed)
    int zpairs;
    // k2c_synthesize kMaskBits*: smoothing inside synthesis (gate_synth.cuh) from the decisions instead of `num`
    const unsigned* bits;          // [n_units][T][FW]
    const unsigned* rowflag;       // [n_units][FW]
    int sm_pad;                    // zero halo bytes before bin 0 of a time-sum row: nf rounded up to a multiple of 16
    int sm_ws;                     // first tap word of bin group i: row word i + sm_ws
    int sm_ntw;                    // tap words (4, 7, 9 or 10)
    unsigned sm_taps[10];          // triangle taps nf+1-|d| as bytes, after (sm_pad - nf) % 4 zero bytes
    // k2_synthesize<.., ADJ = true>: the adjoint of a unit (b200gate_adjoint).  x is the gradient g of the output,
    // read on the unit's centre only and divided by the overlap-add norm; the un-normalised overlap-add of the whole
    // padded span goes to adj[ul][0, Lp) (chunk-local index), which k_adj_gather sums across units.
    float* adj;
    long long adj_pitch;
    const UnitDesc* units;         // k2c_synthesize<.., ROWS = true>: the call's unit table
    StreamWin sw;                  // k2c_synthesize<.., STREAM = true>: zcache / fmask are the stream's rings (zpairs = ring / 2)
    const SessRow* rows;           // k2c_synthesize<.., SESS = true>: row ul's hops [ha, hb), bound T and output offset
};

constexpr int k2_smem_floats(int H) { return 2 * kN + 2 * kN + H + kFPad + kWarps * kExchFloats + 8 + kWarps * 2 * kN; }

// time edge factor of the zero-padded smoothing: sum of the triangle taps that stay inside [0, T)
__device__ __forceinline__ float time_edge(int t, int T, int nt) {
    int s = 0;
    for (int b = -nt; b <= nt; ++b)
        if (t - b >= 0 && t - b < T) s += nt + 1 - (b < 0 ? -b : b);
    return (float)s / (float)((nt + 1) * (nt + 1));
}

// 1 / (sum of w^2 over the frames overlapping chunk-local sample jp): the overlap-add norm k2_synthesize divides by
// (scipy's istft; 1 where the sum is <= 1e-10).  Called for the first and last hops of a unit only: kept out of line so
// the adjoint's interior frames, which read s_invn, carry none of its registers.
#ifdef B200_CUSIM_BUILD
#define B200_NOINLINE
#else
#define B200_NOINLINE __noinline__
#endif
template <int HR>
__device__ B200_NOINLINE float k2_edge_inv_norm(long long jp, int H, int T, const float* s_invn, const float* s_ws,
                                                float ws_to_w) {
    constexpr int NH = 32 / HR;
    const long long q = jp + kN / 2;
    const int hop = (int)(q / H), ro = (int)(q - (long long)hop * H);
    if (hop >= NH - 1 && hop <= T - 1) return s_invn[ro];
    float nrm = 0.f;
    for (int i = 0; i < NH; ++i) {
        const int tf = hop - i;
        if (tf >= 0 && tf <= T - 1) {
            const float w = s_ws[i * H + ro] * ws_to_w;
            nrm = fmaf(w, w, nrm);
        }
    }
    return nrm > 1e-10f ? 1.0f / nrm : 1.0f;
}

// The adjoint's input frame pair (t, t+1): g / norm on the unit's centre [pad, jp_hi), zero elsewhere.  Row r of the
// pair window is row r % HR of hop t + r / HR; when every one of those hops is interior the norm is s_invn's.
template <int HR, typename T>
__device__ __forceinline__ float load_adjoint_pair(float (&re)[32], float (&im)[32], const T* __restrict__ grow, int t,
                                                   long long base, long long i1, long long pad, long long jp_hi, int H,
                                                   int T_, const float* __restrict__ s_invn,
                                                   const float* __restrict__ s_ws, float ws_to_w,
                                                   const float* __restrict__ s_wa, int lane, bool vb) {
    constexpr int NH = 32 / HR;
    const bool interior = t >= NH - 1 && t + (32 + HR - 1) / HR <= T_ - 1;
    float xr[32 + HR];
#pragma unroll
    for (int r = 0; r < 32 + HR; ++r) {
        const long long j = base + lane + 32 * r;
        float v = 0.0f;
        if (j >= pad && j < jp_hi) {
            const float inv = interior ? s_invn[(r % HR) * 32 + lane]
                                       : k2_edge_inv_norm<HR>(j, H, T_, s_invn, s_ws, ws_to_w);
            v = ld_sample(grow + i1 + j) * inv;
        }
        xr[r] = v;
    }
    return pack_frame_pair<HR>(re, im, xr, s_wa, lane, vb);
}

template <int HR, bool FMASK, typename T, bool ADJ = false>
__global__ void __launch_bounds__(kThreads, 3) k2_synthesize(const K2Args a) {
    constexpr int NH = 32 / HR;             // frames overlapping one hop (win / hop)
    B200_DYN_SMEM(float, smem);
    const Geom& g = a.g;
    const int H = g.H;
    float* s_wa = smem;
    float* s_ws = smem + kN;
    float2* s_tw = reinterpret_cast<float2*>(smem + 2 * kN);
    float* s_invn = smem + 4 * kN;
    float* s_ef = s_invn + H;
    float* s_tiles = s_ef + kFPad;
    for (int i = threadIdx.x; i < kN; i += kThreads) {
        s_wa[i] = a.tb.wa[i];
        s_ws[i] = a.tb.ws[i];
        s_tw[i] = a.tb.tw[i];
    }
    for (int i = threadIdx.x; i < H; i += kThreads) s_invn[i] = a.tb.invn[i];
    for (int i = threadIdx.x; i < kFPad; i += kThreads) s_ef[i] = a.tb.ef[i];
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* tile = s_tiles + warp * kExchFloats;
    // per-warp staging buffer of one cached spectrum (8 KB), 16-byte aligned behind the tiles
    float2* zbuf = reinterpret_cast<float2*>(s_tiles + kWarps * kExchFloats + 8) + warp * kN;
    const int pl = (32 - lane) & 31;
    const long long n_items = (long long)g.n_units * a.n_runs;
    const bool blend = (a.one_minus_p != 0.f);

    for (long long item = (long long)blockIdx.x * kWarps + warp; item < n_items;
         item += (long long)gridDim.x * kWarps) {
        const int ul = (int)(item / a.n_runs);
        const int run = (int)(item - (long long)ul * a.n_runs);
        const int u = g.u0 + ul;
        const int ic = u / g.C, c = u - ic * g.C;
        const long long i1 = (long long)ic * g.step - g.pad;
        long long out_len = g.n_total - (long long)ic * g.step;
        if (out_len > g.step) out_len = g.step;
        // valid chunk-local output range [pad, jp_hi), in padded (frame) coordinates + N/2
        long long jp_hi = g.pad + out_len;
        const long long sig_len = (long long)(g.T - 1) * H;          // istft output length
        if (jp_hi > sig_len) jp_hi = sig_len;                        // beyond it the reference leaves zeros
        if (jp_hi <= g.pad) continue;
        const long long jlo = g.pad + kN / 2, jhi = jp_hi + kN / 2;
        const int h_lo = (int)(jlo / H), h_hi = (int)((jhi + H - 1) / H);
        // the adjoint runs the frames [f_lo, f_hi] that touch the centre and writes every hop they overlap
        const int f_lo = ADJ ? max(0, h_lo - (NH - 1)) : 0, f_hi = ADJ ? min(h_hi - 1, g.T - 1) : g.T - 1;
        const int hs = (ADJ ? f_lo : h_lo) + run * a.run;
        const int he = min(hs + a.run, ADJ ? f_hi + NH : h_hi);
        if (hs >= he) continue;
        int t_start = max(f_lo, hs - (NH - 1));
        if (a.zcache) t_start &= ~1;                 // k1 packed frames (2j, 2j+1): walk the same pairs
        const int t_last = min(he - 1, f_hi);
        const T* xrow = static_cast<const T*>(a.x) + (long long)c * g.in_stride;
        T* yrow = static_cast<T*>(a.y) + (long long)c * g.out_stride;
        const unsigned short* mrow = FMASK ? nullptr : a.num + (long long)ul * num_unit_stride(g.T);
        const float* frow = FMASK ? a.fmask + (long long)ul * g.T * kFPad : nullptr;

        float acc[32 + HR];
#pragma unroll
        for (int r = 0; r < 32 + HR; ++r) acc[r] = 0.f;

        auto stage_spectrum = [&](int tt) {            // request pair (tt, tt+1)'s spectrum into zbuf
            const char* src = reinterpret_cast<const char*>(a.zcache + ((long long)ul * a.zpairs + (tt >> 1)) * 1024);
            char* dst = reinterpret_cast<char*>(zbuf);
#pragma unroll
            for (int j = 0; j < 16; ++j) cp_async16(dst + (lane + 32 * j) * 16, src + (lane + 32 * j) * 16);
            cp_async_commit();
        };
        if (a.zcache && t_start <= t_last) stage_spectrum(t_start);

        for (int t = t_start; t < he; t += 2) {
            const bool va = (t <= t_last), vb = (t + 1 <= t_last);
            if (va) {                                   // vb implies va
                const long long base = (long long)t * H - kN / 2;
                float re[32], im[32];
                if (ADJ) load_adjoint_pair<HR>(re, im, xrow, t, base, i1, g.pad, jp_hi, H, g.T, s_invn, s_ws,
                                               a.tb.ws_to_w, s_wa, lane, vb);
                else if (!a.zcache) load_frame_pair<HR>(re, im, xrow, base, i1, g.Lp, g.n_total, s_wa, lane, vb);
                const long long offA = (long long)t * kFPad, offB = (long long)(vb ? t + 1 : t) * kFPad;
                // the masks of this pair are requested now, a whole FFT before the apply step needs them
                float mka[kFW], mkb[FMASK ? kFW : 1];         // uint16 numerators travel packed two per register
#pragma unroll
                for (int q = 0; q < kFW; ++q) {
                    const int k = lane + 32 * q;                         // < FPad, rows are padded
                    if (FMASK) {
                        mka[q] = frow[offA + k];
                        mkb[FMASK ? q : 0] = frow[offB + k];
                    } else {
                        mka[q] = __uint_as_float((unsigned)mrow[num_index(t, k)] | ((unsigned)mrow[num_index(vb ? t + 1 : t, k)] << 16));
                    }
                }
                float eta = 0.f, etb = 0.f;
                if (!FMASK && blend) {
                    eta = a.one_minus_p * time_edge(t, g.T, a.nt);
                    etb = a.one_minus_p * time_edge(t + 1, g.T, a.nt);
                }
                if (a.dbg.ul == ul) {                        // parity tap (tests): the masks this pair applies
#pragma unroll 1
                    for (int k = lane; k < kF; k += 32) {
                        float ma, mb;
                        if (FMASK) {
                            ma = frow[offA + k];
                            mb = frow[offB + k];
                        } else {
                            ma = fmaf((float)mrow[num_index(t, k)], a.pD, eta * s_ef[k]);
                            mb = fmaf((float)mrow[num_index(vb ? t + 1 : t, k)], a.pD, etb * s_ef[k]);
                        }
                        a.dbg.mask[(long long)t * kF + k] = ma;
                        if (vb) a.dbg.mask[(long long)(t + 1) * kF + k] = mb;
                    }
                }
                // phase 0: forward FFT + mask apply; phase 1: inverse FFT.  One copy of the FFT code
                // serves both: the apply step leaves Z' with real/imaginary parts exchanged and in
                // natural slot order, so ifft(Z') = swap(fft(swap(Z'))) is the very same call.
                const bool cached = a.zcache != nullptr;
                if (cached) {                                // the forward transform of this pair was done by k1
                    cp_async_wait_all();
                    __syncwarp();
#pragma unroll
                    for (int q = 0; q < 32; ++q) {
                        const float2 v = zbuf[32 * q + lane];
                        re[brev5(q)] = v.x;
                        im[brev5(q)] = v.y;
                    }
                    __syncwarp();
                    if (t + 2 <= t_last) stage_spectrum(t + 2);   // next pair streams in behind this pair's math
                }
#pragma unroll 1
                for (int ph = 0; ph < 2; ++ph) {
                    if (!(cached && ph == 0)) warp_fft1024(re, im, tile, s_tw, lane);
                    if (ph == 0) {
#pragma unroll
                        for (int q = 0; q < kFW; ++q) {
                            const int sA = brev5(q), sP = brev5(31 - q), s0 = brev5((32 - q) & 31);
                            const int k = lane + 32 * q;
                            float ma, mb;
                            if (FMASK) {
                                ma = mka[q];
                                mb = mkb[FMASK ? q : 0];
                            } else {
                                const unsigned pk = __float_as_uint(mka[q]);
                                ma = fmaf(u16lo_to_float(pk), a.pD, eta * s_ef[k]);
                                mb = fmaf(u16hi_to_float(pk), a.pD, etb * s_ef[k]);
                            }
                            if (!vb) mb = 0.f;
                            const float s = 0.5f * (ma + mb), d = 0.5f * (ma - mb);
                            const float zr = re[sA], zi = im[sA];
                            if (q < 16) {
                                float pr = __shfl_sync(0xffffffffu, re[sP], pl);
                                float pi = __shfl_sync(0xffffffffu, im[sP], pl);
                                if (lane == 0) { pr = re[s0]; pi = im[s0]; }
                                // Z'[k] = s Z[k] + d conj(Z[N-k]);  Z'[N-k] = s Z[N-k] + d conj(Z[k])
                                const float own_r = fmaf(d, pr, s * zr), own_i = fmaf(-d, pi, s * zi);
                                const float oth_r = fmaf(d, zr, s * pr), oth_i = fmaf(-d, zi, s * pi);
                                const float nr = __shfl_sync(0xffffffffu, oth_r, pl);
                                const float ni = __shfl_sync(0xffffffffu, oth_i, pl);
                                re[sA] = own_r;
                                im[sA] = own_i;
                                if (lane != 0) { re[sP] = nr; im[sP] = ni; }
                                else if (q != 0) { re[s0] = oth_r; im[s0] = oth_i; }
                            } else if (lane == 0) {                      // bin N/2 mirrors onto itself
                                re[sA] = fmaf(d, zr, s * zr);
                                im[sA] = fmaf(-d, zi, s * zi);
                            }
                        }
                        // brev slots -> natural slots with re <-> im exchanged, in place (2-cycles of brev5)
#pragma unroll
                        for (int q = 0; q < 32; ++q) {
                            const int b = brev5(q);
                            if (b == q) {
                                const float tr = re[q];
                                re[q] = im[q];
                                im[q] = tr;
                            } else if (q < b) {
                                const float t1 = re[q], t2 = im[q];
                                re[q] = im[b];
                                im[q] = re[b];
                                re[b] = t2;
                                im[b] = t1;
                            }
                        }
                    }
                }
                // now im = N a'[n], re = N b'[n] (n = lane + 32 q) at slot brev5(q)
#pragma unroll
                for (int q = 0; q < 32; ++q) {
                    const float w = s_ws[lane + 32 * q];
                    acc[q] = fmaf(im[brev5(q)], w, acc[q]);
                    acc[q + HR] = fmaf(re[brev5(q)], w, acc[q + HR]);
                }
            }
            // hops t and t+1 are now complete (all frames <= t+1 have been added)
            if (ADJ) {                                       // un-normalised, the whole padded span
                float* arow = a.adj + (long long)ul * a.adj_pitch;
#pragma unroll
                for (int r = 0; r < 2 * HR; ++r) {
                    const int hop = t + r / HR;
                    const long long jp = (long long)t * H - kN / 2 + 32 * r + lane;
                    if (hop >= hs && hop < he && jp >= 0 && jp < g.Lp) arow[jp] = acc[r];
                }
            } else {
                const long long jp0 = (long long)t * H - kN / 2;             // chunk-local index of row 0, lane 0
                if (t >= hs && t + 1 < he && t >= NH - 1 && t + 1 <= g.T - 1 && jp0 >= g.pad &&
                    jp0 + 2 * H <= jp_hi) {
                    // both hops interior and fully inside the chunk centre: 2*HR coalesced row stores
                    T* dst = yrow + i1 + jp0 + lane;
#pragma unroll
                    for (int r = 0; r < 2 * HR; ++r) dst[32 * r] = st_cast<T>(acc[r] * s_invn[(r % HR) * 32 + lane]);
                } else {
#pragma unroll 1
                    for (int r = 0; r < 2 * HR; ++r) {
                        float v = 0.f;
#pragma unroll
                        for (int rr = 0; rr < 2 * HR; ++rr)
                            if (rr == r) v = acc[rr];
                        const int hop = t + r / HR;
                        if (hop < hs || hop >= he) continue;
                        const int ro = (r % HR) * 32 + lane;
                        const long long jp = (long long)hop * H + ro - kN / 2;   // chunk-local output index
                        if (jp < g.pad || jp >= jp_hi) continue;
                        float inv;
                        if (hop >= NH - 1 && hop <= g.T - 1) {
                            inv = s_invn[ro];
                        } else {                                                  // first / last hops
                            float nrm = 0.f;
                            for (int i = 0; i < NH; ++i) {
                                const int tf = hop - i;
                                if (tf >= 0 && tf <= g.T - 1) {
                                    const float w = s_ws[i * H + ro] * a.tb.ws_to_w;
                                    nrm = fmaf(w, w, nrm);
                                }
                            }
                            inv = nrm > 1e-10f ? 1.0f / nrm : 1.0f;
                        }
                        yrow[i1 + jp] = st_cast<T>(v * inv);
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < 32 - HR; ++r) acc[r] = acc[r + 2 * HR];
#pragma unroll
            for (int r = 32 - HR; r < 32 + HR; ++r) acc[r] = 0.f;
        }
    }
}


// =============================================================================================
// Non-stationary gate (nonstationary.py:47-97).
//   k1n_magnitude  frames -> FFT -> |X|                         [n_units][T][FPad] float32
//   k_iir_sigmoid  filtfilt([b],[1,b-1]) along time per bin (forward sweep started at x[0], backward
//                  sweep over the forward output started at its last value -- nonstationary.py:106-115),
//                  then sigmoid(((|X| - S)/S - n_mult) * slope)  (spectralgate/utils.py:4-8)
//   k_smooth_f     separable triangular smoothing (zero padded), then  m * p + (1 - p)
// =============================================================================================
struct K1nArgs {
    Geom g;
    Tables tb;
    const void* x;
    float* mag;                // [n_units][T][FPad]
    DebugTap dbg;
    int run, n_runs;
    float2* zcache;            // optional, as in K1Args
    int zpairs;
    int z_lo, z_hi;
    const UnitDesc* units;     // ROWS instantiations: the call's unit table
    StreamWin sw;              // STREAM instantiations: frames [sw.f0, g.T) into the rings
    const SessRow* rows;       // SESS instantiations: row ul's window and frames [a0, a1); x is the window, g.in_stride its pitch
};

constexpr int k1n_smem_floats() { return kN + 2 * kN + kWarps * kExchFloats; }

template <int HR, typename T, bool ROWS = false, bool STREAM = false, bool SESS = false>
__global__ void __launch_bounds__(kThreads, 3) k1n_magnitude(const K1nArgs a) {
    B200_DYN_SMEM(float, smem);
    float* s_wa = smem;
    float2* s_tw = reinterpret_cast<float2*>(smem + kN);
    float* s_tiles = smem + 3 * kN;
    for (int i = threadIdx.x; i < kN; i += kThreads) {
        s_wa[i] = a.tb.wa[i];
        s_tw[i] = a.tb.tw[i];
    }
    __syncthreads();
    const Geom& g = a.g;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* tile = s_tiles + warp * kExchFloats;
    const int H = g.H;
    const int pl = (32 - lane) & 31;
    const long long n_items = (long long)g.n_units * a.n_runs;
    for (long long item = (long long)blockIdx.x * kWarps + warp; item < n_items;
         item += (long long)gridDim.x * kWarps) {
        const int ul = (int)(item / a.n_runs);
        const int run = (int)(item - (long long)ul * a.n_runs);
        const int u = g.u0 + ul;
        const int ic = u / g.C, c = u - ic * g.C;
        const UnitDesc* d = ROWS ? a.units + u : nullptr;        // ROWS: the unit's own row, span and frames
        const SessRow* sr = SESS ? a.rows + ul : nullptr;        // SESS: the row's own window and frames
        const long long i1 = ROWS ? d->i1 : (long long)ic * g.step - g.pad;
        const T* xrow = ROWS ? static_cast<const T*>(d->x)
                             : static_cast<const T*>(a.x) + (long long)c * g.in_stride - (SESS ? sr->lo : 0);
        const long long Lp_u = ROWS ? d->Lp : SESS ? sr->R : g.Lp, n_u = ROWS ? d->n_total : SESS ? sr->R : g.n_total;
        const int T_u = ROWS ? d->T : SESS ? sr->a1 : g.T;
        const int t0 = (SESS ? sr->a0 : STREAM ? a.sw.f0 : 0) + run * a.run;
        const int t1 = min(t0 + a.run, T_u);
        for (int t = t0; t < t1; t += 2) {
            const bool vb = (t + 1 < t1);
            const long long base = (long long)t * H - kN / 2;
            float re[32], im[32];
            load_frame_pair<HR>(re, im, xrow, base, i1, Lp_u, n_u, s_wa, lane, vb);
            warp_fft1024(re, im, tile, s_tw, lane);
            if (a.zcache && t >= a.z_lo && t < a.z_hi) {
                const long long zrow = STREAM ? (long long)ul * (a.sw.ring >> 1) + ((t >> 1) & ((a.sw.ring >> 1) - 1))
                                              : (long long)ul * a.zpairs + (t >> 1);
                float2* zp = a.zcache + zrow * 1024 + lane;
#pragma unroll
                for (int q = 0; q < 32; ++q) zp[32 * q] = make_float2(re[brev5(q)], im[brev5(q)]);
            }
            if (!a.mag && a.dbg.ul != ul) continue;        // spectra only
            float* dstA = a.mag + (STREAM ? (long long)ul * a.sw.ring + (t & (a.sw.ring - 1)) : (long long)ul * g.T + t) * kFPad;
#pragma unroll
            for (int q = 0; q < kFW; ++q) {
                const int sA = brev5(q), sP = brev5(31 - q), s0 = brev5((32 - q) & 31);
                const float zr = re[sA], zi = im[sA];
                float pr = __shfl_sync(0xffffffffu, re[sP], pl);
                float pi = __shfl_sync(0xffffffffu, im[sP], pl);
                if (lane == 0) { pr = re[s0]; pi = im[s0]; }
                const float ar = zr + pr, ai = zi - pi;
                const float br = zi + pi, bi = pr - zr;
                const int k = lane + 32 * q;
                const bool valid = (q < 16) || (lane == 0);
                const float ma = valid ? 0.5f * sqrtf(fmaf(ar, ar, ai * ai)) : 0.f;
                const float mb = valid ? 0.5f * sqrtf(fmaf(br, br, bi * bi)) : 0.f;
                if (a.mag) {                               // (null: spectra only -- b200gate_torch_apply_masks)
                    dstA[k] = ma;
                    if (vb) dstA[kFPad + k] = mb;
                }
                if (a.dbg.ul == ul && valid && k < kF) {
                    float* sp = a.dbg.spec + ((long long)t * kF + k) * 2;
                    sp[0] = 0.5f * ar; sp[1] = 0.5f * ai;
                    if (vb) { sp[2 * kF] = 0.5f * br; sp[2 * kF + 1] = 0.5f * bi; }
                }
            }
        }
    }
}

struct IirArgs {
    int n_units, T;
    int F, FPad;               // bins and padded row pitch (513/544 for n_fft 1024, 1025/1056 for 2048)
    double b;                  // nonstationary.py:114
    float n_mult, slope;       // thresh_n_mult_nonstationary, sigmoid_slope_nonstationary
    int regen;                 // 1: regenerate the forward sweep in the backward pass instead of storing it
    const float* mag;          // [n_units][T][FPad]
    float* m0;                 // [n_units][T][FPad]: forward sweep, then overwritten by the sigmoid mask
    const UnitDesc* units;     // ROWS instantiations: units + (first unit of the batch); T is then the pitch only
};

template <int FP, bool ROWS = false>                    // padded row pitch: 544 (n_fft 1024) or 1056 (n_fft 2048)
__global__ void __launch_bounds__(128) k_iir_sigmoid(const IirArgs a) {
    const int FF = a.F;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)a.n_units * FP) return;
    const int ul = (int)(idx / FP), f = (int)(idx - (long long)ul * FP);
    const float* __restrict__ A = a.mag + (long long)ul * a.T * FP + f;
    float* M = a.m0 + (long long)ul * a.T * FP + f;
    // ROWS: the unit's own frame count, and its own choice between the two (differently rounding) variants below
    const int T = ROWS ? a.units[ul].T : a.T;
    const int regen = ROWS ? a.units[ul].regen : a.regen;
    if (f >= FF) {
        for (int t = 0; t < T; ++t) M[(long long)t * FP] = 0.f;
        return;
    }
    // The recurrence state stays in float64 (the filter pole 1 - b ~ 0.995 accumulates rounding over hundreds of
    // frames); the follower ratio, exponential and reciprocal run in float32 (the float64 exp / divide of the first
    // version made this kernel 3x longer than both FFT kernels together).  The sweeps are serial per (unit, bin), so
    // what bounds them is the latency of each step and the instructions around it: every recurrence is ONE fused
    // multiply-add on the carried value (the input term b x is formed off the chain); the |X| column is fetched in
    // batches of kB frames through a walking pointer with compile-time offsets (the row pitch is a template parameter),
    // the next batch requested before the current one is consumed, so no load sits between two steps of the chain;
    // the ratio is num * rcp(s) and the sigmoid a correctly rounded reciprocal (no division slow paths in the loop).
    constexpr int kB = 8;
    const double b = a.b, omb = 1.0 - a.b;
    const float n_mult = a.n_mult, slope = a.slope;
    auto sigmoid_mask = [&](double x, double sm) -> float {
        const float num = (float)(x - sm);                     // |X| - S without float32 cancellation
        const float r = num * __frcp_rn((float)sm);
        return __frcp_rn(1.0f + expf(-(r - n_mult) * slope));
    };
    // frames t0 + dir * j, j = 0..kB-1; `full`: all of them exist (compile-time offsets), else clamped (never used)
    auto fetch = [&](const float* src, float (&x)[kB], int t0, int dir) {
        const bool full = dir > 0 ? (t0 >= 0 && t0 + kB <= T) : (t0 < T && t0 - kB + 1 >= 0);
        if (full) {
            const float* p = src + (long long)t0 * FP;
            if (dir > 0) {
#pragma unroll
                for (int j = 0; j < kB; ++j) x[j] = p[j * FP];
            } else {
#pragma unroll
                for (int j = 0; j < kB; ++j) x[j] = p[-j * FP];
            }
        } else {
#pragma unroll
            for (int j = 0; j < kB; ++j) x[j] = src[(long long)min(max(t0 + dir * j, 0), T - 1) * FP];
        }
    };
    double s = (double)A[0];
    if (regen) {
        // The forward sweep is not stored: the backward sweep regenerates it by the inverse recurrence
        // fwd[t-1] = (fwd[t] - b x[t]) / (1 - b) in float64.  One read of |X| less, no forward write.  Its error
        // grows by 1/(1 - b) per step, and what matters is the error RELATIVE TO S, which in a quiet stretch can be
        // (1-b)^T below the loud values that set the absolute error.  Bound (u = 2^-53, f = exact forward sweep):
        //   * a step near frame j (forward fma and product, inverse fma and product, rounded coefficient) injects
        //     at most 5u f[j] / (1-b) (b x[j] <= f[j], f[j-1] <= f[j] / (1-b)); the inverse recurrence carries it to
        //     frame t < j multiplied by (1-b)^-(j-t), and the backward sweep's error is at most 1/(2-b) of that;
        //   * f[u] >= (1-b)^(u-j) f[j] for u >= j, so S[t] >= (1-b)^(j-t) f[j] / (2-b) for every j >= t;
        //   * so |dS[t]| / S[t] <= sum_j 5u/(1-b) (1-b)^-2(j-t)  <=  2.5 u (1-b)^(-2T) / b   (b < 0.5).
        // The host (iir_regen_ok) selects this variant only where that bound stays within 2^-24, the float32
        // rounding the stored variant puts on S: 2 T ln(1/(1-b)) - ln b <= 29 ln 2 - ln 2.5 = 19.19 (config 3: 19.00).
        // Longer chunks store the sweep: with T ln(1/(1-b)) = 19.4 (a 35 s single chunk at 16 kHz) the rebuilt sweep
        // put mask errors of 3e-3 on quiet-then-loud columns.
        {
            float cur[kB], nxt[kB];
            fetch(A, cur, 0, 1);
            int t0 = 0;
            for (; t0 + kB <= T; t0 += kB) {
                fetch(A, nxt, t0 + kB, 1);
#pragma unroll
                for (int j = 0; j < kB; ++j) s = fma(omb, s, b * (double)cur[j]);
#pragma unroll
                for (int j = 0; j < kB; ++j) cur[j] = nxt[j];
            }
#pragma unroll
            for (int j = 0; j < kB; ++j)
                if (t0 + j < T) s = fma(omb, s, b * (double)cur[j]);
        }
        const double inv_omb = 1.0 / omb, nb_inv = -b * inv_omb;
        double fw = s;                                         // fwd[T-1]
        float cur[kB], nxt[kB];
        fetch(A, cur, T - 1, -1);
        int t0 = T - 1;
        for (; t0 - kB + 1 >= 0; t0 -= kB) {
            fetch(A, nxt, t0 - kB, -1);
            float* mp = M + (long long)t0 * FP;
#pragma unroll
            for (int j = 0; j < kB; ++j) {
                const double x = (double)cur[j];
                s = fma(omb, s, b * fw);
                mp[-j * FP] = sigmoid_mask(x, s);
                fw = fma(inv_omb, fw, nb_inv * x);
            }
#pragma unroll
            for (int j = 0; j < kB; ++j) cur[j] = nxt[j];
        }
#pragma unroll
        for (int j = 0; j < kB; ++j) {
            if (t0 - j >= 0) {
                const double x = (double)cur[j];
                s = fma(omb, s, b * fw);
                M[(long long)(t0 - j) * FP] = sigmoid_mask(x, s);
                fw = fma(inv_omb, fw, nb_inv * x);
            }
        }
        return;
    }
    {
        float cur[kB], nxt[kB];
        fetch(A, cur, 0, 1);
        for (int t0 = 0; t0 < T; t0 += kB) {
            fetch(A, nxt, t0 + kB, 1);
#pragma unroll
            for (int j = 0; j < kB; ++j) {
                if (t0 + j < T) {
                    s = fma(omb, s, b * (double)cur[j]);
                    M[(long long)(t0 + j) * FP] = (float)s;
                }
            }
#pragma unroll
            for (int j = 0; j < kB; ++j) cur[j] = nxt[j];
        }
    }
    // (the stored forward sweep is read back through M itself -- each element before it is overwritten)
    const float* Mr = M;
    s = (double)Mr[(long long)(T - 1) * FP];
    for (int t0 = T - 1; t0 >= 0; t0 -= kB) {
        float fwv[kB], xx[kB];
        fetch(Mr, fwv, t0, -1);
        fetch(A, xx, t0, -1);
#pragma unroll
        for (int j = 0; j < kB; ++j) {
            if (t0 - j >= 0) {
                s = fma(omb, s, b * (double)fwv[j]);
                M[(long long)(t0 - j) * FP] = sigmoid_mask((double)xx[j], s);
            }
        }
    }
}

struct SmoothFArgs {
    int n_units, T;
    int F, FPad;
    int nf, nt;
    int tf_lo, tf_hi, TT;
    float p, one_minus_p;
    const float* m0;           // [n_units][T][FPad]
    float* m2;                 // [n_units][T][FPad]
    const UnitDesc* units;     // ROWS instantiations: units + (first unit of the batch); T is then the pitch only and
                               // tf_hi the largest of the batch
    StreamWin sw;              // STREAM instantiations: m0 / m2 are rings of sw.ring rows; T bounds the frames only
    const SessRow* rows;       // SESS instantiations: row ul's frames [s0, s1) and bound T (tf_lo, tf_hi and T unused)
};
__host__ __device__ inline int smoothf_cpitch(int FPad, int nf) { return FPad + 2 * nf + 1; }
inline size_t smoothf_smem_bytes(int TT, int FPad, int nf) { return (size_t)TT * smoothf_cpitch(FPad, nf) * 4; }

__global__ void __launch_bounds__(256) k_smooth_f(const SmoothFArgs a) {
    B200_DYN_SMEM(float, s_c);                         // [TT][cp]
    const int FP = a.FPad, FF = a.F;
    const int nt = a.nt, nf = a.nf, cp = smoothf_cpitch(a.FPad, nf);
    const int ul = blockIdx.y;
    const int t0 = a.tf_lo + blockIdx.x * a.TT;
    if (t0 >= a.tf_hi) return;
    const int tt_n = min(a.TT, a.tf_hi - t0);
    for (int i = threadIdx.x; i < a.TT * cp; i += blockDim.x) s_c[i] = 0.f;
    __syncthreads();
    const float* src = a.m0 + (long long)ul * a.T * FP;
    for (int i = threadIdx.x; i < tt_n * FP; i += blockDim.x) {
        const int tt = i / FP, f = i - tt * FP;
        if (f >= FF) continue;
        const int t = t0 + tt;
        float acc = 0.f;
        for (int bb = -nt; bb <= nt; ++bb) {
            const int tq = t - bb;
            if (tq >= 0 && tq < a.T) acc = fmaf((float)(nt + 1 - (bb < 0 ? -bb : bb)), src[(long long)tq * FP + f], acc);
        }
        s_c[tt * cp + nf + f] = acc;
    }
    __syncthreads();
    const float invD = 1.0f / ((float)((nf + 1) * (nf + 1)) * (float)((nt + 1) * (nt + 1)));
    float* dst = a.m2 + (long long)ul * a.T * FP;
    for (int i = threadIdx.x; i < tt_n * FP; i += blockDim.x) {
        const int tt = i / FP, f = i - tt * FP;
        float v = 0.f;
        if (f < FF) {
            const float* cr = s_c + tt * cp + f;
            float acc = 0.f;
            for (int d = -nf; d <= nf; ++d) acc = fmaf((float)(nf + 1 - (d < 0 ? -d : d)), cr[nf + d], acc);
            v = fmaf(acc * invD, a.p, a.one_minus_p);           // nonstationary.py:82-84
        }
        dst[(long long)(t0 + tt) * FP + f] = v;
    }
}

// Streaming form of the same smoothing (the one that normally runs; k_smooth_f above is kept as its tile-based
// cross-check).  A CTA walks a strip of frames of one unit; thread i owns bins i, i+G, i+2G, i+3G (G = FPad/4, so every
// shared-memory access of a warp is 32 consecutive floats): the last 2 nt + 1 mask rows live in a ring of thread-private
// columns (no barrier needed to refill it), the time-direction triangle is taken straight from the ring, the
// frequency-direction triangle from one zero-haloed row -- two barriers per frame, every mask value read from HBM
// once per strip and written once.
inline size_t smooths_smem_bytes(int FPad, int nf, int nt) { return ((size_t)(2 * nt + 1) * FPad + FPad + 2 * nf + 8) * 4; }

template <bool ROWS = false, bool STREAM = false, bool SESS = false>
__global__ void __launch_bounds__(288) k_smooth_stream(const SmoothFArgs a) {
    B200_DYN_SMEM(float, s_buf);
    const int FP = a.FPad, FF = a.F, nt = a.nt, nf = a.nf, R = 2 * nt + 1;
    const int G = blockDim.x, tid = threadIdx.x;
    float* ring = s_buf;                     // [R][FP]
    float* row = s_buf + (size_t)R * FP;     // [nf | FP | nf]
    const int ul = blockIdx.y;
    const int T = ROWS ? a.units[ul].T : SESS ? a.rows[ul].T : a.T;
    const int tf_hi = ROWS ? a.units[ul].tf_hi : SESS ? a.rows[ul].s1 : a.tf_hi;
    const int t_begin = (SESS ? a.rows[ul].s0 : a.tf_lo) + blockIdx.x * a.TT;
    if (t_begin >= tf_hi) return;
    const int t_end = min(t_begin + a.TT, tf_hi);
    const int pitch = STREAM ? a.sw.ring : a.T, rmask = STREAM ? a.sw.ring - 1 : -1;    // (row t: t & rmask)
    const float* src = a.m0 + (long long)ul * pitch * FP;
    float* dst = a.m2 + (long long)ul * pitch * FP;
    for (int i = tid; i < FP + 2 * nf; i += G) row[i] = 0.f;
    auto load_row = [&](int t, int slot) {
        const bool in = t >= 0 && t < T;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int bin = tid + j * G;
            ring[slot * FP + bin] = (in && bin < FF) ? src[(long long)(t & rmask) * FP + bin] : 0.f;
        }
    };
    // ring slot of frame t: (t - t_begin + nt) mod R, so the newest row t + nt of step t sits at slot (t - t_begin + 2 nt) mod R
    for (int k = 0; k < 2 * nt; ++k) load_row(t_begin - nt + k, k);
    int newest = (2 * nt) % R;
    const float invD = 1.0f / ((float)((nf + 1) * (nf + 1)) * (float)((nt + 1) * (nt + 1)));
    __syncthreads();
    for (int t = t_begin; t < t_end; ++t) {
        load_row(t + nt, newest);
        float c[4] = {0.f, 0.f, 0.f, 0.f};
        int slot = newest;                                  // frame t + nt; walking back to t - nt
        for (int b = -nt; b <= nt; ++b) {
            const float w = (float)(nt + 1 - (b < 0 ? -b : b));
#pragma unroll
            for (int j = 0; j < 4; ++j) c[j] = fmaf(w, ring[slot * FP + tid + j * G], c[j]);
            slot = slot == 0 ? R - 1 : slot - 1;
        }
        newest = newest + 1 == R ? 0 : newest + 1;
        __syncthreads();                                    // the previous frame's frequency pass has read `row`
#pragma unroll
        for (int j = 0; j < 4; ++j) row[nf + tid + j * G] = c[j];
        __syncthreads();
        float o[4] = {0.f, 0.f, 0.f, 0.f};
        for (int d = -nf; d <= nf; ++d) {
            const float w = (float)(nf + 1 - (d < 0 ? -d : d));
#pragma unroll
            for (int j = 0; j < 4; ++j) o[j] = fmaf(w, row[nf + tid + j * G + d], o[j]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int bin = tid + j * G;
            dst[(long long)(t & rmask) * FP + bin] = bin < FF ? fmaf(o[j] * invD, a.p, a.one_minus_p) : 0.f;      // nonstationary.py:82-84
        }
    }
}

// Box form of the streaming smoothing (the one that normally runs for 1 <= nf <= 12).  The triangle taps
// (n + 1 - |d|) are the self-convolution of a length-(n + 1) box, so the frequency direction is two sliding box sums
// instead of 2 nf + 1 multiply-adds per bin: thread i owns the four CONSECUTIVE bins 4i..4i+3 (every shared-memory
// access is one aligned 128-bit vector), takes the first box sum of each pass directly and the other three by
// add-one / drop-one.  Per four bins and frame: ~17 vector loads and ~75 floating-point instructions against the
// tap loops' ~120 scalar loads and ~120 FMAs.  The box sums restart in every thread and every frame, so no rounding
// accumulates along a row or over time.  Row buffers: rowA = time-smoothed row c[] with 16 zero floats either side,
// rowB = first box sums b1[g] = sum_{j=0..nf} c[g + j] stored at index g + 12 (g runs from -12: the second pass
// out[f] = sum_{g=f-nf..f} b1[g] reaches nf bins to the left); bins >= F hold zeros, and FPad - F >= 12.
inline size_t smoothb_smem_bytes(int FPad, int nt) { return ((size_t)(2 * nt + 1) * FPad + (FPad + 32) + (FPad + 16)) * 4; }

template <int NF, bool ROWS = false, bool STREAM = false, bool SESS = false>
__global__ void __launch_bounds__(288) k_smooth_box(const SmoothFArgs a) {
    static_assert(NF >= 1 && NF <= 12, "box smoothing handles 1 <= nf <= 12");
    B200_DYN_SMEM(float, s_buf);
    const int FP = a.FPad, FF = a.F, nt = a.nt, R = 2 * nt + 1;
    const int G = blockDim.x, tid = threadIdx.x;           // G == FP / 4
    float* ring = s_buf;                                   // [R][FP]
    float* rowA = s_buf + (size_t)R * FP;                  // [16 | FP | 16]
    float* rowB = rowA + FP + 32;                          // [FP + 16]
    const int ul = blockIdx.y;
    const int T = ROWS ? a.units[ul].T : SESS ? a.rows[ul].T : a.T;
    const int tf_hi = ROWS ? a.units[ul].tf_hi : SESS ? a.rows[ul].s1 : a.tf_hi;
    const int t_begin = (SESS ? a.rows[ul].s0 : a.tf_lo) + blockIdx.x * a.TT;
    if (t_begin >= tf_hi) return;
    const int t_end = min(t_begin + a.TT, tf_hi);
    const int pitch = STREAM ? a.sw.ring : a.T, rmask = STREAM ? a.sw.ring - 1 : -1;    // (row t: t & rmask)
    const float* src = a.m0 + (long long)ul * pitch * FP;
    float* dst = a.m2 + (long long)ul * pitch * FP;
    for (int i = tid; i < 2 * FP + 48; i += G) rowA[i] = 0.f;          // rowA and rowB are contiguous
    const int b0 = 4 * tid;
    auto fetch_row = [&](int t) -> float4 {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t >= 0 && t < T) {
            v = __ldg(reinterpret_cast<const float4*>(src + (long long)(t & rmask) * FP + b0));
            if (b0 + 0 >= FF) v.x = 0.f;
            if (b0 + 1 >= FF) v.y = 0.f;
            if (b0 + 2 >= FF) v.z = 0.f;
            if (b0 + 3 >= FF) v.w = 0.f;
        }
        return v;
    };
    for (int k = 0; k < 2 * nt; ++k) *reinterpret_cast<float4*>(ring + k * FP + b0) = fetch_row(t_begin - nt + k);
    int newest = (2 * nt) % R;
    const float invD = 1.0f / ((float)((NF + 1) * (NF + 1)) * (float)((nt + 1) * (nt + 1)));
    // the rows of the next two frames are requested while this frame is being smoothed: the only global load of the loop
    // otherwise sits right in front of its first use (long-scoreboard stalls were 3.8 cycles per issued instruction)
    float4 pre0 = fetch_row(t_begin + nt), pre1 = fetch_row(t_begin + nt + 1);
    __syncthreads();
    for (int t = t_begin; t < t_end; ++t) {
        *reinterpret_cast<float4*>(ring + newest * FP + b0) = pre0;
        pre0 = pre1;
        pre1 = (t + 2 < t_end) ? fetch_row(t + nt + 2) : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
        {
            // (measured and dropped: walking the ring in physical order with a rotating tap table -- fewer instructions per
            //  tap, but slower)
            int slot = newest;                              // frame t + nt; walking back to t - nt
            for (int b = -nt; b <= nt; ++b) {
                const float w = (float)(nt + 1 - (b < 0 ? -b : b));
                const float4 r = *reinterpret_cast<const float4*>(ring + slot * FP + b0);
                c.x = fmaf(w, r.x, c.x); c.y = fmaf(w, r.y, c.y); c.z = fmaf(w, r.z, c.z); c.w = fmaf(w, r.w, c.w);
                slot = slot == 0 ? R - 1 : slot - 1;
            }
        }
        newest = newest + 1 == R ? 0 : newest + 1;
        *reinterpret_cast<float4*>(rowA + 16 + b0) = c;     // (the previous frame's first pass finished before its 2nd barrier)
        __syncthreads();
        {   // first box: b1[g], g = b0 - 12 + m, from c[g .. g + NF] = rowA[16 + g ..]
            constexpr int NV = (4 + NF + 3) / 4;
            float v[4 * NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                const float4 q = *reinterpret_cast<const float4*>(rowA + b0 + 4 + 4 * k);
                v[4 * k] = q.x; v[4 * k + 1] = q.y; v[4 * k + 2] = q.z; v[4 * k + 3] = q.w;
            }
            float s0 = v[0];
#pragma unroll
            for (int j = 1; j <= NF; ++j) s0 += v[j];
            const float s1 = s0 + v[NF + 1] - v[0];
            const float s2 = s1 + v[NF + 2] - v[1];
            const float s3 = s2 + v[NF + 3] - v[2];
            *reinterpret_cast<float4*>(rowB + b0) = make_float4(s0, s1, s2, s3);   // (the previous frame's second pass finished before this frame's 1st barrier)
        }
        __syncthreads();
        {   // second box: out[f], f = b0 + m, from b1[f - NF .. f] = rowB[f + 12 - NF .. f + 12]
            constexpr int A0 = (12 - NF) & ~3, O = (12 - NF) & 3, NV = (16 - A0) / 4;
            float u[4 * NV];
#pragma unroll
            for (int k = 0; k < NV; ++k) {
                const float4 q = *reinterpret_cast<const float4*>(rowB + b0 + A0 + 4 * k);
                u[4 * k] = q.x; u[4 * k + 1] = q.y; u[4 * k + 2] = q.z; u[4 * k + 3] = q.w;
            }
            float o0 = u[O];
#pragma unroll
            for (int e = 1; e <= NF; ++e) o0 += u[O + e];
            const float o1 = o0 + u[O + NF + 1] - u[O];
            const float o2 = o1 + u[O + NF + 2] - u[O + 1];
            const float o3 = o2 + u[O + NF + 3] - u[O + 2];
            float4 r;                                                               // nonstationary.py:82-84
            r.x = b0 + 0 < FF ? fmaf(o0 * invD, a.p, a.one_minus_p) : 0.f;
            r.y = b0 + 1 < FF ? fmaf(o1 * invD, a.p, a.one_minus_p) : 0.f;
            r.z = b0 + 2 < FF ? fmaf(o2 * invD, a.p, a.one_minus_p) : 0.f;
            r.w = b0 + 3 < FF ? fmaf(o3 * invD, a.p, a.one_minus_p) : 0.f;
            *reinterpret_cast<float4*>(dst + (long long)(t & rmask) * FP + b0) = r;
        }
    }
}

// =============================================================================================
// TorchGate surface (noisereduce/torchgate/torchgate.py:200-264).  Same analysis / synthesis kernels;
// what differs is the mask: statistics per (row, bin) over the row's own frames (or over xn's),
// top_db = 40, unbiased std (torchgate.py:127-165, torchgate/utils.py:6-23), and for the
// non-stationary variant a moving mean instead of the IIR (torchgate.py:168-198).
// =============================================================================================
struct TStatArgs {
    int n_units, T;
    float in_scale;            // sum(window): TorchGate's STFT is not normalised
    float eps;                 // torch.finfo(float64).eps added in float32
    float top_db;
    float n_std;
    int ddof;
    float* mag;                // in: |X| / sum(w);  out: dB (float32), unclamped
    float* rowmax;             // [n_units][FPad] max_t dB
    float* thr;                // [n_units][FPad] mean + n_std * std of the clamped dB
    const UnitDesc* units;     // ROWS instantiations: units + (first unit of the batch); T is then the pitch only
};

// One CTA per (unit, 32-bin group); its kTgWarps warps share the frames (warp w takes t = w, w + kTgWarps, ...), every access
// of a warp is one 128-byte row segment, and the per-bin max / sum / sum of squares are combined through shared memory in
// warp order (deterministic).  One thread per (unit, bin) walking all T frames -- the first form of these kernels -- left
// a 256-row batch with 139 k threads and the column walks latency-bound (0.38 + 0.29 ms of a 1.47 ms forward).
constexpr int kTgWarps = 8;

template <bool ROWS = false>
__global__ void __launch_bounds__(kTgWarps * 32) k_tgate_stats(const TStatArgs a) {
    __shared__ double s_red[kTgWarps][32];
    __shared__ float s_mx[kTgWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int ul = blockIdx.x / kFW, grp = blockIdx.x - ul * kFW;
    const int T = ROWS ? a.units[ul].T : a.T;             // ROWS: the unit's own frames
    const int f = grp * 32 + lane;
    const long long idx = (long long)ul * kFPad + f;
    float* D = a.mag + (long long)ul * a.T * kFPad + f;
    const bool live = f < kF;
    float mx = -INFINITY;
    if (live) {
#pragma unroll 4
        for (int t = w; t < T; t += kTgWarps) {
            const float db = 20.0f * log10f(D[(long long)t * kFPad] * a.in_scale + a.eps);
            D[(long long)t * kFPad] = db;
            mx = fmaxf(mx, db);
        }
    }
    s_mx[w][lane] = mx;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kTgWarps; ++k) mx = fmaxf(mx, s_mx[k][lane]);
    const float fl = mx - a.top_db;
    double sum = 0.0;
    if (live) {
#pragma unroll 4
        for (int t = w; t < T; t += kTgWarps) sum += (double)fmaxf(D[(long long)t * kFPad], fl);     // (this thread's own stores)
    }
    s_red[w][lane] = sum;
    __syncthreads();
    sum = 0.0;
#pragma unroll
    for (int k = 0; k < kTgWarps; ++k) sum += s_red[k][lane];
    const double mean = sum / T;
    __syncthreads();
    double ss = 0.0;
    if (live) {
#pragma unroll 4
        for (int t = w; t < T; t += kTgWarps) {
            const double d = (double)fmaxf(D[(long long)t * kFPad], fl) - mean;
            ss += d * d;
        }
    }
    s_red[w][lane] = ss;
    __syncthreads();
    if (w == 0) {
        ss = 0.0;
#pragma unroll
        for (int k = 0; k < kTgWarps; ++k) ss += s_red[k][lane];
        const double sd = sqrt(ss / (double)(T - a.ddof));
        a.rowmax[idx] = live ? mx : -INFINITY;
        a.thr[idx] = live ? (float)(mean + sd * (double)a.n_std) : INFINITY;
    }
}

struct TBitsArgs {
    int n_units, T;
    int thr_units;             // rows of thr: n_units (self / per-row xn) or 1 (broadcast)
    float top_db;
    const float* db;           // [n_units][T][FPad]
    const float* rowmax;       // [n_units][FPad]  (of x itself)
    const float* thr;          // [thr_units][FPad]
    unsigned* bits;            // [n_units][T][FW]
    const UnitDesc* units;     // ROWS instantiations: units + (first unit of the batch); T is then the pitch only
};

template <bool ROWS = false>
__global__ void __launch_bounds__(kTgWarps * 32) k_tgate_bits(const TBitsArgs a) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int ul = blockIdx.x / kFW, grp = blockIdx.x - ul * kFW;
    const int T = ROWS ? a.units[ul].T : a.T;             // ROWS: the unit's own frames
    const int f = grp * 32 + lane;
    const float* D = a.db + (long long)ul * a.T * kFPad + f;
    const float fl = a.rowmax[(long long)ul * kFPad + f] - a.top_db;
    const float th = a.thr[(long long)(a.thr_units == 1 ? 0 : ul) * kFPad + f];
    const bool live = f < kF;
    unsigned* brow = a.bits + (long long)ul * a.T * kFW + grp;
    constexpr int kU = 4;                                   // rows requested together, then voted on
    for (int t0 = w; t0 < T; t0 += kU * kTgWarps) {
        float v[kU];
#pragma unroll
        for (int j = 0; j < kU; ++j) {
            const int t = t0 + j * kTgWarps;
            v[j] = (t < T) ? D[(long long)t * kFPad] : -INFINITY;
        }
#pragma unroll
        for (int j = 0; j < kU; ++j) {
            const int t = t0 + j * kTgWarps;
            const unsigned word = __ballot_sync(0xffffffffu, live && (fmaxf(v[j], fl) > th));
            if (t < T && lane == 0) brow[(long long)t * kFW] = word;
        }
    }
}

struct TMovArgs {
    int n_units, T;
    int n_movemean;
    float n_thresh, inv_temp, p;
    const float* mag;
    float* m0;                 // blended sigmoid mask, prop_decrease * (m - 1) + 1 (torchgate.py:241)
    const UnitDesc* units;     // ROWS instantiations: units + (first unit of the batch); T is then the pitch only
    StreamWin sw;              // STREAM instantiations: frames [sw.f0, f1) of the rings; T bounds the frames only
    int f1;
    double* run;               // STREAM: [n_units][FPad] the running sums, carried from one launch to the next
    const SessRow* rows;       // SESS instantiations: row ul's frames [m0, m1) and bound T (sw.f0, f1 and T unused)
};

// STREAM: frames [sw.f0, f1) of a stream whose rows have T frames (T = INT_MAX while the end is not known: the caller
// then has |X| up to frame f1 + right).  The running sum is loaded from a.run, receives the same adds and subtracts in
// the same order as the walk from t = 0 below, and is stored back, so its rounding is that of the whole-row walk.
// SESS: the same per row; a session's first launch starts at frame 0 and builds the sum afresh, so a row that starts a
// new session never reads the sum its previous session left.
template <bool ROWS = false, bool STREAM = false, bool SESS = false>
__global__ void __launch_bounds__(128) k_tgate_movmean(const TMovArgs a) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)a.n_units * kFPad) return;
    const int ul = (int)(idx / kFPad), f = (int)(idx - (long long)ul * kFPad);
    const int T = ROWS ? a.units[ul].T : SESS ? a.rows[ul].T : a.T;   // ROWS: the unit's own frames (conv1d's "same" edges)
    const int pitch = STREAM ? a.sw.ring : a.T, rmask = STREAM ? a.sw.ring - 1 : -1;    // (row t: t & rmask)
    const int t0 = SESS ? a.rows[ul].m0 : STREAM ? a.sw.f0 : 0, t1 = SESS ? a.rows[ul].m1 : STREAM ? a.f1 : T;
    if (SESS && t0 >= t1) return;
    const float* A = a.mag + (long long)ul * pitch * kFPad + f;
    float* M = a.m0 + (long long)ul * pitch * kFPad + f;
    if (f >= kF) {
        for (int t = t0; t < t1; ++t) M[(long long)(t & rmask) * kFPad] = 0.f;
        return;
    }
    // conv1d(ones(n), padding="same"): window [t - left, t + right], zero padded, left = (n-1)/2
    const int n = a.n_movemean, left = (n - 1) / 2, right = n - 1 - left;
    double run = 0.0;
    if (t0 == 0) {
        for (int t = 0; t <= right && t < T; ++t) run += (double)A[(long long)(t & rmask) * kFPad];
    } else {
        run = a.run[idx];
    }
    for (int t = t0; t < t1; ++t) {
        const float Av = A[(long long)(t & rmask) * kFPad];
        const float S = (float)(run / (double)n);
        const float r = (Av - S) / S;
        const float m = 1.0f / (1.0f + expf(-(r - a.n_thresh) * a.inv_temp));
        M[(long long)(t & rmask) * kFPad] = a.p * (m - 1.0f) + 1.0f;
        const int tin = t + 1 + right, tout = t - left;
        if (tin < T) run += (double)A[(long long)(tin & rmask) * kFPad];
        if (tout >= 0) run -= (double)A[(long long)(tout & rmask) * kFPad];
    }
    if (STREAM) a.run[idx] = run;
}

// =============================================================================================
// dtype conversion at the edges (base.py:140 promotes every chunk to float64; :218-226 casts back)
// =============================================================================================
template <typename Tin>
__global__ void k_to_f32(const Tin* __restrict__ src, float* __restrict__ dst, long long C, long long n,
                         long long sstride, long long dstride) {
    const long long total = C * n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long c = i / n, j = i - c * n;
        dst[c * dstride + j] = (float)src[c * sstride + j];
    }
}
template <typename Tout>
__device__ __forceinline__ Tout cast_out(float v);
template <> __device__ __forceinline__ double cast_out<double>(float v) { return (double)v; }
template <> __device__ __forceinline__ short cast_out<short>(float v) {
    // numpy float -> int16 astype: C truncation toward zero, wrapping the low 16 bits
    return (short)(int)v;
}
template <typename Tout>
__global__ void k_from_f32(const float* __restrict__ src, Tout* __restrict__ dst, long long C, long long n,
                           long long sstride, long long dstride) {
    const long long total = C * n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long c = i / n, j = i - c * n;
        dst[c * dstride + j] = cast_out<Tout>(src[c * sstride + j]);
    }
}

// =============================================================================================
// K0: one-time stationary noise statistics (stationary.py:61-81), float64.
// =============================================================================================
// sequential channel sum in channel order (np.mean(axis=0) adds rows in order; float32 stays float32)
template <typename Tin, typename Tacc>
__global__ void k0_channel_sum(const Tin* __restrict__ y, long long C, long long n, long long stride,
                               Tacc* __restrict__ acc, int init) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        Tacc s = init ? (Tacc)0 : acc[i];
        for (long long c = 0; c < C; ++c) s = s + (Tacc)y[c * stride + i];
        acc[i] = s;
    }
}
template <typename Tacc>
__global__ void k0_mean_to_f64(const Tacc* __restrict__ acc, long long n, long long C, double* __restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        out[i] = (double)(acc[i] / (Tacc)C);          // division in the accumulation dtype, as numpy
}

// One CTA per frame: float64 radix-2 FFT in shared memory -> dB (utils.py:15), [Tn][F].
struct K0Args {
    const double* yn;      // [n] collapsed noise clip
    long long n;
    int H, Tn;
    const double* wa64;
    const double2* cs64;
    double eps;
    double* db;            // [Tn][F]
};
// frame t of the clip yn[0, n) into db[t][F] (the body of k0_stft_db and k0_stft_db_rows)
__device__ __forceinline__ void k0_stft_db_frame(const K0Args& a, const double* yn, long long n_yn, int t, double* db,
                                                 double2* s) {
    const long long base = (long long)t * a.H - kN / 2;
    for (int n = threadIdx.x; n < kN; n += blockDim.x) {
        const long long j = base + n;
        const double v = (j >= 0 && j < n_yn) ? yn[j] * a.wa64[n] : 0.0;
        int r = 0;
        for (int b = 0; b < 10; ++b) r |= ((n >> b) & 1) << (9 - b);
        s[r] = make_double2(v, 0.0);
    }
    __syncthreads();
    for (int len = 2; len <= kN; len <<= 1) {
        const int half = len >> 1, stride = kN / len;
        for (int i = threadIdx.x; i < kN / 2; i += blockDim.x) {
            const int blk = i / half, o = i - blk * half;
            const int ia = blk * len + o, ib = ia + half;
            const double2 w = a.cs64[o * stride];                 // exp(-i th) = cos - i sin
            const double2 x = s[ia], y = s[ib];
            const double yr = y.x * w.x + y.y * w.y, yi = y.y * w.x - y.x * w.y;
            s[ia] = make_double2(x.x + yr, x.y + yi);
            s[ib] = make_double2(x.x - yr, x.y - yi);
        }
        __syncthreads();
    }
    for (int f = threadIdx.x; f < kF; f += blockDim.x) {
        const double2 v = s[f];
        db[(long long)t * kF + f] = 20.0 * log10(sqrt(v.x * v.x + v.y * v.y) + a.eps);
    }
}
__global__ void __launch_bounds__(256) k0_stft_db(const K0Args a) {
    B200_DYN_SMEM(double2, s);                      // [N]
    k0_stft_db_frame(a, a.yn, a.n, blockIdx.x, a.db, s);
}

// b200gate_noise_stats_rows: a group of clips, each with its own length and frame count, in one launch of each kernel
struct K0Clip {
    const void* x;          // sample 0 of channel 0: the clip's samples (device clips) or its channel sums (host clips)
    long long stride;       // elements between channels
    long long c_sum;        // channels summed here: C (device clips), 1 (host clips, summed on the host in channel order)
    long long C;            // channels of the clip: the divisor of the mean
    long long n;            // samples after clipping
    long long yn_off;       // offset of its float64 mean in the group's buffer
    long long t_off;        // its frames are rows [t_off, t_off + Tn) of the group's dB buffer
    int Tn;                 // n / H + 1
};

// channel sum in channel order and mean in the accumulation dtype (k0_channel_sum + k0_mean_to_f64); grid.y = clip
template <typename Tin, typename Tacc>
__global__ void k0_clip_mean_rows(const K0Clip* __restrict__ clips, double* __restrict__ yn) {
    const K0Clip c = clips[blockIdx.y];
    const Tin* y = static_cast<const Tin*>(c.x);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < c.n;
         i += (long long)gridDim.x * blockDim.x) {
        Tacc s = (Tacc)0;
        for (long long ch = 0; ch < c.c_sum; ++ch) s = s + (Tacc)y[ch * c.stride + i];
        yn[c.yn_off + i] = (double)(s / (Tacc)c.C);
    }
}

// one CTA per frame of the group (blockIdx.x: row of the group's dB buffer), as k0_stft_db per clip
__global__ void __launch_bounds__(256) k0_stft_db_rows(const K0Args a, const K0Clip* __restrict__ clips, int n_clips) {
    B200_DYN_SMEM(double2, s);                      // [N]
    const int t = blockIdx.x;
    int lo = 0, hi = n_clips - 1;                   // the clip whose frames hold row t
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (clips[mid].t_off <= t) lo = mid; else hi = mid - 1;
    }
    const K0Clip& c = clips[lo];
    k0_stft_db_frame(a, a.yn + c.yn_off, c.n, t - (int)c.t_off, a.db + c.t_off * kF, s);
}

// One CTA per bin: top_db floor, mean, std (ddof), thresh (the body of k0_stats and k0_stats_rows).
__device__ __forceinline__ void k0_stats_bin(const double* __restrict__ db, int Tn, int F, int f, double top_db, int ddof,
                                             double n_std, double* __restrict__ mean_out, double* __restrict__ std_out,
                                             double* __restrict__ thr_out) {
    __shared__ double red[256];
    double m = -1.0e300;
    for (int t = threadIdx.x; t < Tn; t += blockDim.x) m = fmax(m, db[(long long)t * F + f]);
    red[threadIdx.x] = m;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + o]);
        __syncthreads();
    }
    const double fl = red[0] - top_db;
    __syncthreads();
    double sum = 0.0;
    for (int t = threadIdx.x; t < Tn; t += blockDim.x) sum += fmax(db[(long long)t * F + f], fl);
    red[threadIdx.x] = sum;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    const double mean = red[0] / Tn;
    __syncthreads();
    double ss = 0.0;
    for (int t = threadIdx.x; t < Tn; t += blockDim.x) {
        const double d = fmax(db[(long long)t * F + f], fl) - mean;
        ss += d * d;
    }
    red[threadIdx.x] = ss;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double sd = sqrt(red[0] / (double)(Tn - ddof));
        mean_out[f] = mean;
        std_out[f] = sd;
        thr_out[f] = mean + sd * n_std;
    }
}
__global__ void __launch_bounds__(256) k0_stats(const double* __restrict__ db, int Tn, int F, double top_db, int ddof,
                                                double n_std, double* __restrict__ mean_out,
                                                double* __restrict__ std_out, double* __restrict__ thr_out) {
    k0_stats_bin(db, Tn, F, blockIdx.x, top_db, ddof, n_std, mean_out, std_out, thr_out);
}
// grid (F, clips): clip blockIdx.y of the group; res holds [clips][3][F] (mean, std, thresh)
__global__ void __launch_bounds__(256) k0_stats_rows(const double* __restrict__ db, const K0Clip* __restrict__ clips,
                                                     double top_db, int ddof, double n_std, double* __restrict__ res) {
    const K0Clip& c = clips[blockIdx.y];
    double* r = res + (long long)blockIdx.y * 3 * kF;
    k0_stats_bin(db + c.t_off * kF, c.Tn, kF, blockIdx.x, top_db, ddof, n_std, r, r + kF, r + 2 * kF);
}

}  // namespace b200
