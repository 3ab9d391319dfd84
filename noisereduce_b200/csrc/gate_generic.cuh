// gate_generic.cuh -- the general-geometry kernel family (numpy surface).
//
// The tuned kernels (gate_kernels.cuh, gate_kernels_2k.cuh) cover the reference's default STFT geometry.  Every
// other geometry reduce_noise() accepts -- any power-of-two n_fft, any win_length <= n_fft, any hop_length <=
// win_length, both gates (noisereduce.py:13-36, spectralgate/base.py:79-86) -- runs here: the same pipeline,
// staged through HBM in float64, one CTA per frame with a shared-memory radix-2 FFT.  It is the path that makes
// the library a drop-in for those calls, not the one the roofline numbers are quoted on.
//
//   gk_stft      scipy.signal.stft(nfft=N, nperseg=W, noverlap=W-H, padded=False)         stationary.py:87-93
//   gk_decide    _amp_to_db + top_db row floor + `> thresh` + prop_decrease blend          stationary.py:95-110
//   gk_follow    filtfilt one-pole follower + sigmoid mask                                 nonstationary.py:59-76
//   gk_smooth_f / gk_smooth_t   fftconvolve(mask, filter, 'same') as its two integer-tap passes   base.py:14-28
//   gk_istft     irfft of X * mask, synthesis window                                       stationary.py:117-125
//   gk_ola       overlap-add, sum(w^2) normalisation, centre crop, cast                   scipy istft; base.py:150
#pragma once
#include "gate_kernels.cuh"

namespace b200 {

struct GGeom {
    Geom g;                 // chunk table; g.T = (Lp + 2 (W/2) - W) / H + 1
    int N, logN, W, F;      // n_fft, log2 (power-of-two n_fft), frame length (win_length; n_fft on the torch surface), N/2 + 1
    int M, logM;            // n_fft not a power of two: Bluestein length M = 2^logM >= 2 N - 1 (else 0)
    long long out_len;      // > 0: samples written per row (torch surface: (L / H) * H); 0: the chunk centre
    long long crop;         // > 0 (chunked torch surface): the chunk centre is cut to the unit's torch output length
                            // minus the padding, as the reference's slice of a short TorchGate output is
};

struct GTables {
    const double* wa;       // [W] analysis window / sum(w)
    const double* ws;       // [W] synthesis window * sum(w) / N
    const double* w2;       // [W] w^2 (overlap-add norm)
    const double2* cs;      // [N] (cos, sin)(2 pi m / N); Bluestein: [M] for the length-M transforms
    const double2* chirp;   // Bluestein: [N] exp(-i pi n^2 / N)
    const double2* bbr;     // Bluestein: [M] FFT_M of the conjugate chirp kernel, / M, in bit-reversed order
};

// In-place radix-2 DIT FFT of s[N] (input already in bit-reversed order); sgn = -1 forward, +1 inverse (unscaled).
__device__ __forceinline__ void gk_fft_smem(double2* s, int N, const double2* __restrict__ cs, double sgn) {
    for (int len = 2; len <= N; len <<= 1) {
        const int half = len >> 1, stride = N / len;
        for (int i = threadIdx.x; i < N / 2; i += blockDim.x) {
            const int blk = i / half, o = i - blk * half;
            const int ia = blk * len + o, ib = ia + half;
            const double2 w = cs[o * stride];
            const double wi = sgn * w.y;                               // exp(sgn i th)
            const double2 x = s[ia], y = s[ib];
            const double yr = y.x * w.x - y.y * wi, yi = y.y * w.x + y.x * wi;
            s[ia] = make_double2(x.x + yr, x.y + yi);
            s[ib] = make_double2(x.x - yr, x.y - yi);
        }
        __syncthreads();
    }
}
__device__ __forceinline__ int gk_brev(int n, int logN) {
    int r = 0;
    for (int b = 0; b < logN; ++b) r |= ((n >> b) & 1) << (logN - 1 - b);
    return r;
}
// Radix-2 DIF, natural order in -> bit-reversed order out, forward sign.
__device__ __forceinline__ void gk_fft_dif_smem(double2* s, int N, const double2* __restrict__ cs) {
    for (int len = N; len >= 2; len >>= 1) {
        const int half = len >> 1, stride = N / len;
        for (int i = threadIdx.x; i < N / 2; i += blockDim.x) {
            const int blk = i / half, o = i - blk * half;
            const int ia = blk * len + o, ib = ia + half;
            const double2 w = cs[o * stride];                          // exp(-i th) = (cos, -sin)
            const double2 x = s[ia], y = s[ib];
            const double dr = x.x - y.x, di = x.y - y.y;
            s[ia] = make_double2(x.x + y.x, x.y + y.y);
            s[ib] = make_double2(dr * w.x + di * w.y, di * w.x - dr * w.y);
        }
        __syncthreads();
    }
}

// The length-N forward DFT both transforms are built on.
//   power-of-two N : the caller stores element n at s[gk_slot(n)] (bit-reversed), gk_dft returns X in s[0..N).
//   any other N    : Bluestein's chirp-z: the caller stores v[n] * chirp[n] at s[n] and zeros up to M; gk_dft leaves
//                    the circular convolution with the conjugate chirp in s, and X[k] = s[k] * chirp[k].
// gk_in / gk_out apply the chirp factors so the kernels read the same for both.
__device__ __forceinline__ int gk_len(const GGeom& gg) { return gg.M ? gg.M : gg.N; }
__device__ __forceinline__ int gk_slot(const GGeom& gg, int n) { return gg.M ? n : gk_brev(n, gg.logN); }
__device__ __forceinline__ double2 gk_in(const GGeom& gg, const GTables& tb, int n, double2 v) {
    if (!gg.M) return v;
    const double2 c = tb.chirp[n];
    return make_double2(v.x * c.x - v.y * c.y, v.x * c.y + v.y * c.x);
}
__device__ __forceinline__ double2 gk_out(const GGeom& gg, const GTables& tb, int k, double2 v) { return gk_in(gg, tb, k, v); }
__device__ __forceinline__ void gk_dft(double2* s, const GGeom& gg, const GTables& tb) {
    if (!gg.M) {
        gk_fft_smem(s, gg.N, tb.cs, -1.0);
        return;
    }
    gk_fft_dif_smem(s, gg.M, tb.cs);
    for (int i = threadIdx.x; i < gg.M; i += blockDim.x) {
        const double2 a = s[i], b = tb.bbr[i];
        s[i] = make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
    }
    __syncthreads();
    gk_fft_smem(s, gg.M, tb.cs, 1.0);
}

// ---- STFT: one CTA per (frame, unit) ---------------------------------------------------------------------
template <typename T>
struct GStftArgs {
    GGeom gg;
    GTables tb;
    const T* x;
    double2* X;             // [n_units][T][F]
};
// sum of w^2 over the frames overlapping padded-chunk index i (gk_ola's normaliser; 1 where it is <= 1e-10)
__device__ __forceinline__ double gk_norm(const GGeom& gg, const GTables& tb, long long i) {
    const int W = gg.W, H = gg.g.H;
    const long long j = i + W / 2;
    long long t_lo = (j - W + H) / H;
    if (j - W + 1 <= 0) t_lo = 0;
    const long long t_hi = min((long long)(gg.g.T - 1), j / H);
    double nrm = 0.0;
    for (long long t = t_lo; t <= t_hi; ++t) nrm += tb.w2[(int)(j - t * H)];
    return nrm > 1e-10 ? nrm : 1.0;
}

// ADJ (b200gate_adjoint): x is the gradient of the output; the frames read it on the unit's centre only, divided by
// the overlap-add norm, and zero elsewhere (the adjoint of gk_ola's normalise-and-crop)
template <typename T, bool ADJ = false>
__global__ void __launch_bounds__(256) gk_stft(const GStftArgs<T> a) {
    B200_DYN_SMEM(double2, s);
    const Geom& g = a.gg.g;
    const int N = a.gg.N, W = a.gg.W, F = a.gg.F;
    const int t = blockIdx.x, ul = blockIdx.y;
    const int u = g.u0 + ul;
    const long long chunk = u / g.C, ch = u - chunk * g.C;
    const long long i1 = chunk * g.step - g.pad;
    const T* xrow = a.x + ch * g.in_stride;
    const long long base = (long long)t * g.H - W / 2;            // boundary='zeros': W/2 zeros either side
    const int len = gk_len(a.gg);
    long long c_hi = 0;                                            // ADJ: end of the centre the forward writes
    if (ADJ) {
        c_hi = g.pad + min((long long)g.step, (long long)(g.n_total - chunk * g.step));
        c_hi = min(c_hi, (long long)(g.T - 1) * g.H + (W & 1));
    }
    for (int n = threadIdx.x; n < len; n += blockDim.x) {
        double v = 0.0;
        if (ADJ) {
            const long long j = base + n;
            if (n < W && j >= g.pad && j < c_hi) v = ld_sample_f64(xrow + i1 + j) / gk_norm(a.gg, a.tb, j) * a.tb.wa[n];
        } else if (n < W) v = chunk_sample_f64(xrow, base + n, i1, g.Lp, g.n_total) * a.tb.wa[n];
        const double2 z = n < N ? gk_in(a.gg, a.tb, n, make_double2(v, 0.0)) : make_double2(0.0, 0.0);
        s[n < N ? gk_slot(a.gg, n) : n] = z;                      // rfft(n=N): zero-padded at the end
    }
    __syncthreads();
    gk_dft(s, a.gg, a.tb);
    double2* Xr = a.X + ((size_t)ul * g.T + t) * F;
    for (int f = threadIdx.x; f < F; f += blockDim.x) Xr[f] = gk_out(a.gg, a.tb, f, s[f]);
}

// ---- stationary decision ---------------------------------------------------------------------------------
// (1) gk_db_rowmax: dB of every bin (utils.py:15) and the per-(unit, bin) maximum over the frames -- a CTA covers a
//     64-bin x 64-frame tile, reduces its column maxima in shared memory and merges them with one atomicMax per
//     column on an order-preserving integer image of the double;  (2) gk_decide: element-wise floor, compare, blend.
__device__ __forceinline__ unsigned long long gk_ord(double v) {          // monotone double -> uint64
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double gk_unord(unsigned long long k) {
    const unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)b);
}
struct GDbArgs {
    int n_units, T, F;
    double eps;
    const double2* X;
    double* M;                     // [n_units][T][F] dB
    unsigned long long* rowmax;    // [n_units][F] gk_ord(max_t dB); zeroed by the host (0 = below every double)
};
__global__ void __launch_bounds__(256) gk_db_rowmax(const GDbArgs a) {
    __shared__ double red[4][64];
    const int fx = threadIdx.x & 63, ty = threadIdx.x >> 6;
    const int f = blockIdx.x * 64 + fx;
    const int t0 = blockIdx.y * 64;
    const int ul = blockIdx.z;
    double mx = -1.0e300;
    if (f < a.F) {
        const size_t base = (size_t)ul * a.T * a.F + f;
        const int t1 = min(t0 + 64, a.T);
        for (int t = t0 + ty; t < t1; t += 4) {
            const double2 v = a.X[base + (size_t)t * a.F];
            const double db = 20.0 * log10(hypot(v.x, v.y) + a.eps);         // utils.py:15
            a.M[base + (size_t)t * a.F] = db;
            mx = fmax(mx, db);
        }
    }
    red[ty][fx] = mx;
    __syncthreads();
    if (ty == 0 && f < a.F) {
        mx = fmax(fmax(red[0][fx], red[1][fx]), fmax(red[2][fx], red[3][fx]));
        atomicMax(a.rowmax + (size_t)ul * a.F + f, gk_ord(mx));
    }
}

struct GDecideArgs {
    int n_units, T, F;
    double top_db, p;
    const double* thr;      // [thr_units][F] dB (thr_units 1: shared by every unit)
    int thr_units;
    int thr_rows;           // > 0: unit ul reads row (thr_u0 + ul) % thr_rows (the noise clip's rows are channels)
    long long thr_u0;
    const unsigned long long* rowmax;
    double* M;              // dB in, mask0 * p + (1 - p) out
    int dbg_ul, FW;
    unsigned* dbg_bits;     // [T][FW] of the tapped unit (zeroed by the host)
};
__global__ void __launch_bounds__(256) gk_decide(const GDecideArgs a) {
    const long long total = (long long)a.n_units * a.T * a.F;
    const long long TF = (long long)a.T * a.F;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ul = (int)(i / TF);
        const long long r = i - (long long)ul * TF;
        const int t = (int)(r / a.F), f = (int)(r - (long long)t * a.F);
        const double fl = gk_unord(a.rowmax[(size_t)ul * a.F + f]) - a.top_db;
        const long long tr = a.thr_units == 1 ? 0 : (a.thr_rows > 0 ? (a.thr_u0 + ul) % a.thr_rows : ul);
        const double th = a.thr[(size_t)tr * a.F + f];
        const bool on = fmax(a.M[i], fl) > th;                               // utils.py:16, stationary.py:99-106
        a.M[i] = (on ? 1.0 : 0.0) * a.p + (1.0 - a.p);                       // stationary.py:108-110
        if (ul == a.dbg_ul && on) atomicOr(a.dbg_bits + (size_t)t * a.FW + (f >> 5), 1u << (f & 31));
    }
}

// ---- non-stationary follower + sigmoid ------------------------------------------------------------------------
// gk_abs (element-wise |X|) -> gk_follow (one thread per (unit, bin): the two one-pole sweeps, 2 FMAs per frame)
// -> gk_sigmoid (element-wise mask).
__global__ void __launch_bounds__(256) gk_abs(const double2* __restrict__ X, long long n, double* __restrict__ A) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const double2 v = X[i];
        A[i] = hypot(v.x, v.y);
    }
}
struct GFollowArgs {
    int n_units, T, F;
    double b;
    const double* A;        // |X|
    double* S;              // forward sweep, then the smoothed floor
};
__global__ void __launch_bounds__(128) gk_follow(const GFollowArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)a.n_units * a.F) return;
    const int ul = (int)(i / a.F), f = (int)(i - (long long)ul * a.F);
    const size_t o = (size_t)ul * a.T * a.F + f;
    const double* A = a.A + o;
    double* S = a.S + o;
    const double b = a.b, c = 1.0 - a.b;
    double s = A[0];                                                         // lfilter_zi steady state: s[-1] = x[0]
    for (int t = 0; t < a.T; ++t) {
        s = b * A[(size_t)t * a.F] + c * s;
        S[(size_t)t * a.F] = s;
    }
    for (int t = a.T - 1; t >= 0; --t) {                                     // same sweep backwards, started at its last value
        s = b * S[(size_t)t * a.F] + c * s;
        S[(size_t)t * a.F] = s;
    }
}
struct GSigmoidArgs {
    long long n;
    double n_mult, slope, p;
    int blend;              // 1: no smoothing follows -> apply prop_decrease here (nonstationary.py:82-84)
    const double* S;
    double* M;              // |X| in, mask out
};
__global__ void __launch_bounds__(256) gk_sigmoid(const GSigmoidArgs a) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (long long)gridDim.x * blockDim.x) {
        const double s = a.S[i];
        const double r = (a.M[i] - s) / s;                                   // nonstationary.py:70
        double m = 1.0 / (1.0 + exp(-(r - a.n_mult) * a.slope));             // utils.py:4-8
        if (a.blend) m = m * a.p + (1.0 - a.p);
        a.M[i] = m;
    }
}

// ---- smoothing: triangular taps (n + 1 - |k|), zero outside the spectrogram -----------------------------
struct GSmoothArgs {
    int n_units, T, F, nf, nt;
    double inv_D, p;
    int blend;              // time pass: 1 -> out = out * p + (1 - p) (non-stationary gate blends after smoothing)
    const double* src;
    double* dst;
};
__global__ void __launch_bounds__(256) gk_smooth_f(const GSmoothArgs a) {
    const long long total = (long long)a.n_units * a.T * a.F;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int f = (int)(i % a.F);
        const double* row = a.src + (i - f);
        double acc = 0.0;
        const int lo = max(-a.nf, -f), hi = min(a.nf, a.F - 1 - f);
        for (int d = lo; d <= hi; ++d) acc += (double)(a.nf + 1 - abs(d)) * row[f + d];
        a.dst[i] = acc;
    }
}
__global__ void __launch_bounds__(256) gk_smooth_t(const GSmoothArgs a) {
    const long long total = (long long)a.n_units * a.T * a.F;
    const long long TF = (long long)a.T * a.F;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)((i % TF) / a.F);
        double acc = 0.0;
        const int lo = max(-a.nt, -t), hi = min(a.nt, a.T - 1 - t);
        for (int e = lo; e <= hi; ++e) acc += (double)(a.nt + 1 - abs(e)) * a.src[i + (long long)e * a.F];
        double v = acc * a.inv_D;
        if (a.blend) v = v * a.p + (1.0 - a.p);
        a.dst[i] = v;
    }
}

// ---- inverse STFT: one CTA per (frame, unit) -----------------------------------------------------------------
struct GIstftArgs {
    GGeom gg;
    GTables tb;
    const double2* X;
    const double* M;
    double* frames;         // [n_units][T][W]
    int dbg_ul;
    float2* dbg_spec;       // [T][F]
    float* dbg_mask;        // [T][F]
};
__global__ void __launch_bounds__(256) gk_istft(const GIstftArgs a) {
    B200_DYN_SMEM(double2, s);
    const Geom& g = a.gg.g;
    const int N = a.gg.N, W = a.gg.W, F = a.gg.F;
    const int t = blockIdx.x, ul = blockIdx.y;
    const size_t row = ((size_t)ul * g.T + t) * F;
    // inverse real DFT as conj(DFT(conj(Y))): only the real part is kept, so the outer conjugate drops out
    const int len = gk_len(a.gg);
    if (a.gg.M) {
        for (int n = N + threadIdx.x; n < len; n += blockDim.x) s[n] = make_double2(0.0, 0.0);
    }
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        const double2 x = a.X[row + f];
        const double m = a.M[row + f];
        double2 y = make_double2(x.x * m, -x.y * m);                         // conj(X * mask)
        if (ul == a.dbg_ul) {
            a.dbg_spec[(size_t)t * F + f] = make_float2((float)x.x, (float)x.y);
            a.dbg_mask[(size_t)t * F + f] = (float)m;
        }
        if (f == 0 || 2 * f == N) y.y = 0.0;                                 // c2r ignores these imaginary parts
        s[gk_slot(a.gg, f)] = gk_in(a.gg, a.tb, f, y);
        if (f > 0 && 2 * f < N) s[gk_slot(a.gg, N - f)] = gk_in(a.gg, a.tb, N - f, make_double2(y.x, -y.y));
    }
    __syncthreads();
    gk_dft(s, a.gg, a.tb);
    double* fr = a.frames + ((size_t)ul * g.T + t) * W;
    for (int n = threadIdx.x; n < W; n += blockDim.x) fr[n] = gk_out(a.gg, a.tb, n, s[n]).x * a.tb.ws[n];   // irfft(...)[:W] * sum(w) * w
}

// ---- overlap-add + crop + cast: one thread per output sample of the chunk centre ------------------------------
template <typename T>
__device__ __forceinline__ T gk_cast(double v);
template <> __device__ __forceinline__ float gk_cast<float>(double v) { return (float)v; }
template <> __device__ __forceinline__ double gk_cast<double>(double v) { return v; }
template <> __device__ __forceinline__ short gk_cast<short>(double v) { return (short)(int)v; }    // numpy astype: truncate, wrap

template <typename T>
struct GOlaArgs {
    GGeom gg;
    GTables tb;
    const double* frames;
    T* y;
    double* adj;            // ADJ: [n_units][adj_pitch], the un-normalised overlap-add of the padded span [0, Lp)
    long long adj_pitch;
};
template <typename T, bool ADJ = false>
__global__ void __launch_bounds__(256) gk_ola(const GOlaArgs<T> a) {
    const Geom& g = a.gg.g;
    const int W = a.gg.W, H = g.H;
    const int ul = blockIdx.y;
    if (ADJ) {
        double* arow = a.adj + (size_t)ul * a.adj_pitch;
        const double* fr = a.frames + (size_t)ul * g.T * W;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < g.Lp; i += (long long)gridDim.x * blockDim.x) {
            const long long j = i + W / 2;
            long long t_lo = (j - W + H) / H;
            if (j - W + 1 <= 0) t_lo = 0;
            const long long t_hi = min((long long)(g.T - 1), j / H);
            double acc = 0.0;
            for (long long t = t_lo; t <= t_hi; ++t) acc += fr[(size_t)t * W + (int)(j - t * H)];
            arow[i] = acc;
        }
        return;
    }
    const int u = g.u0 + ul;
    const long long chunk = u / g.C, ch = u - chunk * g.C;
    const long long start = chunk * g.step;
    long long out_len = a.gg.out_len > 0 ? a.gg.out_len : min((long long)g.step, (long long)(g.n_total - start));
    if (a.gg.crop > 0) out_len = min(out_len, a.gg.crop);
    const long long sig_len = (long long)(g.T - 1) * H + (W & 1);           // istft length after the boundary crop
    T* yrow = a.y + ch * g.out_stride + start;
    const double* fr = a.frames + (size_t)ul * g.T * W;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < out_len; k += (long long)gridDim.x * blockDim.x) {
        const long long i = g.pad + k;                                       // index into the padded chunk (base.py:150)
        double v = 0.0;
        if (i < sig_len) {
            const long long j = i + W / 2;                                   // index into the un-cropped overlap-add
            long long t_lo = (j - W + H) / H;                                // ceil((j - W + 1) / H)
            if (j - W + 1 <= 0) t_lo = 0;
            const long long t_hi = min((long long)(g.T - 1), j / H);
            double acc = 0.0, nrm = 0.0;
            for (long long t = t_lo; t <= t_hi; ++t) {
                const int n = (int)(j - t * H);
                acc += fr[(size_t)t * W + n];
                nrm += a.tb.w2[n];
            }
            v = acc / (nrm > 1e-10 ? nrm : 1.0);
        }
        yrow[k] = gk_cast<T>(v);                                             // stationary.py:126 leaves the tail zero
    }
}

// ---- noise statistics: dB of the collapsed clip's STFT ------------------------------------------------------
__global__ void __launch_bounds__(256) gk_noise_db(const double2* __restrict__ X, long long n, double eps, double* __restrict__ db) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const double2 v = X[i];
        db[i] = 20.0 * log10(hypot(v.x, v.y) + eps);
    }
}


// ---- TorchGate surface (torchgate.py:127-198): per-row statistics, moving-mean follower --------------------------
struct GTStatArgs {
    int n_units, T, F, ddof;
    double eps, top_db, n_std;
    const double2* X;
    double* scratch;        // [n_units][T][F] dB scratch
    double* thr;            // [n_units][F]
};
__global__ void __launch_bounds__(128) gk_tstats(const GTStatArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)a.n_units * a.F) return;
    const int ul = (int)(i / a.F), f = (int)(i - (long long)ul * a.F);
    const double2* X = a.X + (size_t)ul * a.T * a.F + f;
    double* D = a.scratch + (size_t)ul * a.T * a.F + f;
    double mx = -1.0e300;
    for (int t = 0; t < a.T; ++t) {
        const double2 v = X[(size_t)t * a.F];
        const double db = 20.0 * log10(hypot(v.x, v.y) + a.eps);            // torchgate/utils.py:6-23
        D[(size_t)t * a.F] = db;
        mx = fmax(mx, db);
    }
    const double fl = mx - a.top_db;
    double sum = 0.0;
    for (int t = 0; t < a.T; ++t) sum += fmax(D[(size_t)t * a.F], fl);
    const double mean = sum / a.T;
    double ss = 0.0;
    for (int t = 0; t < a.T; ++t) {
        const double d = fmax(D[(size_t)t * a.F], fl) - mean;
        ss += d * d;
    }
    a.thr[(size_t)ul * a.F + f] = mean + sqrt(ss / (double)(a.T - a.ddof)) * a.n_std;   // torch.std_mean: unbiased
}

struct GMovArgs {
    int n_units, T, F, n;
    double n_thresh, inv_temp, p;
    const double2* X;
    double* M;              // mask out
    double* tmp;            // |X|
};
__global__ void __launch_bounds__(128) gk_movmean(const GMovArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)a.n_units * a.F) return;
    const int ul = (int)(i / a.F), f = (int)(i - (long long)ul * a.F);
    const size_t o = (size_t)ul * a.T * a.F + f;
    const double2* X = a.X + o;
    double* M = a.M + o;
    double* A = a.tmp + o;
    for (int t = 0; t < a.T; ++t) {
        const double2 v = X[(size_t)t * a.F];
        A[(size_t)t * a.F] = hypot(v.x, v.y);
    }
    const int left = (a.n - 1) / 2, right = a.n - 1 - left;                  // conv1d padding='same', zero padded
    for (int t = 0; t < a.T; ++t) {
        double s = 0.0;                                                      // summed in window order like the oracle's cumsum
        const int lo = max(0, t - left), hi = min(a.T - 1, t + right);
        for (int k = lo; k <= hi; ++k) s += A[(size_t)k * a.F];
        s /= (double)a.n;
        const double Av = A[(size_t)t * a.F];
        const double r = (Av - s) / s;
        const double m = 1.0 / (1.0 + exp(-(r - a.n_thresh) * a.inv_temp)); // torchgate/utils.py:39
        M[(size_t)t * a.F] = m * a.p + (1.0 - a.p);                          // torchgate.py:241 blends before smoothing
    }
}

}  // namespace b200
