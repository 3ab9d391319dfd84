// gate_kernels_2k.cuh -- n_fft = 2048 family (BASELINE.json config 3: non-stationary gate, hop 512).
//
// One real frame of 2048 samples rides in one 1024-point complex warp FFT (warp_fft.cuh) by the
// half-length trick:  z[m] = x[2m] + i x[2m+1],  Z = FFT_1024(z),
//     E[k] = (Z[k] + conj Z[1024-k]) / 2,   O[k] = (Z[k] - conj Z[1024-k]) / (2i),   W_k = exp(-i pi k / 1024)
//     X[k] = E[k] + W_k O[k],               X[1024-k] = conj(E[k] - W_k O[k]),       k = 0..512
// and back:  with P = X[k], Q = conj X[1024-k] after masking,
//     E' = (P + Q)/2,  T' = (P - Q)/2,  Z'[k] = E' + i conj(W_k) T',  Z'[1024-k] = conj(E') + i W_k conj(T').
// The mirrored element lives in lane 32-lane, slot 31-slot -- the same shuffle pattern as the 1024
// family.  A hop (512 samples) is 8 rows of 32 sample PAIRS, so the overlap-add again stays in
// registers (32 rows of even samples + 32 rows of odd samples).
#pragma once
#include "gate_kernels.cuh"

namespace b200 {

constexpr int kN2 = 2048;
constexpr int kF2 = kN2 / 2 + 1;        // 1025
constexpr int kFW2 = (kF2 + 31) / 32;   // 33
constexpr int kFPad2 = kFW2 * 32;       // 1056

struct Tables2 {
    const float2* wa2;      // [1024] analysis window pairs (w[2m], w[2m+1]) / sum(w)
    const float2* ws2;      // [1024] synthesis window pairs * sum(w) / 1024
    const float2* tw;       // [32*32] radix-32 inter-pass twiddles
    const float2* w2k;      // [1025] exp(-i pi k / 1024) as (cos, -sin)
    const float2* invn2;    // [256]  1 / overlap-add norm, pairs, interior hops
    float ws_to_w;
};

// |X| for the non-stationary follower: one MUFU.SQRT (relative error <= 2^-22) instead of the correctly rounded sqrtf
// (reciprocal square root + Newton step + slow path, ~10 instructions, 34 of them per frame).  The magnitudes only feed the
// follower's ratio and sigmoid -- a soft mask with tolerance 1e-5 -- never a binary decision.
__device__ __forceinline__ float sqrt_approx(float x) {
#if defined(B200_CUSIM_BUILD) || defined(B200_EXACT_SQRT_2K)
    return sqrtf(x);
#else
    float r;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#endif
}

// frame samples -> packed complex input of the 1024-point FFT, windowed
__device__ __forceinline__ void load_frame_2k(float (&re)[32], float (&im)[32], const float* __restrict__ xrow,
                                              long long base, long long i1, long long Lp, long long n_total,
                                              const float2* __restrict__ s_wa2, int lane) {
    const long long g0 = i1 + base;
    const float* p0 = xrow + g0;
    if (base >= 0 && base + kN2 <= Lp && g0 >= 0 && g0 + kN2 <= n_total && ((reinterpret_cast<uintptr_t>(p0) & 7) == 0)) {
        const float2* p = reinterpret_cast<const float2*>(p0) + lane;
#pragma unroll
        for (int r = 0; r < 32; ++r) {
            const float2 v = __ldg(p + 32 * r);
            const float2 w = s_wa2[lane + 32 * r];
            re[r] = v.x * w.x;
            im[r] = v.y * w.y;
        }
    } else {
#pragma unroll
        for (int r = 0; r < 32; ++r) {
            const long long j = base + 2 * (lane + 32 * r);
            const float2 w = s_wa2[lane + 32 * r];
            re[r] = chunk_sample(xrow, j, i1, Lp, n_total) * w.x;
            im[r] = chunk_sample(xrow, j + 1, i1, Lp, n_total) * w.y;
        }
    }
}

struct K1n2Args {
    Geom g;
    Tables2 tb;
    const float* x;
    float* mag;                // [n_units][T][FPad2]
    DebugTap dbg;              // spec: [T][F2][2]
    int run, n_runs;
    float2* zcache;            // [n_units][T][1024] packed half-length spectra Z of frames [z_lo, z_hi), or null
    int z_lo, z_hi;
};

__host__ __device__ constexpr int k2k_table_floats() { return 2 * 1024 + 2 * 1024 + 2 * kFPad2; }   // wa2, tw, w2k
constexpr int k1n2_smem_floats() { return k2k_table_floats() + kWarps * kExchFloats; }

__global__ void __launch_bounds__(kThreads, 3) k1n_magnitude_2k(const K1n2Args a) {
    B200_DYN_SMEM(float, smem);
    float2* s_wa2 = reinterpret_cast<float2*>(smem);
    float2* s_tw = reinterpret_cast<float2*>(smem + 2048);
    float2* s_w2k = reinterpret_cast<float2*>(smem + 4096);
    float* s_tiles = smem + k2k_table_floats();
    for (int i = threadIdx.x; i < 1024; i += kThreads) {
        s_wa2[i] = a.tb.wa2[i];
        s_tw[i] = a.tb.tw[i];
    }
    for (int i = threadIdx.x; i < kFPad2; i += kThreads) s_w2k[i] = (i < kF2) ? a.tb.w2k[i] : make_float2(0.f, 0.f);
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
        const long long i1 = (long long)ic * g.step - g.pad;
        const float* xrow = a.x + (long long)c * g.in_stride;
        const int t0 = run * a.run;
        const int t1 = min(t0 + a.run, g.T);
        for (int t = t0; t < t1; ++t) {
            const long long base = (long long)t * H - kN2 / 2;
            float re[32], im[32];
            load_frame_2k(re, im, xrow, base, i1, g.Lp, g.n_total, s_wa2, lane);
            warp_fft1024(re, im, tile, s_tw, lane);
            if (a.zcache && t >= a.z_lo && t < a.z_hi) {        // k2c_synthesize_2k loads Z instead of transforming the frame again
                float2* zp = a.zcache + ((long long)ul * g.T + t) * 1024 + lane;
#pragma unroll
                for (int q = 0; q < 32; ++q) zp[32 * q] = make_float2(re[brev5(q)], im[brev5(q)]);
            }
            float* dst = a.mag + ((long long)ul * g.T + t) * kFPad2;
#pragma unroll
            for (int q = 0; q < 17; ++q) {
                const int sA = brev5(q), sP = brev5(31 - q), s0 = brev5((32 - q) & 31);
                const float zr = re[sA], zi = im[sA];
                float pr = __shfl_sync(0xffffffffu, re[sP], pl);
                float pi = __shfl_sync(0xffffffffu, im[sP], pl);
                if (lane == 0) { pr = re[s0]; pi = im[s0]; }
                const int k = lane + 32 * q;
                const bool valid = (q < 16) || (lane == 0);
                const float Er = 0.5f * (zr + pr), Ei = 0.5f * (zi - pi);
                const float Or = 0.5f * (zi + pi), Oi = 0.5f * (pr - zr);
                const float2 W = s_w2k[k];
                const float Tr = fmaf(-Oi, W.y, Or * W.x), Ti = fmaf(Or, W.y, Oi * W.x);
                const float Xr = Er + Tr, Xi = Ei + Ti;              // X[k]
                const float Yr = Er - Tr, Yi = Ti - Ei;              // X[1024-k] = conj(E - T)
                if (valid) {
                    dst[k] = sqrt_approx(fmaf(Xr, Xr, Xi * Xi));
                    if (k != 512) dst[1024 - k] = sqrt_approx(fmaf(Yr, Yr, Yi * Yi));
                    if (a.dbg.ul == ul) {
                        float* sp = a.dbg.spec + ((long long)t * kF2) * 2;
                        sp[2 * k] = Xr; sp[2 * k + 1] = Xi;
                        sp[2 * (1024 - k)] = Yr; sp[2 * (1024 - k) + 1] = Yi;
                    }
                }
            }
        }
    }
}

struct K22Args {
    Geom g;
    Tables2 tb;
    const float* x;
    float* y;
    const float* fmask;        // [n_units][T][FPad2] final multiplicative masks
    int run, n_runs;           // output hops per work item
    DebugTap dbg;              // mask: [T][F2]
    // k2_synthesize_2k<true>: the adjoint of a unit (b200gate_adjoint), as k2_synthesize<.., ADJ>: x is the gradient g,
    // read on the unit's centre only and divided by the overlap-add norm; the un-normalised overlap-add of the padded
    // span goes to adj[ul][0, Lp)
    float* adj;
    long long adj_pitch;
};

// 1 / (sum of w^2 over the frames overlapping sample `ro` of hop `hop`), as k2_synthesize_2k's edge hops compute it
__device__ B200_NOINLINE float inv_norm_2k(int hop, int ro, int H, int T, const float2* __restrict__ s_ws2,
                                             float ws_to_w) {
    float nrm = 0.f;
    for (int i = 0; i < 4; ++i) {
        const int tf = hop - i;
        if (tf >= 0 && tf <= T - 1) {
            const int n = i * H + ro;
            const float2 wp = s_ws2[n >> 1];
            const float w = ((n & 1) ? wp.y : wp.x) * ws_to_w;
            nrm = fmaf(w, w, nrm);
        }
    }
    return nrm > 1e-10f ? 1.0f / nrm : 1.0f;
}

// the adjoint's input frame t: g / norm on the centre [pad, jp_hi), zero elsewhere, windowed (pairs as load_frame_2k).
// Sample 2 (lane + 32 r) + par of the frame is sample (r % 8) * 64 + 2 lane + par of hop t + r / 8.
__device__ __forceinline__ void load_adjoint_2k(float (&re)[32], float (&im)[32], const float* __restrict__ grow, int t,
                                                long long base, long long i1, long long pad, long long jp_hi, int H, int T,
                                                const float2* __restrict__ s_invn2, const float2* __restrict__ s_ws2,
                                                float ws_to_w, const float2* __restrict__ s_wa2, int lane) {
    const bool interior = t >= 3 && t + 3 <= T - 1;          // every hop of the frame has the interior norm
#pragma unroll
    for (int r = 0; r < 32; ++r) {
        const long long j = base + 2 * (lane + 32 * r);
        const float2 w = s_wa2[lane + 32 * r];
        float2 inv;
        if (interior) {
            inv = s_invn2[(r & 7) * 32 + lane];
        } else {
            const int ro = (r & 7) * 64 + 2 * lane;
            inv = make_float2(inv_norm_2k(t + (r >> 3), ro, H, T, s_ws2, ws_to_w),
                              inv_norm_2k(t + (r >> 3), ro + 1, H, T, s_ws2, ws_to_w));
        }
        re[r] = (j >= pad && j < jp_hi) ? __ldg(grow + i1 + j) * inv.x * w.x : 0.0f;
        im[r] = (j + 1 >= pad && j + 1 < jp_hi) ? __ldg(grow + i1 + j + 1) * inv.y * w.y : 0.0f;
    }
}

constexpr int k22_smem_floats() { return k2k_table_floats() + 2 * 1024 + 2 * 256 + kWarps * kExchFloats; }

template <bool ADJ = false>
__global__ void __launch_bounds__(kThreads, 2) k2_synthesize_2k(const K22Args a) {
    constexpr int HR = 8, NH = 4;
    B200_DYN_SMEM(float, smem);
    float2* s_wa2 = reinterpret_cast<float2*>(smem);
    float2* s_tw = reinterpret_cast<float2*>(smem + 2048);
    float2* s_w2k = reinterpret_cast<float2*>(smem + 4096);
    float2* s_ws2 = reinterpret_cast<float2*>(smem + k2k_table_floats());
    float2* s_invn2 = s_ws2 + 1024;
    float* s_tiles = smem + k2k_table_floats() + 2 * 1024 + 2 * 256;
    for (int i = threadIdx.x; i < 1024; i += kThreads) {
        s_wa2[i] = a.tb.wa2[i];
        s_tw[i] = a.tb.tw[i];
        s_ws2[i] = a.tb.ws2[i];
    }
    for (int i = threadIdx.x; i < kFPad2; i += kThreads) s_w2k[i] = (i < kF2) ? a.tb.w2k[i] : make_float2(0.f, 0.f);
    for (int i = threadIdx.x; i < 256; i += kThreads) s_invn2[i] = a.tb.invn2[i];
    __syncthreads();

    const Geom& g = a.g;
    const int H = g.H;                                   // 512
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* tile = s_tiles + warp * kExchFloats;
    const int pl = (32 - lane) & 31;
    const long long n_items = (long long)g.n_units * a.n_runs;

    for (long long item = (long long)blockIdx.x * kWarps + warp; item < n_items;
         item += (long long)gridDim.x * kWarps) {
        const int ul = (int)(item / a.n_runs);
        const int run = (int)(item - (long long)ul * a.n_runs);
        const int u = g.u0 + ul;
        const int ic = u / g.C, c = u - ic * g.C;
        const long long i1 = (long long)ic * g.step - g.pad;
        long long out_len = g.n_total - (long long)ic * g.step;
        if (out_len > g.step) out_len = g.step;
        long long jp_hi = g.pad + out_len;
        const long long sig_len = (long long)(g.T - 1) * H;
        if (jp_hi > sig_len) jp_hi = sig_len;
        if (jp_hi <= g.pad) continue;
        const long long jlo = g.pad + kN2 / 2, jhi = jp_hi + kN2 / 2;
        const int h_lo = (int)(jlo / H), h_hi = (int)((jhi + H - 1) / H);
        // the adjoint runs the frames [f_lo, f_hi] that touch the centre and writes every hop they overlap
        const int f_lo = ADJ ? max(0, h_lo - (NH - 1)) : 0, f_hi = ADJ ? min(h_hi - 1, g.T - 1) : g.T - 1;
        const int hs = (ADJ ? f_lo : h_lo) + run * a.run;
        const int he = min(hs + a.run, ADJ ? f_hi + NH : h_hi);
        if (hs >= he) continue;
        const int t_start = max(f_lo, hs - (NH - 1));
        const int t_last = min(he - 1, f_hi);
        const float* xrow = a.x + (long long)c * g.in_stride;
        float* yrow = a.y + (long long)c * g.out_stride;
        const float* frow = a.fmask + (long long)ul * g.T * kFPad2;

        float acc_e[32], acc_o[32];                      // even / odd samples of the overlap-add window
#pragma unroll
        for (int r = 0; r < 32; ++r) { acc_e[r] = 0.f; acc_o[r] = 0.f; }

        for (int t = t_start; t < he; ++t) {
            if (t <= t_last) {
                const long long base = (long long)t * H - kN2 / 2;
                float re[32], im[32];
                if (ADJ) load_adjoint_2k(re, im, xrow, t, base, i1, g.pad, jp_hi, H, g.T, s_invn2, s_ws2, a.tb.ws_to_w,
                                         s_wa2, lane);
                else load_frame_2k(re, im, xrow, base, i1, g.Lp, g.n_total, s_wa2, lane);
                const float* mrow = frow + (long long)t * kFPad2;
                if (a.dbg.ul == ul) {
#pragma unroll 1
                    for (int k = lane; k < kF2; k += 32) a.dbg.mask[(long long)t * kF2 + k] = mrow[k];
                }
#pragma unroll 1
                for (int ph = 0; ph < 2; ++ph) {
                    warp_fft1024(re, im, tile, s_tw, lane);
                    if (ph == 0) {
#pragma unroll
                        for (int q = 0; q < 17; ++q) {
                            const int sA = brev5(q), sP = brev5(31 - q), s0 = brev5((32 - q) & 31);
                            const int k = lane + 32 * q;                       // <= 543 < FPad2
                            const float zr = re[sA], zi = im[sA];
                            float pr, pi;
                            if (q < 16) {
                                pr = __shfl_sync(0xffffffffu, re[sP], pl);
                                pi = __shfl_sync(0xffffffffu, im[sP], pl);
                                if (lane == 0) { pr = re[s0]; pi = im[s0]; }
                            } else {
                                pr = zr; pi = zi;                              // only lane 0 (k = 512) matters
                            }
                            const float m = mrow[k];
                            const float mp = mrow[(1024 - k) & 2047];          // k' = 1024-k (>= 481 for q = 16 lanes)
                            const float Er = 0.5f * (zr + pr), Ei = 0.5f * (zi - pi);
                            const float Or = 0.5f * (zi + pi), Oi = 0.5f * (pr - zr);
                            const float2 W = s_w2k[k];
                            const float Tr = fmaf(-Oi, W.y, Or * W.x), Ti = fmaf(Or, W.y, Oi * W.x);
                            // P = X[k] = E + T,  Q = conj X[1024-k] = E - T;  masks applied to X[k], X[1024-k]
                            const float Pr = m * (Er + Tr), Pi = m * (Ei + Ti);
                            const float Qr = mp * (Er - Tr), Qi = mp * (Ei - Ti);
                            const float Epr = 0.5f * (Pr + Qr), Epi = 0.5f * (Pi + Qi);
                            const float Tpr = 0.5f * (Pr - Qr), Tpi = 0.5f * (Pi - Qi);
                            // V = conj(W) T'   (W = (W.x, W.y) with W.y = -sin)
                            const float Vr = fmaf(Tpi, W.y, Tpr * W.x), Vi = fmaf(-Tpr, W.y, Tpi * W.x);
                            const float own_r = Epr - Vi, own_i = Epi + Vr;    // Z'[k]      = E' + i V
                            const float oth_r = Epr + Vi, oth_i = Vr - Epi;    // Z'[1024-k] = conj(E') + i conj(V)
                            if (q < 16) {
                                const float nr = __shfl_sync(0xffffffffu, oth_r, pl);
                                const float ni = __shfl_sync(0xffffffffu, oth_i, pl);
                                re[sA] = own_r;
                                im[sA] = own_i;
                                if (lane != 0) { re[sP] = nr; im[sP] = ni; }
                                else if (q != 0) { re[s0] = oth_r; im[s0] = oth_i; }
                            } else if (lane == 0) {
                                re[sA] = own_r;
                                im[sA] = own_i;
                            }
                        }
                        // brev slots -> natural slots with re <-> im exchanged, in place
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
                // now im = 1024 * y[2m], re = 1024 * y[2m+1]  (m = lane + 32 q) at slot brev5(q)
#pragma unroll
                for (int q = 0; q < 32; ++q) {
                    const float2 w = s_ws2[lane + 32 * q];
                    acc_e[q] = fmaf(im[brev5(q)], w.x, acc_e[q]);
                    acc_o[q] = fmaf(re[brev5(q)], w.y, acc_o[q]);
                }
            }
            // hop t is complete: rows 0..7 (pairs) = samples [t*512, (t+1)*512)
            if (ADJ) {                                       // un-normalised, the whole padded span
                if (t >= hs) {
                    float* arow = a.adj + (long long)ul * a.adj_pitch;
                    const long long jp0 = (long long)t * H - kN2 / 2;
#pragma unroll
                    for (int r = 0; r < HR; ++r) {
                        const long long jp = jp0 + 64 * r + 2 * lane;
                        if (jp >= 0 && jp < g.Lp) arow[jp] = acc_e[r];
                        if (jp + 1 >= 0 && jp + 1 < g.Lp) arow[jp + 1] = acc_o[r];
                    }
                }
            } else if (t >= hs) {
                const long long jp0 = (long long)t * H - kN2 / 2;          // chunk-local index of row 0, pair 0
                float* d0 = yrow + i1 + jp0 + 2 * lane;
                if (t >= NH - 1 && t <= g.T - 1 && jp0 >= g.pad && jp0 + H <= jp_hi &&
                    ((reinterpret_cast<uintptr_t>(d0) & 7) == 0)) {
#pragma unroll
                    for (int r = 0; r < HR; ++r) {
                        const float2 inv = s_invn2[r * 32 + lane];
                        *reinterpret_cast<float2*>(d0 + 64 * r) = make_float2(acc_e[r] * inv.x, acc_o[r] * inv.y);
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < HR; ++r) {
#pragma unroll
                        for (int par = 0; par < 2; ++par) {
                            const int ro = r * 64 + 2 * lane + par;         // sample offset within the hop
                            const long long jp = jp0 + ro;
                            if (jp < g.pad || jp >= jp_hi) continue;
                            float nrm = 0.f;
                            for (int i = 0; i < NH; ++i) {
                                const int tf = t - i;
                                if (tf >= 0 && tf <= g.T - 1) {
                                    const int n = i * H + ro;               // window index of this sample in frame tf
                                    const float2 wp = s_ws2[n >> 1];
                                    const float w = ((n & 1) ? wp.y : wp.x) * a.tb.ws_to_w;
                                    nrm = fmaf(w, w, nrm);
                                }
                            }
                            const float inv = nrm > 1e-10f ? 1.0f / nrm : 1.0f;
                            yrow[i1 + jp] = (par ? acc_o[r] : acc_e[r]) * inv;
                        }
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < 32 - HR; ++r) { acc_e[r] = acc_e[r + HR]; acc_o[r] = acc_o[r + HR]; }
#pragma unroll
            for (int r = 32 - HR; r < 32; ++r) { acc_e[r] = 0.f; acc_o[r] = 0.f; }
        }
    }
}

}  // namespace b200
