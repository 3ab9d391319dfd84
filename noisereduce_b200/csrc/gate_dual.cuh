// gate_dual.cuh -- the stationary gate's two FFT kernels in DUAL form: one warp carries two (chunk, channel) units
// -- channels c and c+1 of the same chunk -- through every step, unit A in the low half and unit B in the high half
// of each 64-bit register pair (warp_fft.cuh, "Dual transform").  Both units share the control flow exactly (same
// chunk geometry, same frame indices, same edge cases), so the whole butterfly network, the inter-pass twiddles,
// the window, the mask apply and the overlap-add run on FP32 pairs and every shared-memory access moves 8 or 16
// bytes per lane.  sm_90 has no packed FP32 instructions, so the pairs cost two scalar instructions each and these
// kernels (more registers, fewer warps per SM) are slower than the single-unit ones: they run on request only
// (path_flags bit 4).
//
// Reference semantics are those of gate_kernels.cuh / gate_synth.cuh (paths relative to the reference checkout):
//   k1d_analyze     scipy.signal.stft as called at noisereduce/spectralgate/stationary.py:87-93, _amp_to_db +
//                   threshold compare (spectralgate/utils.py:11-16, stationary.py:96-110) in the linear power domain
//                   with the float64 re-decision of guard-band bins
//   k2d_synthesize  X * mask (stationary.py:117), scipy.signal.istft (stationary.py:120-126), chunk centre (base.py:150)
//
// Spectrum cache (dual layout): zd[dual][pair][k] = float4 (Re Z_A, Re Z_B, Im Z_A, Im Z_B)[k], Z = X_a + i X_b the
// packed spectrum of frames (2j, 2j+1); 16 KB per dual pair, written by k1d and bulk-copied (TMA) by k2d.
#pragma once
#include "gate_synth.cuh"

namespace b200 {

#ifndef B200_K2D_WARPS
#define B200_K2D_WARPS 7
#endif
constexpr int kDualWarpsK2 = B200_K2D_WARPS;                 // one CTA per SM; 7 x (16 KB spectrum + masks + exchange tile) + tables = 226 KB
#ifndef B200_K1D_WARPS
#define B200_K1D_WARPS 8
#endif
constexpr int kDualWarpsK1 = B200_K1D_WARPS;

// 64-bit / 128-bit shared and global accesses on FP32 pairs
struct __align__(16) f2x2 { f2 a, b; };

__device__ __forceinline__ f2 f2_dup(float c) { return f2_pack(c, c); }
__device__ __forceinline__ float f2_lo(f2 v) { float a, b; f2_unpack(v, a, b); return a; }
__device__ __forceinline__ float f2_hi(f2 v) { float a, b; f2_unpack(v, a, b); return b; }

// =============================================================================================
// k2d: synthesis of two units per warp from the dual spectrum cache.
// =============================================================================================
struct K2dArgs {
    Geom g;                        // n_units even, u0 even, C even: duals are (2d, 2d+1)
    Tables tb;
    void* y;                       // [C][out_stride], caller dtype
    const unsigned short* num;     // [n_units][ceil(T/2)][FPad][2] mask numerators (num_index layout)
    const float4* zd;              // [n_units/2][zpairs][1024]
    int zpairs;
    float pD, one_minus_p;
    int nt;
    int run, n_runs;
    DebugTap dbg;
};

constexpr int kK2dTableBytes = kN * 4 + kN * 8 + kFPad * 4;                  // synthesis window, twiddles, frequency edge factors
constexpr int kK2dWarpBytes = kN * 16 + 2 * (2 * kFPad * 2) + kExchDual * 8 + 16;   // spectrum, 2 mask rows, tile, mbarrier
constexpr int k2d_smem_bytes() { return kK2dTableBytes + kDualWarpsK2 * kK2dWarpBytes; }
static_assert(kExchDual * 8 >= 513 * 16, "mirror buffer must fit the dual exchange tile");

template <int HR, bool BLEND, typename T>
__global__ void __launch_bounds__(kDualWarpsK2 * 32, 1) k2d_synthesize(const K2dArgs a) {
    constexpr int NH = 32 / HR;
    constexpr int MB = 2 * kFPad * 2;          // one unit's mask row pair (2176 bytes)
    B200_DYN_SMEM(unsigned char, smraw);
    const Geom& g = a.g;
    const int H = g.H;
    float* s_ws = reinterpret_cast<float*>(smraw);
    float2* s_tw = reinterpret_cast<float2*>(smraw + kN * 4);
    float* s_ef = reinterpret_cast<float*>(smraw + kN * 12);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* wbase = smraw + kK2dTableBytes + warp * kK2dWarpBytes;
    const f2x2* zbuf = reinterpret_cast<const f2x2*>(wbase);                 // [1024] (re pair, im pair)
    const unsigned* mA32 = reinterpret_cast<const unsigned*>(wbase + kN * 16);
    const unsigned* mB32 = reinterpret_cast<const unsigned*>(wbase + kN * 16 + MB);
    f2* tile = reinterpret_cast<f2*>(wbase + kN * 16 + 2 * MB);
    f2x2* qbuf = reinterpret_cast<f2x2*>(tile);
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(wbase + kN * 16 + 2 * MB + kExchDual * 8);
    const int nthr = kDualWarpsK2 * 32;
    for (int i = threadIdx.x; i < kN; i += nthr) {
        s_ws[i] = a.tb.ws[i];
        s_tw[i] = a.tb.tw[i];
    }
    for (int i = threadIdx.x; i < kFPad; i += nthr) s_ef[i] = a.tb.ef[i];
    if (lane == 0) mbar_init(bar, 1);
    mbar_init_fence();
    __syncthreads();
    unsigned phase = 0;

    float invn[HR];                          // interior overlap-add norm of this lane's HR rows of a hop
#pragma unroll
    for (int r = 0; r < HR; ++r) invn[r] = a.tb.invn[r * 32 + lane];

    const int n_duals = g.n_units >> 1;
    const long long n_items = (long long)n_duals * a.n_runs;
    for (long long item = (long long)blockIdx.x * kDualWarpsK2 + warp; item < n_items;
         item += (long long)gridDim.x * kDualWarpsK2) {
        const int dl = (int)(item / a.n_runs);
        const int run = (int)(item - (long long)dl * a.n_runs);
        const int ulA = 2 * dl;
        const int u = g.u0 + ulA;
        const int ic = u / g.C, c = u - ic * g.C;                    // unit B is channel c + 1 of the same chunk
        const long long i1 = (long long)ic * g.step - g.pad;
        long long out_len = g.n_total - (long long)ic * g.step;
        if (out_len > g.step) out_len = g.step;
        long long jp_hi = g.pad + out_len;
        const long long sig_len = (long long)(g.T - 1) * H;
        if (jp_hi > sig_len) jp_hi = sig_len;
        if (jp_hi <= g.pad) continue;
        const long long jlo = g.pad + kN / 2, jhi = jp_hi + kN / 2;
        const int h_lo = (int)(jlo / H), h_hi = (int)((jhi + H - 1) / H);
        const int hs = h_lo + run * a.run;
        const int he = min(hs + a.run, h_hi);
        if (hs >= he) continue;
        const int t_start = max(0, hs - (NH - 1)) & ~1;
        const int t_last = min(he - 1, g.T - 1);
        T* yA = static_cast<T*>(a.y) + (long long)c * g.out_stride;
        T* yB = yA + g.out_stride;
        const float4* zunit = a.zd + (long long)dl * a.zpairs * 1024;
        const unsigned short* muA = a.num + (long long)ulA * a.zpairs * (2 * kFPad);
        const unsigned short* muB = muA + (long long)a.zpairs * (2 * kFPad);

        // overlap-add state: rows 0..23 = the partial sums of the next three hops (8 register rows each)
        f2 P[32 - HR];
#pragma unroll
        for (int r = 0; r < 32 - HR; ++r) P[r] = f2_dup(0.f);

        auto stage = [&](int tt) {               // all lanes have finished reading the buffers
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) {
                mbar_expect_tx(bar, (unsigned)(kN * 16 + 2 * MB));
                bulk_g2s(wbase, zunit + (long long)(tt >> 1) * 1024, kN * 16, bar);
                bulk_g2s(wbase + kN * 16, muA + (long long)(tt >> 1) * (2 * kFPad), MB, bar);
                bulk_g2s(wbase + kN * 16 + MB, muB + (long long)(tt >> 1) * (2 * kFPad), MB, bar);
            }
        };
        if (t_start <= t_last) stage(t_start);

        for (int t = t_start; t < he; t += 2) {
            const bool va = (t <= t_last), vb = (t + 1 <= t_last);
            f2 out[2 * HR];                             // the two hops this iteration completes
            if (va) {
                f2 re[32], im[32];                      // what the FFT call sees: re = Im Z', im = Re Z'
                mbar_wait(bar, phase);
                phase ^= 1u;
                const float pa = 0.5f * a.pD;
                const f2 pa2 = f2_dup(pa), pb2 = f2_dup(vb ? pa : 0.f);
                const f2 ca2 = f2_dup(-8388608.0f * pa), cb2 = f2_dup(vb ? -8388608.0f * pa : 0.f);
                float eta = 0.f, etb = 0.f;
                if (BLEND) {
                    eta = 0.5f * a.one_minus_p * time_edge(t, g.T, a.nt);
                    etb = vb ? 0.5f * a.one_minus_p * time_edge(t + 1, g.T, a.nt) : 0.f;
                }
                // halved masks (m_a / 2, m_b / 2) of bin kk for (unit A, unit B)
                auto half_masks = [&](int kk, f2& ma, f2& mb) {
                    const unsigned pkA = mA32[kk], pkB = mB32[kk];
                    const f2 fa = f2_pack(__uint_as_float(prmt(pkA, 0x4B00u, 0x5410u)), __uint_as_float(prmt(pkB, 0x4B00u, 0x5410u)));
                    const f2 fb = f2_pack(__uint_as_float(prmt(pkA, 0x4B00u, 0x5432u)), __uint_as_float(prmt(pkB, 0x4B00u, 0x5432u)));
                    if (BLEND) {
                        const float e = s_ef[kk];
                        ma = f2_fma(f2_sub(fa, f2_dup(8388608.0f)), pa2, f2_dup(eta * e));
                        mb = f2_fma(f2_sub(fb, f2_dup(8388608.0f)), pb2, f2_dup(etb * e));
                    } else {
                        ma = f2_fma(fa, pa2, ca2);
                        mb = f2_fma(fb, pb2, cb2);
                    }
                };
                if (a.dbg.ul == ulA || a.dbg.ul == ulA + 1) {      // parity tap (tests): the masks this pair applies
                    const bool hi = a.dbg.ul == ulA + 1;
#pragma unroll 1
                    for (int k = lane; k < kF; k += 32) {
                        f2 ma, mb;
                        half_masks(k, ma, mb);
                        a.dbg.mask[(long long)t * kF + k] = 2.0f * (hi ? f2_hi(ma) : f2_lo(ma));
                        if (vb) a.dbg.mask[(long long)(t + 1) * kF + k] = 2.0f * (hi ? f2_hi(mb) : f2_lo(mb));
                    }
                }
                // ---- lower pairs k = lane + 32 q < 512: both members ----------------------------------
#pragma unroll
                for (int q = 0; q < 16; ++q) {
                    const int k = 32 * q + lane;
                    const f2x2 own = zbuf[k];
                    const f2x2 par = zbuf[q == 0 ? ((kN - lane) & (kN - 1)) : (kN - k)];
                    f2 ma, mb;
                    half_masks(k, ma, mb);
                    const f2 s = f2_add(ma, mb), d = f2_sub(ma, mb), nd = f2_sub(mb, ma);
                    // Z'[k] = s Z[k] + d conj(Z[N-k]);  Z'[N-k] = s Z[N-k] + d conj(Z[k])
                    im[q] = f2_fma(d, par.a, f2_mul(s, own.a));
                    re[q] = f2_fma(nd, par.b, f2_mul(s, own.b));
                    f2x2 qv;
                    qv.a = f2_fma(nd, own.b, f2_mul(s, par.b));           // Im Z'[N-k]  (the FFT's "re")
                    qv.b = f2_fma(d, own.a, f2_mul(s, par.a));            // Re Z'[N-k]  (the FFT's "im")
                    qbuf[512 - k] = qv;
                }
                {   // slot 16: bins 512 + lane directly (lane 0 = the self-mirrored bin N/2)
                    const f2x2 own = zbuf[512 + lane];
                    const f2x2 par = zbuf[512 - lane];
                    f2 ma, mb;
                    half_masks(512 - lane, ma, mb);
                    const f2 s = f2_add(ma, mb), d = f2_sub(ma, mb), nd = f2_sub(mb, ma);
                    im[16] = f2_fma(d, par.a, f2_mul(s, own.a));
                    re[16] = f2_fma(nd, par.b, f2_mul(s, own.b));
                }
                __syncwarp();
#pragma unroll
                for (int q = 17; q < 32; ++q) {
                    const f2x2 v = qbuf[32 * (q - 16) + lane];
                    re[q] = v.a;
                    im[q] = v.b;
                }
                __syncwarp();
                if (t + 2 <= t_last) stage(t + 2);
                warp_fft1024_dual(re, im, tile, s_tw, lane);
                // now im = N a'[n], re = N b'[n] (n = lane + 32 q) at slot brev5(q), for both units.  Overlap-add written so
                // that every sum is born in the register it lives in next (no register-to-register shifts): rows
                // 0..15 complete hops t, t+1; rows 16..39 become the new state.
                float w[32];
#pragma unroll
                for (int q = 0; q < 32; ++q) w[q] = s_ws[lane + 32 * q];
#pragma unroll
                for (int r = 0; r < HR; ++r) out[r] = f2_fma_s(im[brev5(r)], w[r], P[r]);
                // (summation order as k2c_synthesize's accumulate-then-shift loop: frame b's row before frame a's)
#pragma unroll
                for (int r = 0; r < HR; ++r)
                    out[HR + r] = f2_fma_s(im[brev5(HR + r)], w[HR + r], f2_fma_s(re[brev5(r)], w[r], P[HR + r]));
#pragma unroll
                for (int r = 0; r < HR; ++r)
                    P[r] = f2_fma_s(im[brev5(2 * HR + r)], w[2 * HR + r], f2_fma_s(re[brev5(HR + r)], w[HR + r], P[2 * HR + r]));
#pragma unroll
                for (int r = 0; r < HR; ++r)
                    P[HR + r] = f2_fma_s(im[brev5(3 * HR + r)], w[3 * HR + r], f2_mul_s(re[brev5(2 * HR + r)], w[2 * HR + r]));
#pragma unroll
                for (int r = 0; r < HR; ++r) P[2 * HR + r] = f2_mul_s(re[brev5(3 * HR + r)], w[3 * HR + r]);
            } else {                                    // past the last frame: flush the state
#pragma unroll
                for (int r = 0; r < 2 * HR; ++r) out[r] = P[r];
#pragma unroll
                for (int r = 0; r < HR; ++r) P[r] = P[2 * HR + r];
#pragma unroll
                for (int r = HR; r < 3 * HR; ++r) P[r] = f2_dup(0.f);
            }
            // hops t and t+1 are now complete
            {
                const long long jp0 = (long long)t * H - kN / 2;
                if (t >= hs && t + 1 < he && t >= NH - 1 && t + 1 <= g.T - 1 && jp0 >= g.pad &&
                    jp0 + 2 * H <= jp_hi) {
                    T* dA = yA + i1 + jp0 + lane;
                    T* dB = yB + i1 + jp0 + lane;
#pragma unroll
                    for (int r = 0; r < 2 * HR; ++r) {
                        const f2 v = f2_mul_s(out[r], invn[r % HR]);
                        dA[32 * r] = st_cast<T>(f2_lo(v));
                        dB[32 * r] = st_cast<T>(f2_hi(v));
                    }
                } else {
#pragma unroll 1
                    for (int r = 0; r < 2 * HR; ++r) {
                        f2 v2 = f2_dup(0.f);
#pragma unroll
                        for (int rr = 0; rr < 2 * HR; ++rr)
                            if (rr == r) v2 = out[rr];
                        const int hop = t + r / HR;
                        if (hop < hs || hop >= he) continue;
                        const int ro = (r % HR) * 32 + lane;
                        const long long jp = (long long)hop * H + ro - kN / 2;
                        if (jp < g.pad || jp >= jp_hi) continue;
                        float inv;
                        if (hop >= NH - 1 && hop <= g.T - 1) {
                            inv = a.tb.invn[ro];
                        } else {
                            float nrm = 0.f;
                            for (int i = 0; i < NH; ++i) {
                                const int tf = hop - i;
                                if (tf >= 0 && tf <= g.T - 1) {
                                    const float ww = a.tb.ws[i * H + ro] * a.tb.ws_to_w;
                                    nrm = fmaf(ww, ww, nrm);
                                }
                            }
                            inv = nrm > 1e-10f ? 1.0f / nrm : 1.0f;
                        }
                        yA[i1 + jp] = st_cast<T>(f2_lo(v2) * inv);
                        yB[i1 + jp] = st_cast<T>(f2_hi(v2) * inv);
                    }
                }
            }
        }
    }
}

// =============================================================================================
// k1d: analysis of two units per warp.  bits[(ul*T + t)*FW + w] as k1_analyze; spectra to the dual cache.
// The top_db row floor (spectralgate/utils.py:16) is not tracked per bin here: |X_t[f]|^2 <= N * sum (w x)^2 bounds
// every bin of a frame by its energy, and only if that bound reaches the smallest floor of any bin is `need_rowmax`
// raised -- the host then lets the single-unit kernel (which keeps the running maxima) redo the batch.
// =============================================================================================
struct K1dArgs {
    Geom g;                    // n_units even, u0 even, C even
    Tables tb;
    const void* x;
    unsigned* bits;            // [n_units][T][FW]
    float4* zd;                // [n_units/2][zpairs][1024]
    int zpairs, z_lo, z_hi;
    Counters* cnt;
    unsigned* need_rowmax;     // device flag
    float min_floor4;          // min over bins of 4 * (10^((thresh + top_db)/20) - eps)^2
    float wa_max;              // max of the scaled analysis window
    DebugTap dbg;
    int run, n_runs;
};

constexpr int kK1dTableBytes = kN * 4 + kN * 8 + 2 * kFPad * 4;
constexpr int kK1dWarpBytes = kN * 16 + kExchDual * 8 + 4 * kFW * 4 + 16;     // dual spectrum, exchange tile, guard-band words
constexpr int k1d_smem_bytes() { return kK1dTableBytes + kDualWarpsK1 * kK1dWarpBytes; }

template <int HR, typename T>
__global__ void __launch_bounds__(kDualWarpsK1 * 32, 1) k1d_analyze(const K1dArgs a) {
    B200_DYN_SMEM(unsigned char, smraw);
    float* s_wa = reinterpret_cast<float*>(smraw);
    float2* s_tw = reinterpret_cast<float2*>(smraw + kN * 4);
    float* s_thr4 = reinterpret_cast<float*>(smraw + kN * 12);
    float* s_gco = s_thr4 + kFPad;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* wbase = smraw + kK1dTableBytes + warp * kK1dWarpBytes;
    f2x2* zs = reinterpret_cast<f2x2*>(wbase);                                    // [1024] the pair's dual spectrum
    f2* tile = reinterpret_cast<f2*>(wbase + kN * 16);
    unsigned* s_amb = reinterpret_cast<unsigned*>(wbase + kN * 16 + kExchDual * 8);      // [4][FW]
    const int nthr = kDualWarpsK1 * 32;
    for (int i = threadIdx.x; i < kN; i += nthr) {
        s_wa[i] = a.tb.wa[i];
        s_tw[i] = a.tb.tw[i];
    }
    for (int i = threadIdx.x; i < kFPad; i += nthr) {
        s_thr4[i] = a.tb.thr4[i];
        s_gco[i] = a.tb.gco[i];
    }
    __syncthreads();

    const Geom& g = a.g;
    const int H = g.H;
    const int n_duals = g.n_units >> 1;
    const long long n_items = (long long)n_duals * a.n_runs;

    for (long long item = (long long)blockIdx.x * kDualWarpsK1 + warp; item < n_items;
         item += (long long)gridDim.x * kDualWarpsK1) {
        const int dl = (int)(item / a.n_runs);
        const int run = (int)(item - (long long)dl * a.n_runs);
        const int ulA = 2 * dl;
        const int u = g.u0 + ulA;
        const int ic = u / g.C, c = u - ic * g.C;
        const long long i1 = (long long)ic * g.step - g.pad;
        const T* xrowA = static_cast<const T*>(a.x) + (long long)c * g.in_stride;
        const T* xrowB = xrowA + g.in_stride;
        const int t0 = run * a.run;
        const int t1 = min(t0 + a.run, g.T);
        float emax = 0.f;                                   // largest frame-energy bound of this run (row floor test)

        for (int t = t0; t < t1; t += 2) {
            const bool vb = (t + 1 < t1);
            const long long base = (long long)t * H - kN / 2;
            float S_A, S_B;
            {
                f2 re[32], im[32];
                {
                    f2 xr[32 + HR];
                    if (pair_window_interior<HR>(base, i1, g.Lp, g.n_total)) {
                        const T* pA = xrowA + i1 + base + lane;
                        const T* pB = xrowB + i1 + base + lane;
#pragma unroll
                        for (int r = 0; r < 32 + HR; ++r) xr[r] = f2_pack(ld_sample(pA + 32 * r), ld_sample(pB + 32 * r));
                    } else {                                   // chunk / recording edges: zero-extended samples
#pragma unroll
                        for (int r = 0; r < 32 + HR; ++r)
                            xr[r] = f2_pack(chunk_sample(xrowA, base + lane + 32 * r, i1, g.Lp, g.n_total),
                                            chunk_sample(xrowB, base + lane + 32 * r, i1, g.Lp, g.n_total));
                    }
                    f2 e2 = f2_dup(0.f);
#pragma unroll
                    for (int r = 0; r < 32 + HR; ++r) e2 = f2_fma(xr[r], xr[r], e2);
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) e2 = f2_add(e2, f2_shfl_xor(e2, o));
                    // every frame's windowed energy <= wa_max^2 * (energy of the pair's 40 rows): S bounds ||frame pair||_2
                    const float eA = f2_lo(e2) * a.wa_max * a.wa_max, eB = f2_hi(e2) * a.wa_max * a.wa_max;
                    S_A = sqrtf(2.0f * eA);
                    S_B = sqrtf(2.0f * eB);
                    emax = fmaxf(emax, fmaxf(eA, eB));
#pragma unroll
                    for (int r = 0; r < 32; ++r) {
                        const float w = s_wa[lane + 32 * r];
                        re[r] = f2_mul_s(xr[r], w);
                        im[r] = f2_mul_s(xr[r + HR], vb ? w : 0.f);      // odd frame count: the pair's second frame does not exist
                    }
                }
                warp_fft1024_dual(re, im, tile, s_tw, lane);
                // the spectrum goes to shared memory once: the decisions below read bins and their mirrors from there by flat
                // index (no shuffles, no lane-0 special case), and ONE bulk copy (TMA store) takes it to the dual cache
                bulk_wait_read_all();                         // (the previous pair's store has read zs)
                __syncwarp();
#pragma unroll
                for (int q = 0; q < 32; ++q) {
                    f2x2 v;
                    v.a = re[brev5(q)];
                    v.b = im[brev5(q)];
                    zs[32 * q + lane] = v;
                }
            }
            fence_proxy_async_smem();
            __syncwarp();
            if (t >= a.z_lo && t < a.z_hi && lane == 0)       // warp-uniform condition
                bulk_s2g(reinterpret_cast<f2x2*>(a.zd) + ((long long)dl * a.zpairs + (t >> 1)) * 1024, zs, kN * 16);

            unsigned wAa = 0u, wAb = 0u, wBa = 0u, wBb = 0u;      // lane q keeps word q of (unit, frame)
            unsigned anyamb = 0u;
            const f2 S2 = f2_pack(S_A, S_B);
            // decisions of bin k of (unit A, unit B) x (frame a, frame b); a missing frame b compares against +inf
            auto decide = [&](int q, int k, bool valid) {
                const f2x2 own = zs[k];
                const f2x2 par = zs[(kN - k) & (kN - 1)];
                // 2 X_a = Z + conj(Zp),  2 X_b = (Z - conj(Zp)) / i
                const f2 ar = f2_add(own.a, par.a), ai = f2_sub(own.b, par.b);
                const f2 br = f2_add(own.b, par.b), bi = f2_sub(par.a, own.a);
                const f2 PA = f2_fma(ar, ar, f2_mul(ai, ai));
                const f2 PB = f2_fma(br, br, f2_mul(bi, bi));
                const float th = valid ? s_thr4[k] : INFINITY;                 // (invalid lanes of the N/2 slot: never set, never ambiguous)
                const float thb = vb ? th : INFINITY;
                // guard band of (unit A, unit B); -1 on the invalid lanes of the N/2 slot (never ambiguous: their "bins" do not exist)
                const f2 gg = f2_fma_s(S2, valid ? s_gco[k] : 0.f, f2_dup(valid ? th * 8.0e-7f : -1.0f));
                const f2 dA = f2_add(PA, f2_dup(-th)), dB = f2_add(PB, f2_dup(-thb));
                const float dAa = f2_lo(dA), dBa = f2_hi(dA), dAb = f2_lo(dB), dBb = f2_hi(dB);
                const float ggA = f2_lo(gg), ggB = f2_hi(gg);
                const unsigned bAa = __ballot_sync(0xffffffffu, dAa > 0.f);
                const unsigned bAb = __ballot_sync(0xffffffffu, dAb > 0.f);
                const unsigned bBa = __ballot_sync(0xffffffffu, dBa > 0.f);
                const unsigned bBb = __ballot_sync(0xffffffffu, dBb > 0.f);
                if (lane == q) { wAa = bAa; wAb = bAb; wBa = bBa; wBb = bBb; }
                const bool mAa = fabsf(dAa) <= ggA, mAb = fabsf(dAb) <= ggA;     // (|-inf| <= gg is false; inf - inf = NaN compares false)
                const bool mBa = fabsf(dBa) <= ggB, mBb = fabsf(dBb) <= ggB;
                if (__any_sync(0xffffffffu, mAa || mAb || mBa || mBb)) {      // rare: remember the bins inside the guard band
                    const unsigned x0 = __ballot_sync(0xffffffffu, mAa), x1 = __ballot_sync(0xffffffffu, mAb);
                    const unsigned x2 = __ballot_sync(0xffffffffu, mBa), x3 = __ballot_sync(0xffffffffu, mBb);
                    anyamb |= 1u << q;
                    if (lane == 0) { s_amb[q] = x0; s_amb[kFW + q] = x1; s_amb[2 * kFW + q] = x2; s_amb[3 * kFW + q] = x3; }
                }
            };
#pragma unroll 2
            for (int q = 0; q < 16; ++q) decide(q, 32 * q + lane, true);
            decide(16, 512 + lane, lane == 0);                 // bin N/2 (lane 0); the other lanes' slots hold mirrored bins
            if (a.dbg.ul == ulA || a.dbg.ul == ulA + 1) {    // parity tap (tests): the FP32 STFT itself
                const bool hi = a.dbg.ul == ulA + 1;
#pragma unroll 1
                for (int k = lane; k < kF; k += 32) {
                    const f2x2 own = zs[k], par = zs[(kN - k) & (kN - 1)];
                    const float zr = hi ? f2_hi(own.a) : f2_lo(own.a), zi = hi ? f2_hi(own.b) : f2_lo(own.b);
                    const float pr = hi ? f2_hi(par.a) : f2_lo(par.a), pi = hi ? f2_hi(par.b) : f2_lo(par.b);
                    float* sp = a.dbg.spec + ((long long)t * kF + k) * 2;
                    sp[0] = 0.5f * (zr + pr); sp[1] = 0.5f * (zi - pi);
                    if (vb) { sp[2 * kF] = 0.5f * (zi + pi); sp[2 * kF + 1] = 0.5f * (pr - zr); }
                }
            }
            if (anyamb) {                             // warp-uniform, rare: redo those bins in float64
                __syncwarp();
                unsigned nre = 0, nun = 0;
                for (int q = 0; q < kFW; ++q) {
                    if (!((anyamb >> q) & 1u)) continue;
                    for (int uf = 0; uf < 4; ++uf) {  // (unit A frame a, A b, B a, B b)
                        unsigned m = s_amb[uf * kFW + q];
                        const T* xrow = (uf & 2) ? xrowB : xrowA;
                        while (m) {
                            const int src = __ffs((int)m) - 1;
                            m &= m - 1;
                            const int r = recheck_bin_fp64(xrow, base + (long long)(uf & 1) * H, i1, g.Lp, g.n_total,
                                                           src + 32 * q, a.tb.wa64, a.tb.cs64, a.tb.thr2_64, lane);
                            ++nre;
                            if (r == 0) { ++nun; continue; }
                            if (lane == q) {
                                const unsigned bit = 1u << src;
                                if (uf == 0) wAa = (r == 2) ? (wAa | bit) : (wAa & ~bit);
                                else if (uf == 1) wAb = (r == 2) ? (wAb | bit) : (wAb & ~bit);
                                else if (uf == 2) wBa = (r == 2) ? (wBa | bit) : (wBa & ~bit);
                                else wBb = (r == 2) ? (wBb | bit) : (wBb & ~bit);
                            }
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) {
                    atomicAdd(&a.cnt->rechecked, (unsigned long long)nre);
                    if (nun) atomicAdd(&a.cnt->unresolved, (unsigned long long)nun);
                }
            }
            if (lane < kFW) {
                unsigned* dA = a.bits + ((long long)ulA * g.T + t) * kFW + lane;
                unsigned* dB = dA + (long long)g.T * kFW;
                dA[0] = wAa;
                dB[0] = wBa;
                if (vb) { dA[kFW] = wAb; dB[kFW] = wBb; }
            }
        }
        // |X|^2 <= N * (frame energy): could any bin of this run have reached its top_db floor?
        if (4.0f * (float)kN * emax >= 0.999f * a.min_floor4 && lane == 0) atomicOr(a.need_rowmax, 1u);
    }
    bulk_wait_read_all();                                     // no bulk store may outlive the CTA's shared memory
}

}  // namespace b200
