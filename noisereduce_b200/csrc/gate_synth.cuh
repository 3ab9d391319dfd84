// gate_synth.cuh -- k2c_synthesize: the synthesis half of the gate when the analysis kernel kept the spectra.
//
// Reference semantics (paths relative to the reference checkout): mask apply  X * mask  at
// noisereduce/spectralgate/stationary.py:117 / nonstationary.py:87, scipy.signal.istft as called at
// stationary.py:120-126 (window, overlap-add, sum-of-squares normalisation, centre crop), chunk centre
// written back at base.py:150.
//
// One warp owns a run of output hops of one (chunk, channel) unit and walks its frame pairs.  Per pair:
//   1. the pair's packed spectrum Z = X_a + i X_b (8 KB, written by k1 / k1n) and its two mask rows arrive in
//      this warp's shared-memory buffers by 1-D bulk asynchronous copies (cp.async.bulk -> TMA engine, SASS
//      UBLKCP) signalled on a per-warp mbarrier; the copies of pair t+2 are issued as soon as pair t has been
//      read, so they travel behind a whole inverse transform (kMaskBits*: only the spectrum is copied; the kernel
//      smooths the pair's mask rows from the 1-bit decisions itself, see below);
//   2. masks are applied on the packed spectrum,  Z'[k] = s Z[k] + d conj(Z[N-k]),  s, d = (m_a +- m_b)/2.
//      The mirrored bin is read from the same shared buffer by its FLAT index (N - k) & (N - 1), which is what
//      makes lane 0 (bins 0, 32, ... whose mirrors live in other SLOTS of the same lane) an ordinary lane: no
//      shuffles, no per-lane selects.  A lane computes both members of its 16 lower pairs; the upper members
//      travel to their owners through the (idle) FFT exchange tile;
//   3. ONE inverse 1024-point FFT (ifft(z) = swap(fft(swap z)): the apply step writes real/imaginary parts
//      exchanged), synthesis window, overlap-add in registers, normalise, store the chunk centre.
#pragma once
#include "gate_kernels.cuh"

namespace b200 {

__device__ __forceinline__ unsigned prmt(unsigned a, unsigned b, unsigned sel) {
#ifdef B200_CUSIM_BUILD
    const unsigned long long v = ((unsigned long long)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((sel >> (4 * i)) & 7))) & 0xFFu) << (8 * i);
    return r;
#else
    return __byte_perm(a, b, sel);
#endif
}

// Mask modes.  kMaskU16*: the pair's integer numerators are bulk-copied from `num` (written by k_smooth_packed /
// k_smooth_generic).  kMaskBits*: the kernel smooths the mask itself from the 1-bit decisions (`bits` | `rowflag`),
// with k_smooth_packed's integer arithmetic, so the numerators never leave shared memory:
//   time direction   per-bin second-difference recurrence (triangle = box * box) in byte lanes, 4 bins per word;
//                    a lane owns bins 16 lane .. 16 lane + 15 (one nibble of bits per 4 bins) and lane 0 also bins
//                    512..515; the (d1, s2) state of the warp's unit lives in shared memory between pairs and is warmed
//                    up from the 2 nt frames before the item's first pair;
//   frequency        dp4a dot products of the time sums (two byte rows, one per frame, in the idle exchange tile) with
//                    the packed triangle taps; the results go to `mbuf` in the num_index pair layout, which is what the
//                    kMaskU16 modes would have copied there.
// *Blend: prop_decrease < 1 (the edge-factor term of the zero-padded smoothing).
enum { kMaskU16 = 0, kMaskU16Blend = 1, kMaskF32 = 2, kMaskBits = 3, kMaskBitsBlend = 4 };
#ifndef B200_K2C_PTW
#define B200_K2C_PTW 0              // inter-pass twiddles on packed register pairs (warp_fft1024_ptw)
#endif


constexpr int kK2cTableBytes = kN * 4 + kN * 8 + kFPad * 4;          // synthesis window, twiddles, frequency edge factors
constexpr int kK2cTileBytes = kExchFloats * 4;                        // 4224: FFT exchange tile, also the 513 x float2 mirror buffer
constexpr int kSynGroups = kF / 4 + 1;                                // 129 four-bin groups: bins 0..515
constexpr int kSynNumBytes = kSynGroups * 16;                         // 2064: the pair's numerators, bins 0..515
constexpr int kSynStateBytes = (kSynGroups * 8 + 15) & ~15;           // 1040: (d1, s2) per group
constexpr int kSynRowPitch = 32 + 640;                                // time-sum row: <= 32 halo bytes + 160 groups of 4 bins
constexpr int kSynMaxTapWords = 10;
static_assert(2 * kSynRowPitch <= kK2cTileBytes, "time-sum rows must fit the exchange tile");
template <int MK> __host__ __device__ constexpr int k2c_mask_bytes() {
    return MK == kMaskF32 ? 2 * kFPad * 4 : (MK >= kMaskBits ? kSynNumBytes + kSynStateBytes : 2 * kFPad * 2);
}
template <int MK> __host__ __device__ constexpr int k2c_warp_bytes() { return kN * 8 + k2c_mask_bytes<MK>() + kK2cTileBytes + 16; }
template <int MK> __host__ __device__ constexpr int k2c_smem_bytes() { return kK2cTableBytes + kWarps * k2c_warp_bytes<MK>(); }
static_assert(kK2cTileBytes >= 513 * 8, "mirror buffer must fit the exchange tile");

// kMaskBits*, frequency direction of one frame pair: rows = the two time-sum byte rows (row byte sm_pad + k = bin k),
// num = the pair's numerators (num_index pair layout, bins 0..515).  Group i (bins 4i..4i+3) goes to lane i % 32, so
// the row words a lane reads and the 16-byte results it stores are consecutive across the warp.
template <int NTW>
__device__ __forceinline__ void k2c_freq_taps(const unsigned char* rows, unsigned char* num, const K2Args& a, int lane) {
    unsigned taps[NTW];
#pragma unroll
    for (int m = 0; m < NTW; ++m) taps[m] = a.sm_taps[m];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
        const int i = lane + 32 * j;
        if (j == 4 && i >= kSynGroups) break;                  // the fifth group is lane 0's (bins 512..515)
        unsigned o[2][4];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const unsigned* rw = reinterpret_cast<const unsigned*>(rows + r * kSynRowPitch) + i + a.sm_ws;
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
                o[r][jj] = acc;
            }
        }
        *reinterpret_cast<uint4*>(num + 16 * i) = uint4{o[0][0] | (o[1][0] << 16), o[0][1] | (o[1][1] << 16),
                                                        o[0][2] | (o[1][2] << 16), o[0][3] | (o[1][3] << 16)};
    }
}

#ifndef B200_K2C_MINBLOCKS
#define B200_K2C_MINBLOCKS 3
#endif
template <int HR, int MK, typename T>
__global__ void __launch_bounds__(kThreads, B200_K2C_MINBLOCKS) k2c_synthesize(const K2Args a) {
    constexpr int NH = 32 / HR;             // frames overlapping one hop (win / hop)
    constexpr int MB = k2c_mask_bytes<MK>();
    constexpr int WB = k2c_warp_bytes<MK>();
    constexpr bool kBits = MK == kMaskBits || MK == kMaskBitsBlend;                 // smoothing in this kernel
    constexpr bool kBlend = MK == kMaskU16Blend || MK == kMaskBitsBlend;
    B200_DYN_SMEM(unsigned char, smraw);
    const Geom& g = a.g;
    const int H = g.H;
    float* s_ws = reinterpret_cast<float*>(smraw);
#if B200_K2C_PTW
    tw4_t* s_tw4 = reinterpret_cast<tw4_t*>(smraw + kN * 4);
#else
    float2* s_tw = reinterpret_cast<float2*>(smraw + kN * 4);
#endif
    float* s_ef = reinterpret_cast<float*>(smraw + kN * 12);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* wbase = smraw + kK2cTableBytes + warp * WB;
    float2* zbuf = reinterpret_cast<float2*>(wbase);
    unsigned char* mbuf = wbase + kN * 8;
    float* tile = reinterpret_cast<float*>(wbase + kN * 8 + MB);
    float2* qbuf = reinterpret_cast<float2*>(tile);
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(wbase + kN * 8 + MB + kK2cTileBytes);
    for (int i = threadIdx.x; i < kN; i += kThreads) {
        s_ws[i] = a.tb.ws[i];
#if !B200_K2C_PTW
        s_tw[i] = a.tb.tw[i];
#endif
    }
#if B200_K2C_PTW
    build_tw4(s_tw4, a.tb.tw, threadIdx.x, kThreads);
#endif
    for (int i = threadIdx.x; i < kFPad; i += kThreads) s_ef[i] = a.tb.ef[i];
    if (lane == 0) mbar_init(bar, 1);
    mbar_init_fence();
    __syncthreads();
    unsigned phase = 0;

    float invn[HR];                          // interior overlap-add norm of this lane's HR rows of a hop
#pragma unroll
    for (int r = 0; r < HR; ++r) invn[r] = a.tb.invn[r * 32 + lane];

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
        const long long sig_len = (long long)(g.T - 1) * H;          // istft output length
        if (jp_hi > sig_len) jp_hi = sig_len;                        // beyond it the reference leaves zeros
        if (jp_hi <= g.pad) continue;
        const long long jlo = g.pad + kN / 2, jhi = jp_hi + kN / 2;
        const int h_lo = (int)(jlo / H), h_hi = (int)((jhi + H - 1) / H);
        const int hs = h_lo + run * a.run;
        const int he = min(hs + a.run, h_hi);
        if (hs >= he) continue;
        const int t_start = max(0, hs - (NH - 1)) & ~1;              // k1 packed frames (2j, 2j+1): walk the same pairs
        const int t_last = min(he - 1, g.T - 1);
        T* yrow = static_cast<T*>(a.y) + (long long)c * g.out_stride;
        const float2* zunit = a.zcache + (long long)ul * a.zpairs * 1024;
        const unsigned short* munit = (MK == kMaskF32 || kBits) ? nullptr : a.num + (long long)ul * a.zpairs * (2 * kFPad);
        const float* funit = (MK == kMaskF32) ? a.fmask + (long long)ul * g.T * kFPad : nullptr;

        float acc[32 + HR];
#pragma unroll
        for (int r = 0; r < 32 + HR; ++r) acc[r] = 0.f;

        // request pair (tt, tt+1): spectrum + mask rows.  All lanes have finished reading the buffers.
        auto stage = [&](int tt) {
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) {
                const bool vb2 = tt + 1 <= t_last;
                const unsigned mbytes = kBits ? 0u : ((MK == kMaskF32 && !vb2) ? (unsigned)(kFPad * 4) : (unsigned)MB);
                mbar_expect_tx(bar, (unsigned)(kN * 8) + mbytes);
                bulk_g2s(zbuf, zunit + (long long)(tt >> 1) * 1024, kN * 8, bar);
                if (MK == kMaskF32) bulk_g2s(mbuf, funit + (long long)tt * kFPad, mbytes, bar);
                else if (!kBits) bulk_g2s(mbuf, munit + (long long)(tt >> 1) * (2 * kFPad), mbytes, bar);
            }
        };
        if (t_start <= t_last) stage(t_start);

        // ---- kMaskBits*: time-direction recurrence of k_smooth_packed, frames fed from tau_s = t_start - nt on ------
        const int aa = a.nt + 1, tau_s = t_start - a.nt;
        const unsigned* bunit = kBits ? a.bits + (long long)ul * g.T * kFW : nullptr;
        uint2* sstate = reinterpret_cast<uint2*>(mbuf + kSynNumBytes);     // [4][32] lane groups, then group 128
        // the top_db row flags of this lane's bins (x: its bits word, y: bins 512..515), OR-ed into every frame
        auto rowflags = [&]() -> uint2 {
            return uint2{__ldg(a.rowflag + ul * kFW + (lane >> 1)), __ldg(a.rowflag + ul * kFW + 16)};
        };
        // this lane's decisions of frame tau: x = its 16 bins (4 bits per group), y = bins 512..515 (lane 0 only);
        // frames before tau_s count as zero, as in k_smooth_packed
        auto fetch = [&](int tau, uint2 fl) -> uint2 {
            if (tau < tau_s || tau < 0 || tau >= g.T) return uint2{0u, 0u};
            const unsigned* row = bunit + (long long)tau * kFW;
            const unsigned w = __ldg(row + (lane >> 1)) | fl.x;
            const unsigned w5 = (__ldg(row + 16) | fl.y) & 0xFu;
            return uint2{w >> ((lane & 1) * 16), lane == 0 ? w5 : 0u};
        };
        auto advance = [&](int tau, uint2 fl, unsigned (&d1)[5], unsigned (&s2)[5]) {
            const uint2 na = fetch(tau, fl), nb = fetch(tau - aa, fl), nc = fetch(tau - 2 * aa, fl);
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                const unsigned xa = j < 4 ? na.x >> (4 * j) : na.y;
                const unsigned xb = j < 4 ? nb.x >> (4 * j) : nb.y;
                const unsigned xc = j < 4 ? nc.x >> (4 * j) : nc.y;
                const unsigned ea = ((xa & 0xFu) * 0x00204081u) & 0x01010101u;         // nibble -> one bit per byte
                const unsigned eb = ((xb & 0xFu) * 0x00204081u) & 0x01010101u;
                const unsigned ec = ((xc & 0xFu) * 0x00204081u) & 0x01010101u;
                d1[j] = d1[j] + ea + ec - 2u * eb;                                       // biased by 0x10 per byte
                s2[j] = s2[j] + d1[j] - 0x10101010u;
            }
        };
        auto save_state = [&](const unsigned (&d1)[5], const unsigned (&s2)[5]) {
#pragma unroll
            for (int j = 0; j < 4; ++j) sstate[32 * j + lane] = uint2{d1[j], s2[j]};
            if (lane == 0) sstate[128] = uint2{d1[4], s2[4]};
        };
        if (kBits && t_start <= t_last) {               // warm-up: the 2 nt frames before the first pair's centre
            unsigned d1[5], s2[5];
#pragma unroll
            for (int j = 0; j < 5; ++j) { d1[j] = 0x10101010u; s2[j] = 0u; }
            const uint2 fl = rowflags();
#pragma unroll 1
            for (int tau = tau_s; tau < t_start + a.nt; ++tau) advance(tau, fl, d1, s2);
            save_state(d1, s2);
        }

        for (int t = t_start; t < he; t += 2) {
            const bool va = (t <= t_last), vb = (t + 1 <= t_last);
            if (va) {                                   // vb implies va
                if (kBits) {                            // this pair's numerators, into mbuf
                    unsigned d1[5], s2[5];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint2 v = sstate[32 * j + lane];
                        d1[j] = v.x;
                        s2[j] = v.y;
                    }
                    {
                        const uint2 v = sstate[128];
                        d1[4] = lane == 0 ? v.x : 0x10101010u;
                        s2[4] = lane == 0 ? v.y : 0u;
                    }
                    const uint2 fl = rowflags();
                    unsigned char* rows = reinterpret_cast<unsigned char*>(tile);
                    __syncwarp();                       // the previous pair's transform is done with the tile
#pragma unroll
                    for (int r = 0; r < 2; ++r) {       // time sums of frames t, t+1 (centres of tau = t + nt, t + 1 + nt)
                        advance(t + r + a.nt, fl, d1, s2);
                        unsigned char* row = rows + r * kSynRowPitch;
                        *reinterpret_cast<uint4*>(row + a.sm_pad + 16 * lane) = uint4{s2[0], s2[1], s2[2], s2[3]};
                        // lane 0: bins 512..515; lanes 1..31: the zero tail the taps of the last bins read
                        *reinterpret_cast<unsigned*>(row + a.sm_pad + 512 + 4 * lane) = s2[4];
                        if (4 * lane < a.sm_pad) reinterpret_cast<unsigned*>(row)[lane] = 0u;     // zero halo
                    }
                    save_state(d1, s2);
                    __syncwarp();
                    switch (a.sm_ntw) {
                        case 4: k2c_freq_taps<4>(rows, mbuf, a, lane); break;
                        case 7: k2c_freq_taps<7>(rows, mbuf, a, lane); break;
                        case 9: k2c_freq_taps<9>(rows, mbuf, a, lane); break;
                        default: k2c_freq_taps<kSynMaxTapWords>(rows, mbuf, a, lane); break;
                    }
                    __syncwarp();                       // numerators visible; the tile is free for the mirror buffer
                }
                float re[32], im[32];                   // what the FFT call sees: re = Im Z', im = Re Z'
                mbar_wait(bar, phase);
                phase ^= 1u;
                // ---- mask scalars of this pair --------------------------------------------------------------
                float pa = 0.f, ca = 0.f, pb = 0.f, cb = 0.f, eta = 0.f, etb = 0.f;
                const float* mA = reinterpret_cast<const float*>(mbuf);
                const float* mB = vb ? mA + kFPad : mA;
                const unsigned* m32 = reinterpret_cast<const unsigned*>(mbuf);
                if (MK == kMaskF32) {
                    pa = 0.5f;
                    pb = vb ? 0.5f : 0.f;
                } else {
                    pa = 0.5f * a.pD;                   // masks are formed already halved: s, d = m_a/2 +- m_b/2
                    ca = -8388608.0f * pa;              // the 2^23 of the integer -> float bit pattern, folded into the FMA
                    pb = vb ? pa : 0.f;
                    cb = vb ? ca : 0.f;
                    if (kBlend) {
                        eta = 0.5f * a.one_minus_p * time_edge(t, g.T, a.nt);
                        etb = vb ? 0.5f * a.one_minus_p * time_edge(t + 1, g.T, a.nt) : 0.f;
                    }
                }
                auto half_masks = [&](int kk, float& ma, float& mb) {      // m_a / 2, m_b / 2 at bin kk
                    if (MK == kMaskF32) {
                        ma = pa * mA[kk];
                        mb = pb * mB[kk];
                    } else {
                        const unsigned pk = m32[kk];
                        const float fa = __uint_as_float(prmt(pk, 0x4B00u, 0x5410u));     // 2^23 + n_a
                        const float fb = __uint_as_float(prmt(pk, 0x4B00u, 0x5432u));     // 2^23 + n_b
                        if (kBlend) {
                            const float e = s_ef[kk];
                            ma = fmaf(fa - 8388608.0f, pa, eta * e);
                            mb = fmaf(fb - 8388608.0f, pb, etb * e);
                        } else {
                            ma = fmaf(fa, pa, ca);
                            mb = fmaf(fb, pb, cb);
                        }
                    }
                };
                if (a.dbg.ul == ul) {                        // parity tap (tests): the masks this pair applies
#pragma unroll 1
                    for (int k = lane; k < kF; k += 32) {
                        float ma, mb;
                        half_masks(k, ma, mb);
                        a.dbg.mask[(long long)t * kF + k] = 2.0f * ma;
                        if (vb) a.dbg.mask[(long long)(t + 1) * kF + k] = 2.0f * mb;
                    }
                }
                // Float masks: a non-finite value in one frame's row would reach its partner through s and d (both
                // frames share Z).  The apply below notes any non-finite s; only then (a warp vote per pair) is the
                // offending frame found, its row zeroed in this warp's buffer, the apply redone and the frame's whole
                // overlap-add span made NaN after the transform -- the reference's istft of a NaN row.  Finite masks
                // take one pass and the very same arithmetic as before.
                bool nan_a = false, nan_b = false;
#pragma unroll 1
                for (int pass = 0;; ++pass) {
                    bool bad = false;
                    // ---- lower pairs k = lane + 32 q < 512: both members -------------------------------------------
#pragma unroll
                    for (int q = 0; q < 16; ++q) {
                        const int k = 32 * q + lane;
                        const float2 own = zbuf[k];
                        const float2 par = zbuf[q == 0 ? ((kN - lane) & (kN - 1)) : (kN - k)];
                        float ma, mb;
                        half_masks(k, ma, mb);
                        const float s = ma + mb, d = ma - mb;
                        if (MK == kMaskF32) bad |= !(fabsf(s) < INFINITY);
                        // Z'[k] = s Z[k] + d conj(Z[N-k]);  Z'[N-k] = s Z[N-k] + d conj(Z[k])
                        im[q] = fmaf(d, par.x, s * own.x);
                        re[q] = fmaf(-d, par.y, s * own.y);
                        const float qr = fmaf(d, own.x, s * par.x), qi = fmaf(-d, own.y, s * par.y);
                        qbuf[512 - k] = make_float2(qi, qr);             // slot of bin N - k, stored (re, im) as the FFT wants them
                    }
                    {   // slot 16: bins 512 + lane, computed directly (lane 0 = the self-mirrored bin N/2)
                        const float2 own = zbuf[512 + lane];
                        const float2 par = zbuf[512 - lane];
                        float ma, mb;
                        half_masks(512 - lane, ma, mb);
                        const float s = ma + mb, d = ma - mb;
                        if (MK == kMaskF32) bad |= !(fabsf(s) < INFINITY);
                        im[16] = fmaf(d, par.x, s * own.x);
                        re[16] = fmaf(-d, par.y, s * own.y);
                    }
                    __syncwarp();
#pragma unroll
                    for (int q = 17; q < 32; ++q) {
                        const float2 v = qbuf[32 * (q - 16) + lane];
                        re[q] = v.x;
                        im[q] = v.y;
                    }
                    __syncwarp();
                    if (MK != kMaskF32 || pass > 0 || !__any_sync(0xffffffffu, bad)) break;
                    float* mw = reinterpret_cast<float*>(mbuf);
                    bool ba = false, bb = false;
                    for (int k = lane; k < kF; k += 32) {
                        ba |= !(fabsf(mw[k]) < INFINITY);
                        bb |= !(fabsf(mw[kFPad + k]) < INFINITY);
                    }
                    nan_a = __any_sync(0xffffffffu, ba);
                    nan_b = vb && __any_sync(0xffffffffu, bb);
                    for (int k = lane; k < kF; k += 32) {
                        if (nan_a) mw[k] = 0.f;
                        if (nan_b) mw[kFPad + k] = 0.f;
                    }
                    __syncwarp();
                }
                if (t + 2 <= t_last) stage(t + 2);           // next pair streams in behind this pair's transform
#if B200_K2C_PTW
                warp_fft1024_ptw(re, im, tile, s_tw4, lane);
#else
                warp_fft1024(re, im, tile, s_tw, lane);
#endif
                // now im = N a'[n], re = N b'[n] (n = lane + 32 q) at slot brev5(q)
                if (MK == kMaskF32 && (nan_a || nan_b)) {
#pragma unroll
                    for (int q = 0; q < 32; ++q) {
                        if (nan_a) im[q] = __uint_as_float(0x7fc00000u);
                        if (nan_b) re[q] = __uint_as_float(0x7fc00000u);
                    }
                }
#pragma unroll
                for (int q = 0; q < 32; ++q) {
                    const float w = s_ws[lane + 32 * q];
                    acc[q] = fmaf(im[brev5(q)], w, acc[q]);
                    acc[q + HR] = fmaf(re[brev5(q)], w, acc[q + HR]);
                }
            }
            // hops t and t+1 are now complete (all frames <= t+1 have been added)
            {
                const long long jp0 = (long long)t * H - kN / 2;             // chunk-local index of row 0, lane 0
                if (t >= hs && t + 1 < he && t >= NH - 1 && t + 1 <= g.T - 1 && jp0 >= g.pad &&
                    jp0 + 2 * H <= jp_hi) {
                    // both hops interior and fully inside the chunk centre: 2*HR coalesced row stores
                    T* dst = yrow + i1 + jp0 + lane;
#pragma unroll
                    for (int r = 0; r < 2 * HR; ++r) dst[32 * r] = st_cast<T>(acc[r] * invn[r % HR]);
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
                            inv = a.tb.invn[ro];
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

}  // namespace b200
