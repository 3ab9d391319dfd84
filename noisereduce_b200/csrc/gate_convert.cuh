// gate_convert.cuh -- sample-format conversions for callers whose samples already live on the device
// (b200gate_convert, include/b200gate.h).
//
// reduce_noise() runs any dtype other than float32 / int16 / float64 the reference's way: the samples are promoted to
// float64 (base.py:140), gated, and the result is cast back with ndarray.astype (base.py:218-226).  The stationary
// thresholds start from np.mean(noise, axis=0) in the clip's own dtype rules (stationary.py:61).  These kernels do the
// same three steps on device memory, bit for bit as numpy does them on x86-64 for unit-stride rows (the rows the
// numpy route casts; numpy's strided cast loops can map out-of-range values to uint32 / uint64 differently):
//   * promote: exact for every format except 64-bit integers beyond 2^53, which round to nearest even like numpy's
//     int64 -> float64 cast;
//   * demote: float16 rounds once (numpy's double -> half, not through float32); bool is v != 0 (NaN is True); integers
//     truncate toward zero, and NaN, +-inf and out-of-range values take x86-64's cvttsd2si "integer indefinite" result
//     (0x80000000 / 0x8000000000000000) before the truncation to 8 or 16 bits; uint32 / uint64 follow the compiler's
//     unsigned sequence (v >= 2^31 ? cvtt(v - 2^31) ^ 2^31 : cvtt(v), and the same with 2^63);
//   * channel mean: float16 and float32 sum in float32 in channel order and divide once, float16 then rounds to half;
//     every other format sums in float64 in channel order.  (numpy sums pairwise when the reduced axis is the
//     contiguous one, i.e. channel-adjacent layouts; the caller hands these kernels row-major samples.)
// Every value is computed with explicit range checks and integer arithmetic, never with the hardware's saturating
// float -> integer conversions, so the CPU simulator build computes the same bits.
#pragma once

#include "cuda_compat.h"
#include "../../include/b200gate.h"

#ifndef B200_CUSIM_BUILD
#include <cuda_fp16.h>
#endif

namespace b200 {

__host__ __device__ inline int cv_size(int dt) {
    switch (dt) {
        case B200GATE_F32: case B200GATE_I32: case B200GATE_U32: return 4;
        case B200GATE_I16: case B200GATE_U16: case B200GATE_F16: return 2;
        case B200GATE_F64: case B200GATE_I64: case B200GATE_U64: return 8;
        case B200GATE_BOOL: case B200GATE_I8: case B200GATE_U8: return 1;
        default: return 0;
    }
}

// x86-64 cvttsd2si: truncation toward zero, "integer indefinite" (the most negative value) for NaN / out of range
__device__ __forceinline__ int cv_cvtt32(double v) {
    return (v > -2147483649.0 && v < 2147483648.0) ? (int)v : (int)0x80000000u;
}
__device__ __forceinline__ long long cv_cvtt64(double v) {
    return (v >= -9223372036854775808.0 && v < 9223372036854775808.0) ? (long long)v : (long long)0x8000000000000000ull;
}

__device__ __forceinline__ unsigned long long cv_f64_bits(double v) {
#ifdef B200_CUSIM_BUILD
    unsigned long long b; memcpy(&b, &v, 8); return b;
#else
    return (unsigned long long)__double_as_longlong(v);
#endif
}
__device__ __forceinline__ double cv_bits_f64(unsigned long long b) {
#ifdef B200_CUSIM_BUILD
    double v; memcpy(&v, &b, 8); return v;
#else
    return __longlong_as_double((long long)b);
#endif
}

// half bits -> double, exact (a NaN keeps its sign and payload, as numpy's npy_half_to_double)
__device__ __forceinline__ double cv_half_to_f64(unsigned short h) {
    const unsigned long long sign = (unsigned long long)(h & 0x8000u) << 48;
    const int e = (h >> 10) & 0x1f;
    const unsigned m = h & 0x3ffu;
    if (e == 0x1f) return cv_bits_f64(sign | 0x7ff0000000000000ull | ((unsigned long long)m << 42));
    const double mag = e == 0 ? (double)m * 0x1p-24 : (double)(m | 0x400u) * ldexp(1.0, e - 25);
    return sign ? -mag : mag;
}

// double -> half bits, one rounding to nearest even (numpy's npy_double_to_half); NaN keeps its sign and the top of
// its payload (0x7c00 + payload >> 42, never 0x7c00), as numpy does
__device__ __forceinline__ unsigned short cv_f64_to_half(double v) {
    const unsigned long long b = cv_f64_bits(v);
    const unsigned short sign = (unsigned short)((b >> 48) & 0x8000u);
    if ((b & 0x7ff0000000000000ull) == 0x7ff0000000000000ull && (b & 0x000fffffffffffffull)) {
        unsigned short r = (unsigned short)(0x7c00u + ((b & 0x000fffffffffffffull) >> 42));
        if (r == 0x7c00u) ++r;
        return sign | r;
    }
#ifdef B200_CUSIM_BUILD
    const int ex = (int)((b >> 52) & 0x7ff);
    if (ex == 0x7ff) return sign | 0x7c00u;                               // +-inf
    const int e = ex - 1023;
    if (e > 15) return sign | 0x7c00u;                                    // >= 65536: overflows to inf
    if (e < -25 || ex == 0) return sign;                                  // < 2^-25: rounds to zero
    const unsigned long long m = (b & 0x000fffffffffffffull) | (1ull << 52);
    const int shift = e >= -14 ? 42 : 42 + (-14 - e);                     // subnormal halves keep fewer bits
    unsigned long long q = m >> shift;
    const unsigned long long rem = m & ((1ull << shift) - 1), halfway = 1ull << (shift - 1);
    if (rem > halfway || (rem == halfway && (q & 1))) ++q;
    if (e >= -14) return sign | (unsigned short)(((unsigned)(e + 15) << 10) + (unsigned)(q - 1024));   // a carry moves the exponent
    return sign | (unsigned short)q;                                      // q == 1024 is the smallest normal half
#else
    return __half_as_ushort(__double2half(v));                           // cvt.rn.f16.f64: one rounding
#endif
}

template <int DT>
__device__ __forceinline__ double cv_load(const void* p, long long i) {
    if (DT == B200GATE_F32) return (double)((const float*)p)[i];
    if (DT == B200GATE_F64) return ((const double*)p)[i];
    if (DT == B200GATE_F16) return cv_half_to_f64(((const unsigned short*)p)[i]);
    if (DT == B200GATE_BOOL) return ((const unsigned char*)p)[i] != 0 ? 1.0 : 0.0;
    if (DT == B200GATE_I8) return (double)((const signed char*)p)[i];
    if (DT == B200GATE_U8) return (double)((const unsigned char*)p)[i];
    if (DT == B200GATE_I16) return (double)((const short*)p)[i];
    if (DT == B200GATE_U16) return (double)((const unsigned short*)p)[i];
    if (DT == B200GATE_I32) return (double)((const int*)p)[i];
    if (DT == B200GATE_U32) return (double)((const unsigned*)p)[i];
#ifdef B200_CUSIM_BUILD
    if (DT == B200GATE_I64) return (double)((const long long*)p)[i];
    return (double)((const unsigned long long*)p)[i];
#else
    if (DT == B200GATE_I64) return __ll2double_rn(((const long long*)p)[i]);
    return __ull2double_rn(((const unsigned long long*)p)[i]);
#endif
}

template <int DT>
__device__ __forceinline__ void cv_store(void* p, long long i, double v) {
    if (DT == B200GATE_F32) ((float*)p)[i] = (float)v;
    else if (DT == B200GATE_F64) ((double*)p)[i] = v;
    else if (DT == B200GATE_F16) ((unsigned short*)p)[i] = cv_f64_to_half(v);
    else if (DT == B200GATE_BOOL) ((unsigned char*)p)[i] = v != 0.0 ? 1 : 0;          // NaN != 0: True
    else if (DT == B200GATE_I8) ((signed char*)p)[i] = (signed char)cv_cvtt32(v);
    else if (DT == B200GATE_U8) ((unsigned char*)p)[i] = (unsigned char)cv_cvtt32(v);
    else if (DT == B200GATE_I16) ((short*)p)[i] = (short)cv_cvtt32(v);
    else if (DT == B200GATE_U16) ((unsigned short*)p)[i] = (unsigned short)cv_cvtt32(v);
    else if (DT == B200GATE_I32) ((int*)p)[i] = cv_cvtt32(v);
    else if (DT == B200GATE_U32)                 // v >= 2^31 ? cvtt32(v - 2^31) ^ 2^31 : cvtt32(v)
        ((unsigned*)p)[i] = v >= 2147483648.0 ? ((unsigned)cv_cvtt32(v - 2147483648.0) ^ 0x80000000u) : (unsigned)cv_cvtt32(v);
    else if (DT == B200GATE_I64) ((long long*)p)[i] = cv_cvtt64(v);
    else                                         // v >= 2^63 ? cvtt64(v - 2^63) ^ 2^63 : cvtt64(v)
        ((unsigned long long*)p)[i] = v >= 9223372036854775808.0
            ? ((unsigned long long)cv_cvtt64(v - 9223372036854775808.0) ^ 0x8000000000000000ull)
            : (unsigned long long)cv_cvtt64(v);
}

// dst[c][j] = src[c][j] converted, rows with their own strides (elements)
template <int SDT, int DDT>
__global__ void k_convert(const void* __restrict__ src, long long ss, void* __restrict__ dst, long long ds, long long C,
                          long long N) {
    for (long long c = blockIdx.y; c < C; c += gridDim.y)
        for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (long long)gridDim.x * blockDim.x)
            cv_store<DDT>(dst, c * ds + j, cv_load<SDT>(src, c * ss + j));
}

// dst[j] = np.mean(src[:, j]) widened to float64 (exact: a float32 / half mean is representable)
template <int SDT>
__global__ void k_channel_mean(const void* __restrict__ src, long long ss, double* __restrict__ dst, long long C,
                               long long n) {
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) {
        if (SDT == B200GATE_F16 || SDT == B200GATE_F32) {
            float s = 0.f;                                   // umr_sum(..., dtype=float32): rows added in order
            for (long long c = 0; c < C; ++c) s = s + (float)cv_load<SDT>(src, c * ss + j);
            const float m = (float)((double)s / (double)C);  // true_divide(ret, intp(C), out=ret): float64 loop, cast back
            dst[j] = SDT == B200GATE_F16 ? cv_half_to_f64(cv_f64_to_half((double)m)) : (double)m;
        } else {
            double s = 0.0;
            for (long long c = 0; c < C; ++c) s = s + cv_load<SDT>(src, c * ss + j);
            dst[j] = s / (double)C;
        }
    }
}

}  // namespace b200
