// gate_adjoint.cuh -- the cross-unit sum of the gate's adjoint (b200gate_adjoint).
//
// With its masks held fixed, unit u = (chunk i, channel c) is a linear map of its padded span [i cs - pad, (i + 1) cs + pad)
// (base.py:130-156).  The adjoint synthesis kernels (k2_synthesize<.., ADJ>, gk_stft / gk_ola<.., ADJ>) write each unit's
// transposed map applied to the output gradient over that whole span; this kernel adds the spans of overlapping units
// into the input gradient.  Every sample is owned by one thread, which adds the units covering it in increasing unit
// order onto what earlier batches left there: no atomics, so the gradient is the same in every bit from run to run and
// for any split of the units into workspace batches, however many units overlap (padding >= chunk_size included).
#pragma once
#include "gate_kernels.cuh"

namespace b200 {

__device__ __forceinline__ long long adj_floordiv(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// units [g.u0, g.u0 + g.n_units) of this batch; adj[ul][j] is unit g.u0 + ul's value at chunk-local index j in [0, Lp);
// samples [s_lo, s_hi) of channels c0 + blockIdx.y are updated
template <typename S, typename G>
__global__ void __launch_bounds__(256) k_adj_gather(const S* __restrict__ adj, long long adj_pitch, G* __restrict__ grad,
                                                    long long grad_stride, const Geom g, long long s_lo, long long s_hi,
                                                    int c0) {
    const int c = c0 + (int)blockIdx.y;
    G* grow = grad + (long long)c * grad_stride;
    const long long i_first = g.u0 / g.C, i_last = (g.u0 + g.n_units - 1) / g.C;
    for (long long s = s_lo + (long long)blockIdx.x * blockDim.x + threadIdx.x; s < s_hi;
         s += (long long)gridDim.x * blockDim.x) {
        // chunks i whose padded span holds s: i cs - pad <= s < (i + 1) cs + pad
        const long long i_lo = max(i_first, adj_floordiv(s - g.pad, g.step));
        const long long i_hi = min(i_last, adj_floordiv(s + g.pad, g.step));
        G v = grow[s];
        for (long long i = i_lo; i <= i_hi; ++i) {
            const long long u = i * g.C + c;
            if (u < g.u0 || u >= g.u0 + g.n_units) continue;
            v += (G)adj[(u - g.u0) * adj_pitch + (s - (i * g.step - g.pad))];
        }
        grow[s] = v;
    }
}

}  // namespace b200
