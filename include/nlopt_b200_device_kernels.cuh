// nlopt_b200_device_kernels.cuh -- the device-only part of nlopt_b200_device.cuh: the map and fold kernels of the
// asynchronous functor form (nlopt_b200_dfunc2 / nlopt_b200_dmfunc2) and the functor traits.
//
// It needs no system or CUDA runtime header, so the same text compiles under nvcc (through nlopt_b200_device.cuh) and
// under NVRTC, where the library embeds it and instantiates map_group_kernel / map_group_mkernel for a functor given as
// source (nlopt_b200_jit_create, include/nlopt_b200.h).  Both compilers see one definition of every kernel, so a functor
// compiled either way reduces its terms in the same order to the same bits.
#pragma once

#include "nlopt_b200.h"

namespace nlopt_b200 {

namespace detail {

constexpr int kThreads = 256;

__device__ __forceinline__ double block_sum(double v, double *smem)
{
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, off));
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kThreads / 32; ++w) s = __dadd_rn(s, smem[w]);
    __syncthreads();
    return s;                            // valid in thread 0
}

// one CTA per group: thread t takes variables lo + t, lo + t + 256, ... of the group
template <class F>
__global__ void __launch_bounds__(kThreads) map_group_kernel(F f, nlopt_b200_shard sh, const double *x, double *grad, double *partials)
{
    __shared__ double smem[kThreads / 32];
    const unsigned g = sh.group0 + blockIdx.x;
    const unsigned long long c_lo = (unsigned long long) g * sh.nchunks / sh.groups_total - sh.chunk0;
    const unsigned long long c_hi = (unsigned long long) (g + 1) * sh.nchunks / sh.groups_total - sh.chunk0;
    long long lo = (long long) (c_lo * 512), hi = (long long) (c_hi * 512);
    if (hi > (long long) sh.n_local) hi = (long long) sh.n_local;
    double acc = 0.0;
    for (long long jl = lo + threadIdx.x; jl < hi; jl += kThreads)
        acc = __dadd_rn(acc, f(sh.j0 + (unsigned long long) jl, sh.n, jl, (long long) sh.n_local, x, grad ? grad + jl : nullptr));
    const double s = block_sum(acc, smem);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

// one CTA per local virtual shard: its P group sums in a fixed order
__global__ void __launch_bounds__(kThreads) fold_groups_kernel(const double *partials, unsigned P, double *vsums /* at vshard0 */)
{
    __shared__ double smem[kThreads / 32];
    const double *base = partials + (size_t) blockIdx.x * P;
    double acc = 0.0;
    for (unsigned r = threadIdx.x; r < P; r += kThreads) acc = __dadd_rn(acc, base[r]);
    const double s = block_sum(acc, smem);
    if (threadIdx.x == 0) vsums[blockIdx.x] = s;
}

// ---- vector functors (nlopt_b200_dmfunc2): F::m components from one visit of each variable ---------------------
// map_group_mkernel is map_group_kernel with F::m accumulators per thread: the same thread->variable map, every term
// added with __dadd_rn from +0.0, and each component reduced by block_sum's tree (xor butterfly 16..1, then the 8 warp
// sums in warp order from +0.0; thread i does the final adds of component i).  So component i ends in the same bits
// as a scalar functor whose terms are component i's terms.  Group sums go out as [m][groups_local].
template <class F>
__global__ void __launch_bounds__(kThreads) map_group_mkernel(F f, nlopt_b200_shard sh, const double *x, double *grad,
                                                              long long grad_ld, double *partials)
{
    constexpr int M = F::m;
    __shared__ double smem[M][kThreads / 32];
    const unsigned g = sh.group0 + blockIdx.x;
    const unsigned long long c_lo = (unsigned long long) g * sh.nchunks / sh.groups_total - sh.chunk0;
    const unsigned long long c_hi = (unsigned long long) (g + 1) * sh.nchunks / sh.groups_total - sh.chunk0;
    long long lo = (long long) (c_lo * 512), hi = (long long) (c_hi * 512);
    if (hi > (long long) sh.n_local) hi = (long long) sh.n_local;
    double acc[M];
#pragma unroll
    for (int i = 0; i < M; ++i) acc[i] = 0.0;
    for (long long jl = lo + threadIdx.x; jl < hi; jl += kThreads) {
        double t[M];
        f(sh.j0 + (unsigned long long) jl, sh.n, jl, (long long) sh.n_local, x, t, grad ? grad + jl : nullptr, grad_ld);
#pragma unroll
        for (int i = 0; i < M; ++i) acc[i] = __dadd_rn(acc[i], t[i]);
    }
#pragma unroll
    for (int i = 0; i < M; ++i) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc[i] = __dadd_rn(acc[i], __shfl_xor_sync(0xffffffffu, acc[i], off));
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int i = 0; i < M; ++i) smem[i][threadIdx.x >> 5] = acc[i];
    }
    __syncthreads();
    if (threadIdx.x < M) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) s = __dadd_rn(s, smem[threadIdx.x][w]);
        partials[(size_t) threadIdx.x * gridDim.x + blockIdx.x] = s;
    }
}

// fold_groups_kernel for every row: CTA (v, i) folds the P group sums of local virtual shard v of row i in the same
// fixed order; row i of the partials starts at partials + i * groups_local, of the sums at vsums + 8 i
__global__ void __launch_bounds__(kThreads) fold_groups_mkernel(const double *partials, unsigned groups_local, unsigned P,
                                                                double *vsums /* row 0 at vshard0 */)
{
    __shared__ double smem[kThreads / 32];
    const double *base = partials + (size_t) blockIdx.y * groups_local + (size_t) blockIdx.x * P;
    double acc = 0.0;
    for (unsigned r = threadIdx.x; r < P; r += kThreads) acc = __dadd_rn(acc, base[r]);
    const double s = block_sum(acc, smem);
    if (threadIdx.x == 0) vsums[(size_t) blockIdx.y * 8 + blockIdx.x] = s;
}

template <class F, class = void>
struct halo_of { static constexpr int value = 0; };
template <class F>
struct halo_of<F, decltype((void) F::halo)> { static constexpr int value = F::halo; };

// components of a vector functor (F::m), 0 for a scalar functor
template <class F, class = void>
struct m_of { static constexpr int value = 0; };
template <class F>
struct m_of<F, decltype((void) F::m)> { static constexpr int value = F::m; };

}  // namespace detail

}  // namespace nlopt_b200
