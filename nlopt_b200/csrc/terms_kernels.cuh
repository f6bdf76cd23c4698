// terms_kernels.cuh -- the library-side reduction of per-variable terms (nlopt_b200_dtfunc, include/nlopt_b200.h).
//
// A terms callback leaves term i of local variable jl at terms[i * ld + jl].  terms_group_kernel is map_group_kernel /
// map_group_mkernel of include/nlopt_b200_device.cuh with the functor call replaced by a load: CTA (g, i) reduces row i
// of local group g, thread t adds terms lo + t, lo + t + 256, ... in that order with __dadd_rn from +0.0, and the 256
// thread sums go through the header's block_sum (xor butterfly 16..1, then the 8 warp sums in warp order from +0.0).
// The group sums go out as [m][groups_local] and the header's fold_groups_mkernel folds them into the virtual-shard
// sums.  So terms that are bit-equal to a functor's terms give the functor's sums, bit for bit.  The order is the
// contract: a thread issues up to 8 loads ahead of its adds, but the adds keep their order.
//
// Bytes per callback: 8 n_local m read (the terms) + 16 groups m (the group sums, written and read once).
#pragma once

#include "../../include/nlopt_b200_device.cuh"

namespace nb200 {

constexpr int kTermsThreads = nlopt_b200::detail::kThreads;
constexpr int kTermsAhead = 8;           // loads in flight per thread

__global__ void __launch_bounds__(kTermsThreads) terms_group_kernel(const nlopt_b200_shard sh, const double *__restrict__ terms,
                                                                    unsigned long long ld, double *__restrict__ partials)
{
    __shared__ double smem[kTermsThreads / 32];
    const unsigned g = sh.group0 + blockIdx.x;
    const unsigned long long c_lo = (unsigned long long) g * sh.nchunks / sh.groups_total - sh.chunk0;
    const unsigned long long c_hi = (unsigned long long) (g + 1) * sh.nchunks / sh.groups_total - sh.chunk0;
    long long lo = (long long) (c_lo * 512), hi = (long long) (c_hi * 512);
    if (hi > (long long) sh.n_local) hi = (long long) sh.n_local;
    const double *row = terms + (unsigned long long) blockIdx.y * ld;
    double acc = 0.0;
    long long jl = lo + threadIdx.x;
    for (; jl + (kTermsAhead - 1) * kTermsThreads < hi; jl += kTermsAhead * kTermsThreads) {
        double t[kTermsAhead];
#pragma unroll
        for (int k = 0; k < kTermsAhead; ++k) t[k] = __ldg(row + jl + k * kTermsThreads);
#pragma unroll
        for (int k = 0; k < kTermsAhead; ++k) acc = __dadd_rn(acc, t[k]);
    }
    for (; jl < hi; jl += kTermsThreads) acc = __dadd_rn(acc, __ldg(row + jl));
    const double s = nlopt_b200::detail::block_sum(acc, smem);
    if (threadIdx.x == 0) partials[(unsigned long long) blockIdx.y * gridDim.x + blockIdx.x] = s;
}

}  // namespace nb200
