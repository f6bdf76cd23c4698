// nlopt_b200_device.cuh -- supply the objective / constraints as __device__ code.
//
// NLopt's callbacks (src/api/nlopt.h:60-62) are host functions reading x and writing the gradient
// in host memory.  For the GPU path that means one D2H of x and one H2D per gradient row per
// inner iteration.  This header removes the trip: a user functor with a __device__ operator() is
// instantiated into a map + fixed-tree-reduce kernel in the USER's translation unit and registered
// through the plain C entry points nlopt_b200_set_min_objective_device /
// nlopt_b200_add_inequality_constraint_device (include/nlopt_b200.h).
//
// Functor concept (separable-sum functions  F(x) = finish( sum_j term_j )):
//
//   struct MyF {
//       // value contribution of variable j and d F / d x_j (write iff grad_j != nullptr).
//       // x points at this rank's shard; jl is the index inside it, j = j0 + jl the global index,
//       // n_local the shard length, n the global length.  A functor that declares
//       //     static constexpr int halo = 1;
//       // may also read x[jl-1] and x[jl+1] for every variable whose global neighbour exists (j > 0, j + 1 < n):
//       // with several ranks the library fills the cells x[-1] and x[n_local] from the neighbouring ranks.
//       __device__ double operator()(unsigned long long j, unsigned long long n, long long jl,
//                                    long long n_local, const double *x, double *grad_j) const;
//       // optional constant / scaling applied once to the global sum on the host
//       double finish(double sum) const { return sum; }
//   };
//
// Usage:   nlopt_b200::set_min_objective(opt, &functor);     // functor must outlive opt
//          nlopt_b200::set_max_objective(opt, &functor);     // maximise: the library negates value and gradient
//          nlopt_b200::add_inequality_constraint(opt, &cfunctor, tol);
//          nlopt_b200::add_equality_constraint(opt, &hfunctor, tol);      // NLOPT_AUGLAG* only
//
// Vector functors: m constraint rows from one visit of each variable (nlopt_b200_dmfunc2), e.g. local volumes:
//
//   struct LocalVolumes {
//       static constexpr int m = 4;                     // 1 <= m <= 16
//       static constexpr int halo = 0;                  // optional, as for scalar functors
//       // terms of variable j for the m components into t[0..m-1]; if grad != nullptr, d c_i / d x_j into
//       // grad[i * grad_ld] (grad already points at variable jl of row 0)
//       __device__ void operator()(unsigned long long j, unsigned long long n, long long jl, long long n_local,
//                                  const double *x, double *t, double *grad, long long grad_ld) const;
//       void finish(const double *totals, double *c) const;   // host: c[i] from the m global totals
//   };
//   nlopt_b200::add_inequality_mconstraint(opt, &f, tol /* F::m doubles or nullptr */);
//   nlopt_b200::add_equality_mconstraint(opt, &f, tol);            // NLOPT_AUGLAG* only
//
// Component i is reduced in exactly the scalar order, so it has the same bits as a scalar functor whose terms are
// component i's terms; the m components cost one map + fold launch pair instead of m.
//
// The reduction is deterministic AND independent of the number of ranks: the variables are cut into the library's
// groups and 8 virtual shards (a function of n alone, nlopt_b200_shard_geometry); one CTA reduces one group with a
// fixed thread->variable map and a fixed shuffle / shared-memory tree, a second kernel folds the group sums of each
// virtual shard in a fixed order, and the library adds the 8 shard sums of all ranks in index order -- all in un-fused
// IEEE double adds.  Nothing synchronises the host per function: the callbacks of a point are enqueued back to back
// and the library collects all values with one copy (nlopt_b200_dfunc2, include/nlopt_b200.h).
#pragma once

#include <cuda_runtime.h>

#include "nlopt_b200_device_kernels.cuh"

namespace nlopt_b200 {

namespace detail {

constexpr int kBlocks = 1056;            // 8 CTAs per SM on a 132-SM H100

struct Workspace {
    double *partials = nullptr;          // [kBlocks]
    unsigned *ticket = nullptr;
    double *result_host = nullptr;       // pinned
    double *result_dev = nullptr;
};

inline Workspace &workspace()
{
    static Workspace w;
    if (!w.partials) {
        cudaMalloc(&w.partials, kBlocks * sizeof(double));
        cudaMalloc(&w.ticket, sizeof(unsigned));
        cudaMemset(w.ticket, 0, sizeof(unsigned));
        cudaMalloc(&w.result_dev, sizeof(double));
        cudaHostAlloc(&w.result_host, sizeof(double), cudaHostAllocDefault);
        // the memset runs on the legacy default stream, which does not order work on a non-blocking stream (the
        // library's): let it complete before the first map_reduce_kernel reads the ticket
        cudaDeviceSynchronize();
    }
    return w;
}

template <class F>
__global__ void __launch_bounds__(kThreads) map_reduce_kernel(F f, unsigned long long j0, unsigned long long n,
                                                              long long n_local, const double *x, double *grad,
                                                              double *partials, unsigned *ticket, double *result)
{
    __shared__ double smem[kThreads / 32];
    __shared__ int last;
    // contiguous chunk per block, so the summation order is a function of n_local only
    const long long per = (n_local + gridDim.x - 1) / gridDim.x;
    const long long lo = (long long) blockIdx.x * per;
    long long hi = lo + per;
    if (hi > n_local) hi = n_local;
    double acc = 0.0;
    for (long long jl = lo + threadIdx.x; jl < hi; jl += kThreads)
        acc = __dadd_rn(acc, f(j0 + (unsigned long long) jl, n, jl, n_local, x, grad ? grad + jl : nullptr));
    const double s = block_sum(acc, smem);
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    acc = 0.0;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += kThreads) acc = __dadd_rn(acc, __ldcg(partials + b));
    const double total = block_sum(acc, smem);
    if (threadIdx.x == 0) {
        *result = total;
        *ticket = 0;
    }
}

template <class F>
double evaluate(const F &f, unsigned n_local, unsigned long long j0, unsigned long long n, const double *x_dev,
                double *grad_dev, cudaStream_t s)
{
    Workspace &w = workspace();
    map_reduce_kernel<F><<<kBlocks, kThreads, 0, s>>>(f, j0, n, (long long) n_local, x_dev, grad_dev, w.partials,
                                                      w.ticket, w.result_dev);
    cudaMemcpyAsync(w.result_host, w.result_dev, sizeof(double), cudaMemcpyDeviceToHost, s);
    cudaStreamSynchronize(s);
    return *w.result_host;
}

// ---- asynchronous, rank-count-independent form (nlopt_b200_dfunc2) ---------------------------------------------
struct Workspace2 {
    double *partials = nullptr;
    unsigned cap = 0;
};
inline double *partials2(unsigned groups)
{
    static Workspace2 w;
    if (groups > w.cap) {
        if (w.partials) cudaFree(w.partials);
        w.cap = groups + 64;
        cudaMalloc(&w.partials, (size_t) w.cap * sizeof(double));
    }
    return w.partials;
}

template <class F>
void mtrampoline2(unsigned /* = F::m, registered by the front ends below */, const nlopt_b200_shard *sh, const double *x_dev,
                  double *grad_dev, unsigned long long grad_ld, double *vsums_dev, void *data, void *stream)
{
    const F *f = static_cast<const F *>(data);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (sh->groups_local == 0) return;
    double *part = partials2(F::m * sh->groups_local);
    map_group_mkernel<F><<<sh->groups_local, kThreads, 0, s>>>(*f, *sh, x_dev, grad_dev, (long long) grad_ld, part);
    fold_groups_mkernel<<<dim3(sh->local_vshards, F::m), kThreads, 0, s>>>(part, sh->groups_local, sh->groups_per_vshard,
                                                                           vsums_dev + sh->vshard0);
}

template <class F>
void mfinish2(unsigned, const double *totals, double *result, void *data)
{
    static_cast<const F *>(data)->finish(totals, result);
}

template <class F>
void trampoline2(const nlopt_b200_shard *sh, const double *x_dev, double *grad_dev, double *vsums_dev, void *data, void *stream)
{
    const F *f = static_cast<const F *>(data);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (sh->groups_local == 0) return;
    double *part = partials2(sh->groups_local);
    map_group_kernel<F><<<sh->groups_local, kThreads, 0, s>>>(*f, *sh, x_dev, grad_dev, part);
    fold_groups_kernel<<<sh->local_vshards, kThreads, 0, s>>>(part, sh->groups_per_vshard, vsums_dev + sh->vshard0);
}

template <class F>
double finish2(double total, void *data)
{
    return static_cast<const F *>(data)->finish(total);
}

template <class F>
struct Bound {
    const F *f;
    unsigned long long n;
};

template <class F>
double trampoline(unsigned n_local, unsigned long long j0, const double *x_dev, double *grad_dev, void *data,
                  void *stream)
{
    const Bound<F> *b = static_cast<const Bound<F> *>(data);
    const double sum = evaluate(*b->f, n_local, j0, b->n, x_dev, grad_dev, static_cast<cudaStream_t>(stream));
    // the constant of finish() must enter the cross-rank sum exactly once: rank owning j = 0 adds it
    return j0 == 0 ? b->f->finish(sum) : b->f->finish(sum) - b->f->finish(0.0);
}

}  // namespace detail

// `f` (host object holding the functor's parameters) must stay alive and unchanged while `opt` uses it.
template <class F>
nlopt_result set_min_objective(nlopt_opt opt, const F *f)
{
    return nlopt_b200_set_min_objective_device2(opt, &detail::trampoline2<F>, &detail::finish2<F>, const_cast<F *>(f),
                                                detail::halo_of<F>::value);
}

// maximise F (nlopt_b200_set_max_objective_device2): the library minimises -F and reports opt_f = F at the optimum
template <class F>
nlopt_result set_max_objective(nlopt_opt opt, const F *f)
{
    return nlopt_b200_set_max_objective_device2(opt, &detail::trampoline2<F>, &detail::finish2<F>, const_cast<F *>(f),
                                                detail::halo_of<F>::value);
}

template <class F>
nlopt_result add_inequality_constraint(nlopt_opt opt, const F *f, double tol)
{
    return nlopt_b200_add_inequality_constraint_device2(opt, &detail::trampoline2<F>, &detail::finish2<F>, const_cast<F *>(f), tol,
                                                        detail::halo_of<F>::value);
}

// h(x) = 0 within tol (the AUGLAG family): the same kernels, so the same summation order as the inequality form
template <class F>
nlopt_result add_equality_constraint(nlopt_opt opt, const F *f, double tol)
{
    return nlopt_b200_add_equality_constraint_device2(opt, &detail::trampoline2<F>, &detail::finish2<F>, const_cast<F *>(f), tol,
                                                      detail::halo_of<F>::value);
}

// F::m constraint rows from one vector functor (one pass over x, one launch pair); tol: F::m doubles or nullptr (zeros)
template <class F>
nlopt_result add_inequality_mconstraint(nlopt_opt opt, const F *f, const double *tol)
{
    static_assert(F::m >= 1 && F::m <= 16, "a vector functor has 1 to 16 components");
    return nlopt_b200_add_inequality_mconstraint_device2(opt, F::m, &detail::mtrampoline2<F>, &detail::mfinish2<F>,
                                                         const_cast<F *>(f), tol, detail::halo_of<F>::value);
}

// h_i(x) = 0 within tol[i] (the AUGLAG family)
template <class F>
nlopt_result add_equality_mconstraint(nlopt_opt opt, const F *f, const double *tol)
{
    static_assert(F::m >= 1 && F::m <= 16, "a vector functor has 1 to 16 components");
    return nlopt_b200_add_equality_mconstraint_device2(opt, F::m, &detail::mtrampoline2<F>, &detail::mfinish2<F>,
                                                       const_cast<F *>(f), tol, detail::halo_of<F>::value);
}

// the first form of the interface (one synchronous evaluation per call, nlopt_b200_dfunc), kept for callers that
// want a value right away: rank-local sums, summed over ranks by the library
template <class F>
nlopt_result set_min_objective_sync(nlopt_opt opt, const F *f)
{
    auto *b = new detail::Bound<F>{f, nlopt_get_dimension(opt)};      // lives as long as the process
    return nlopt_b200_set_min_objective_device(opt, &detail::trampoline<F>, b);
}

template <class F>
nlopt_result set_max_objective_sync(nlopt_opt opt, const F *f)
{
    auto *b = new detail::Bound<F>{f, nlopt_get_dimension(opt)};      // lives as long as the process
    return nlopt_b200_set_max_objective_device(opt, &detail::trampoline<F>, b);
}

template <class F>
nlopt_result add_inequality_constraint_sync(nlopt_opt opt, const F *f, double tol)
{
    auto *b = new detail::Bound<F>{f, nlopt_get_dimension(opt)};
    return nlopt_b200_add_inequality_constraint_device(opt, &detail::trampoline<F>, b, tol);
}

template <class F>
nlopt_result add_equality_constraint_sync(nlopt_opt opt, const F *f, double tol)
{
    auto *b = new detail::Bound<F>{f, nlopt_get_dimension(opt)};
    return nlopt_b200_add_equality_constraint_device(opt, &detail::trampoline<F>, b, tol);
}

}  // namespace nlopt_b200
