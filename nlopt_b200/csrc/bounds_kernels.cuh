// bounds_kernels.cuh -- box bounds and per-variable options held in device memory (nlopt_b200_set_*_bounds_device,
// nlopt_b200_set_{xtol_abs,x_weights,initial_step}_device): the snap of the bound setters, the start-point check of
// nlopt_optimize and the option setters' check, as element-wise kernels.  Included by device_backend.cu only.
#pragma once

#include <cuda_runtime.h>

#include <cfloat>

namespace nb200 {

// The setters' snap (options.c:375-377 / :429-431, nlopt_istiny stop.c:230-245): a subnormally thin interval is shut.
// `b` already holds the caller's values; `other` is the opposite bound.  lower: lb <- ub where the gap is tiny, else
// ub <- lb.  Comparisons and the one subtraction are exact, so the bits equal the host setter's.
__global__ void __launch_bounds__(256) snap_bounds_kernel(double *__restrict__ b, const double *__restrict__ other,
                                                          bool lower, unsigned n)
{
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        const double v = b[i], o = other[i];
        const double lo = lower ? v : o, hi = lower ? o : v;
        const double gap = hi - lo;
        if (lo < hi && (gap == 0.0 || fabs(gap) < DBL_MIN)) b[i] = o;
    }
}

// What bounds_check_kernel hands back; the host reads it once, after the synchronisation that ends the set-up.
struct BoundsReport {
    unsigned first_bad;         // smallest i with lb > ub or x outside [lb, ub]; 0xffffffff: none
    unsigned nonuniform;        // bit 0: some lb lane's bits differ from lb[0]'s; bit 1: the same for ub
    unsigned done;              // CTAs finished (the last one fills the values below and rearms the counter)
    unsigned pad;
    double lb, x, ub;           // the three values at first_bad
    double lb0, ub0;            // lane 0: the scalars of the scalar-bounds kernels when the arrays are uniform
};

// One pass over lb, ub and the start point x: the reference's test of optimize.c:547-551 (NaN passes, as there), as a
// min-reduction of the failing index (independent of scheduling), and whether lb and ub are each bitwise uniform (value
// equality is not enough: the scalar-bounds kernels hand every lane lane 0's bits, so -0.0 next to +0.0 keeps the
// arrays).  r: first_bad = 0xffffffff, nonuniform = done = 0 on entry.
__global__ void __launch_bounds__(256) bounds_check_kernel(const double *__restrict__ lb, const double *__restrict__ ub,
                                                           const double *__restrict__ x, unsigned n, BoundsReport *r)
{
    const long long lb0 = __double_as_longlong(lb[0]), ub0 = __double_as_longlong(ub[0]);
    unsigned bad = 0xffffffffu, flags = 0;
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        const double l = lb[i], u = ub[i], xi = x[i];
        if ((l > u || xi < l || xi > u) && i < bad) bad = (unsigned) i;
        flags |= (__double_as_longlong(l) != lb0 ? 1u : 0u) | (__double_as_longlong(u) != ub0 ? 2u : 0u);
    }
    bad = __reduce_min_sync(0xffffffffu, bad);
    flags = __reduce_or_sync(0xffffffffu, flags);
    if ((threadIdx.x & 31) == 0) {
        if (bad != 0xffffffffu) atomicMin(&r->first_bad, bad);
        if (flags) atomicOr(&r->nonuniform, flags);
    }
    __syncthreads();
    __shared__ bool last;
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(&r->done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        __threadfence();
        const unsigned i = *(volatile unsigned *) &r->first_bad;
        if (i < n) {
            r->lb = lb[i];
            r->x = x[i];
            r->ub = ub[i];
        }
        r->lb0 = lb[0];
        r->ub0 = ub[0];
        r->done = 0;
    }
}

// The rule of a per-variable option's host setter (options.c): x_weights refuse a negative entry, the initial step a
// zero one (+0.0 or -0.0); xtol_abs takes any value.  NaN passes every rule, as on the host.
enum OptionRule : int { kAnyValue = 0, kNoNegative = 1, kNoZero = 2 };

// What option_check_kernel hands back; the host reads it once, with the synchronisation that ends the setter.
struct OptionReport {
    unsigned flags;             // bit 0: some lane fails the rule; bit 1: some lane's bits differ from lane 0's
    unsigned done;              // CTAs finished (the last one fills v0 and rearms the counter)
    double v0;                  // lane 0: sigma_0 of the sigma palette when the initial step is uniform
};

// One pass over a per-variable option v (nlopt_b200_set_{x_weights,initial_step,xtol_abs}_device): whether any lane
// fails the setter's rule, and whether every lane has the bits of lane 0 (a -0.0 next to +0.0 is not uniform: a uniform
// step hands every lane lane 0's bits, as nlopt_set_initial_step1 does).  r: flags = done = 0 on entry.
__global__ void __launch_bounds__(256) option_check_kernel(const double *__restrict__ v, unsigned n, int rule,
                                                           OptionReport *r)
{
    const long long b0 = __double_as_longlong(v[0]);
    unsigned flags = 0;
    for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
        const double x = v[i];
        const bool bad = (rule == kNoNegative && x < 0.0) || (rule == kNoZero && x == 0.0);
        flags |= (bad ? 1u : 0u) | (__double_as_longlong(x) != b0 ? 2u : 0u);
    }
    flags = __reduce_or_sync(0xffffffffu, flags);
    if ((threadIdx.x & 31) == 0 && flags) atomicOr(&r->flags, flags);
    __syncthreads();
    __shared__ bool last;
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(&r->done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        r->v0 = v[0];
        r->done = 0;
    }
}

}  // namespace nb200
