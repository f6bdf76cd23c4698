// backend_factory.hpp -- how the API layer obtains the n-dimensional state holder.
// The product links device_backend.cu (CUDA, sm_90a).  Nothing else implements this in
// libnlopt_b200.so; if no CUDA device is usable make_backend fails with a message and
// nlopt_optimize returns NLOPT_FAILURE -- there is deliberately no CPU path.
#pragma once

#include <string>
#include <vector>

#include "../../include/nlopt_b200.h"
#include "backend.hpp"

namespace nb200 {

// one user function: exactly one of f / mf / df is set
struct FuncSpec {
    unsigned m = 1;
    nlopt_func f = nullptr;
    nlopt_mfunc mf = nullptr;
    nlopt_b200_dfunc df = nullptr;
    nlopt_b200_dfunc2 df2 = nullptr;         // asynchronous device callback (takes precedence over df) ...
    nlopt_b200_dfinish dfin = nullptr;       // ... and its host-side finish
    nlopt_b200_dmfunc2 dmf2 = nullptr;       // vector asynchronous device callback, m rows (constraints only) ...
    nlopt_b200_dmfinish dmfin = nullptr;     // ... and its host-side finish of the m totals
    nlopt_b200_dtfunc dtf = nullptr;         // per-variable terms, m rows, reduced by the library; finish in dfin, or in
                                             // dmfin for the vector form
    int halo = 0;
    nlopt_b200_sfunc sf = nullptr;           // sharded host callback
    void *data = nullptr;
    bool negate = false;                     // objective of a maximisation (device / sharded callbacks only): the
                                             // backend minimises -f -- final value and gradient change sign

    // an asynchronous device callback: enqueued on the library stream, its value settled by finish_evals()
    bool async_device() const { return df2 || dmf2 || dtf; }
};

// The augmented-Lagrangian objective of NLOPT_AUGLAG* (src/algs/auglag/auglag.c:25-65), evaluated by the backend:
//   L(x) = f(x) + rho/2 sum_k (h_k(x) + lambda_k/rho)^2 + rho/2 sum_k max(0, c_k(x) + mu_k/rho)^2
// and, where a gradient is wanted, grad L = grad f + sum_k coef_k grad(h_k | c_k) accumulated in the reference's
// order.  The caller owns the multipliers and changes them (and rho) between sub-optimisations.
struct PenaltySpec {
    std::vector<FuncSpec> eq, ineq;          // constraint objects folded into the objective
    double rho = 1.0;
    const double *lambda = nullptr;          // one per scalar equality constraint
    const double *mu = nullptr;              // one per scalar inequality constraint
    int *nevals_p = nullptr;                 // the outer object's evaluation counter (auglag.c:38)
    const int *force_stop = nullptr;         // the outer object's force-stop flag (auglag.c:39)
};

// The start-point test of optimize.c:547-551 run on the device: the smallest failing index and its three values.
struct StartCheck {
    long long bad = -1;          // -1: every lb <= x <= ub
    double lb = 0, x = 0, ub = 0;
};

struct BackendConfig {
    Variant variant = kMMA;
    unsigned n = 0;                          // global problem size
    FuncSpec objective;
    const PenaltySpec *penalty = nullptr;    // non-null: `objective` is f of the augmented Lagrangian above
    std::vector<FuncSpec> constraints;       // inequality constraint objects, in registration order
    const double *lb = nullptr, *ub = nullptr;   // host, n entries
    bool lb_uniform = false, ub_uniform = false; // all entries equal lb[0] / ub[0]: fill on the device, no H2D
    // ... or device bounds (an object in device mode, one rank): copied D2D, checked against the start point on the
    // device, and read as two scalars where each array is bitwise uniform.  A failed check is reported in *start_check
    // and the set-up still succeeds; the caller ends the run.
    const double *lb_dev = nullptr, *ub_dev = nullptr;
    StartCheck *start_check = nullptr;
    const double *x0_host = nullptr;         // host start point (n entries) ...
    double *x_dev = nullptr;                 // ... or this rank's device shard (device mode, in/out)
    const double *sigma_init = nullptr;      // nlopt initial step (host) or null
    const double *x_weights = nullptr;       // host or null
    const double *xtol_abs = nullptr;        // host or null
    // ... or the same three from an object whose option is in device mode (one rank, n entries): read in place, never
    // copied or freed by the backend.  The step's uniformity and lane 0 come from the setter's check.
    const double *sigma_init_dev = nullptr;
    bool sigma_init_uniform = false;         // every lane has the bits of sigma_init0
    double sigma_init0 = 0.0;
    const double *x_weights_dev = nullptr, *xtol_abs_dev = nullptr;
    nlopt_b200_stats *stats = nullptr;       // h2d/d2h bytes, launches, kernel time
    bool values_only = false;                // x, the best point and the callback workspace only (Backend::point_device)
};

Backend *make_backend(const BackendConfig &cfg, std::string *err);

// The bounds of an nlopt_opt in device mode (nlopt_b200_set_*_bounds_device, implemented in device_backend.cu): n
// doubles each, on the device that was current at the first device setter.  The API layer reaches them through this
// interface only, so nlopt_api.cpp references no CUDA code (the host-logic tests link it without device_backend.cu).
// Methods return false with a message in *err.
class DeviceBounds {
public:
    virtual ~DeviceBounds() {}
    virtual const double *lb() const = 0;
    virtual const double *ub() const = 0;
    virtual bool download(double *lb_host, double *ub_host, std::string *err) const = 0;
    // *dst (allocated on this object's device when null) <- these values, device to device
    virtual bool copy_into(DeviceBounds **dst, std::string *err) const = 0;
    // a run may use them: one rank, and their device is the current one
    virtual bool runs_here(std::string *err) const = 0;
    // the start-point test against these bounds, for a start point in host memory or on the device (one of them)
    virtual bool check(const double *x_host, const double *x_dev, StartCheck *out, std::string *err) const = 0;
};

// One per-variable option of an nlopt_opt in device mode (xtol_abs, x_weights or the initial step, set by
// nlopt_b200_set_*_device in device_backend.cu): n doubles on the device that was current at the setter, which checked
// them with the host setter's rule.  Reached by the API layer through this interface only, as DeviceBounds.
class DeviceVector {
public:
    virtual ~DeviceVector() {}
    virtual const double *data() const = 0;
    virtual bool uniform() const = 0;        // every lane has the bits of lane0()
    virtual double lane0() const = 0;
    virtual bool download(double *host, std::string *err) const = 0;
    // *dst (allocated on this object's device when null) <- these values, device to device
    virtual bool copy_into(DeviceVector **dst, std::string *err) const = 0;
    // a run may use them: one rank, and their device is the current one
    virtual bool runs_here(std::string *err) const = 0;
};

}  // namespace nb200
