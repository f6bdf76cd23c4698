// backend.hpp -- the seam between the host-side CCSA driver and whatever holds the
// n-dimensional state.
//
// The driver (ccsa_driver.cpp) restates the outer/inner loop of the reference
// (src/algs/mma/mma.c:145-452, ccsa_quadratic.c:211-606) on scalars only.  Every O(n)
// array of that loop -- x, bounds, sigma, the gradients, xcur/xprev/xprevprev -- lives behind
// this interface.  The product implementation is DeviceBackend (device_backend.cu: HBM-resident
// arrays, CUDA kernels).  There is no CPU implementation in the product; tests/ build their own
// (oracle-backed) one to exercise the driver logic on a machine without a GPU.
#pragma once

#include <string>

namespace nb200 {

enum Variant { kMMA = 0, kCCSAQ = 1 };

// where a user-function evaluation reads x and deposits its gradient
enum Slot {
    kBase = 0,       // the accepted point x           -> grad_f / grad_c
    kCandidate = 1   // the trial point xcur = x*(y)   -> grad_f_cur / grad_c_cur
};

// scalars one dual evaluation reads besides y (reference dual_data: fval, rho, fcval, rhoc)
struct DualScalars {
    double fval = 0, rho = 0;
    const double *fcval = nullptr;   // [m]
    const double *rhoc = nullptr;    // [m]
};

// what one dual evaluation hands back: the n-term sums only; the caller adds the O(m) constants
// (fval, y_i * fcval_i ...) in the reference's order.  gc has room for m entries.
struct DualSums {
    double val = 0;    // sum_j of the `val +=` terms        (mma.c:119 / ccsa_quadratic.c:134)
    double gval = 0;   // sum_j of the `gval +=` terms       (mma.c:123 / ccsa_quadratic.c:137)
    double wval = 0;   // sum_j of the `wval +=` terms       (mma.c:125 / ccsa_quadratic.c:138)
    double *gc = nullptr;  // [m] sum_j of the `gcval[i] +=` terms (mma.c:126 / ccsa_quadratic.c:139)
};

class Backend {
public:
    virtual ~Backend() {}

    virtual unsigned n() const = 0;              // global number of variables
    virtual unsigned m() const = 0;              // total number of scalar inequality constraints
    virtual unsigned num_constraint_objects() const = 0;
    virtual unsigned constraint_dim(unsigned ic) const = 0;

    // sigma_j <- initial step / bound-derived default, floored by sigma_min (mma.c:202-210)
    virtual bool init_sigma(double sigma_min) = 0;

    // User functions.  Values come back to the host; gradients stay in the slot's buffers.
    // `seconds_in_callback` accumulates wall time spent inside user code.
    virtual bool eval_objective(Slot slot, bool want_grad, double *value) = 0;
    virtual bool eval_constraint(Slot slot, unsigned ic, unsigned row0, bool want_grad, double *values) = 0;

    // Called once after the objective and all constraints of one point have been evaluated.  A backend may have
    // returned rank-local partial values from eval_objective / eval_constraint (device callbacks on several
    // ranks); this turns them into the global values with ONE exchange.  Default: values are final already.
    virtual bool finish_evals(double *fvalue, double *cvalues)
    {
        (void) fvalue; (void) cvalues;
        return true;
    }

    // One dual evaluation for multipliers y[m] (mma.c:59-137 / ccsa_quadratic.c:79-148).
    // In the MMA flavour a NaN sc.fcval[i] switches constraint i off (mma.c:78,103,126).
    // materialize == true also stores x*(y) into xcur.
    virtual bool dual_eval(const double *y, const DualScalars &sc, bool materialize, DualSums *out) = 0;

    // Optional: the whole dual solve (mma.c:275-288: optimise y in [lo, hi] from the warm start, then
    // the final evaluation that materialises x*(y)) as ONE device-side operation.  `stop6` =
    // {ftol_rel, ftol_abs, xtol_rel, xtol_abs, maxeval, maxtime}.  On success y holds the solution, `out`
    // the raw sums at it, *ret the dual optimiser's nlopt_result, *nevals its evaluation count (the final
    // evaluation not included).  Backends without it return false from supports_dual_solve().
    virtual bool supports_dual_solve() const { return false; }
    virtual bool dual_solve(double *y, const double *lo, const double *hi, const double *stop6, const DualScalars &sc,
                            DualSums *out, int *ret, long *nevals)
    {
        (void) y; (void) lo; (void) hi; (void) stop6; (void) sc; (void) out; (void) ret; (void) nevals;
        return false;
    }

    // x <- xcur, gradients <- candidate gradients (mma.c:374-377); O(1) buffer swaps
    virtual void accept_candidate() = 0;

    // top of outer iteration 1: xprev <- xcur (mma.c:265)
    virtual bool first_outer() = 0;
    // End of outer iteration k (k >= 1), fused: the two L1 norms of nlopt_stop_x
    // (stop.c:98-108: sum w|xcur-xprev|, sum w|xcur|, and whether every |xcur-xprev| < xtol_abs),
    // then -- as the next iteration will need them -- the sigma update for k > 1
    // (mma.c:431-442) and the rotation xprevprev <- xprev, xprev <- xcur (mma.c:264-265).
    virtual bool end_outer(unsigned k, double sigma_min, double *dnorm, double *xnorm, bool *all_below_abs) = 0;

    // copy the accepted point to host memory (or a device pointer in device mode); values-only backends: the best point
    virtual bool fetch_x(double *x_out) = 0;

    // Values-only backends (BackendConfig::values_only: the outer loop of NLOPT_AUGLAG*) hold a point x and a best
    // point, and evaluate the functions at x with eval_objective / eval_constraint (kBase, no gradient) + finish_evals.
    // point_device(): the device array of x; a caller that overwrites it calls point_moved() before the next evaluation.
    virtual double *point_device() { return nullptr; }
    virtual void point_moved() {}
    // nlopt_stop_x between x and the best point (stop.c:98-108, the sums of end_outer), then best <- x: one pass
    virtual bool stop_x_keep(double *dnorm, double *xnorm, bool *all_below_abs)
    {
        (void) dnorm; (void) xnorm; (void) all_below_abs;
        return false;
    }
    // number of ranks the state is sharded over
    virtual int ranks() const { return 1; }

    // Collective OR of a rank-local decision (time limits): with one rank, the identity.  Every rank of a sharded
    // run calls it at the same points of the loop.
    virtual bool agree_any(bool local) { return local; }

    // implementation knobs (e.g. "time_kernels"); unknown keys return false
    virtual bool configure(const char *key, long long value) { (void) key; (void) value; return false; }

    virtual const std::string &error() const = 0;
    virtual double seconds_in_callbacks() const = 0;
};

}  // namespace nb200
