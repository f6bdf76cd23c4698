// dual_mma.hpp -- the m-dimensional dual optimiser (m is tiny).
//
// In the reference the dual problem  max_{y >= 0} g(y)  is handed to a second nlopt object
// whose algorithm is again NLOPT_LD_MMA (src/api/optimize.c:818-826, deprecated.c:27), i.e. the
// same mma_minimize runs one level down with n' = m variables and m' = 0 constraints, and ITS
// dual problem has dimension 0, which nlopt_optimize_ short-circuits to a single evaluation
// (optimize.c:536-539) -- the closed-form MMA step.
//
// This file states that two-level recursion directly for the m' = 0 case, as an explicit state
// machine (`DualMachine`): the caller evaluates F(trial()) -- one launch of the n-dimensional dual
// kernel -- and feeds the value and gradient back; the machine answers with the next trial point
// or with a result code.  This is the HOST form (any m; DualMMA::solve drives it, one kernel launch per
// evaluation).  The persistent dual-solve kernel carries the same algorithm as a warp-parallel,
// register-resident machine (WarpDualMachine, ccsa_kernels.cuh: lane i owns multiplier i) that performs the
// same IEEE operations in the same order.  Both are replayed on the reference's own trajectories, bit for bit:
// tests/test_dual_machine.py (this file) and tests/test_dual_machine_gpu.py (the warp form).
//   DualMachine::feed  = mma.c:145-452 specialised to "no constraints, always feasible"
//   DualMachine::step  = mma.c:59-137 with m = 0 (the level-3 evaluation)
#pragma once

#include <chrono>
#include <cmath>
#include <vector>

#ifdef __CUDACC__
#define NB_HD __host__ __device__
#else
#define NB_HD
using std::fabs;
using std::isinf;
using std::sqrt;
#endif

namespace nb200 {


inline double wall_seconds()
{
    using clk = std::chrono::steady_clock;
    static const clk::time_point t0 = clk::now();
    return std::chrono::duration<double>(clk::now() - t0).count();
}

// nlopt_isinf (stop.c:219-228): also treats |x| >= 0.99 HUGE_VAL as infinite
NB_HD inline bool nl_isinf(double x) { return fabs(x) >= HUGE_VAL * 0.99 || isinf(x); }

// relstop (stop.c:81-86)
NB_HD inline bool rel_stop(double vold, double vnew, double reltol, double abstol)
{
    if (nl_isinf(vold)) return false;
    const double d = fabs(vnew - vold);
    return d < abstol || d < reltol * (fabs(vnew) + fabs(vold)) * 0.5 || (reltol > 0 && vnew == vold);
}

struct DualStop {              // plain aggregate (it lives in kernel parameters and shared memory)
    double ftol_rel, ftol_abs, xtol_rel, xtol_abs;   // optimize.c:822-825: defaults 1e-14, 0, 0, 0
    int maxeval;                                     // optimize.c:826: default 100000
    double maxtime;            // <= 0: unlimited (optimize.c:1104-1105 semantics already applied)
};

// return codes are nlopt_result values
enum { kRetSuccess = 1, kRetFtol = 3, kRetXtol = 4, kRetMaxeval = 5, kRetMaxtime = 6, kRetFailure = -1,
       kRetInvalid = -2 };

struct DualMachine {
    int m = 0;
    // m entries each, carved out of one block owned by the machine (no cap on m: the reference has none, mma.c:173)
    double *y = nullptr;            // accepted multipliers (in: warm start, out: result)
    double *g = nullptr;            // gradient of F at y
    double *sigma = nullptr, *ycur = nullptr, *yprev = nullptr, *yprevprev = nullptr;
    double *lo = nullptr, *hi = nullptr;
    std::vector<double> store;
    double rho, fbase, fmin, fcur, fprev, gval, wval;
    unsigned k;
    long nevals;
    int awaiting_first;             // 1: the pending evaluation is F(y) at the start point
    int ret;
    DualStop st;

    // returns kRetSuccess when an evaluation at trial() is wanted, else the final code (kRetInvalid)
    int start(int m_, const double *y0, const double *lo_, const double *hi_, const DualStop &stop)
    {
        m = m_;
        store.assign(8 * (size_t) (m > 0 ? m : 1), 0.0);
        {
            double *p = store.data();
            const size_t mm = (size_t) (m > 0 ? m : 1);
            y = p; g = p + mm; sigma = p + 2 * mm; ycur = p + 3 * mm; yprev = p + 4 * mm; yprevprev = p + 5 * mm;
            lo = p + 6 * mm; hi = p + 7 * mm;
        }
        st = stop;
        ret = kRetSuccess;
        nevals = 0;
        k = 0;
        for (int i = 0; i < m; ++i) {
            y[i] = y0[i]; lo[i] = lo_[i]; hi[i] = hi_[i];
            if (lo[i] > hi[i] || y[i] < lo[i] || y[i] > hi[i]) ret = kRetInvalid;       // optimize.c:547-551
        }
        for (int i = 0; i < m; ++i)                      // mma.c:202-210 (no initial step, sigma_min 0)
            sigma[i] = (nl_isinf(hi[i]) || nl_isinf(lo[i])) ? 1.0 : 0.5 * (hi[i] - lo[i]);
        rho = 1.0;                                       // rho_init default
        awaiting_first = 1;
        return ret;
    }

    const double *trial() const { return awaiting_first ? y : ycur; }

    // Feed F(trial()) and its gradient; `elapsed` = seconds since start().  Returns true when finished
    // (result code in ret, multipliers in y, best value in fmin).
    bool feed(double F, const double *grad, double elapsed)
    {
        if (feed_pre(F, grad, elapsed)) return true;
        step();
        return false;
    }

    // feed() without the closing step(): a warp runs step_term(i) on m lanes side by side and then
    // step_sum() on one (same operations in the same order => same bits as step()).
    bool feed_pre(double F, const double *grad, double elapsed)
    {
        if (awaiting_first) {                            // mma.c:218
            awaiting_first = 0;
            for (int i = 0; i < m; ++i) { g[i] = grad[i]; ycur[i] = y[i]; }
            fbase = fmin = fcur = F;
            nevals = 1;
            return outer_top(elapsed);
        }
        fcur = F;                                        // mma.c:297
        ++nevals;
        const bool inner_done = gval >= fcur;            // mma.c:304
        if (fcur < fmin) {                               // mma.c:334 with m' = 0: always "feasible"
            fbase = fmin = fcur;
            for (int i = 0; i < m; ++i) { y[i] = ycur[i]; g[i] = grad[i]; }
        }
        if (limits_hit(elapsed)) return true;
        if (inner_done) {
            if (outer_end()) return true;
            if (outer_top(elapsed)) return true;
        } else if (fcur > gval) {                        // mma.c:403-404
            const double a = 10 * rho, b = 1.1 * (rho + (fcur - gval) / wval);
            rho = a < b ? a : b;
        }
        return false;
    }

    // Term i of the MMA dual evaluation with zero constraints on the m dual variables (mma.c:59-137, m = 0):
    // ycur_i <- argmin of the separable approximant around y; false: sigma_i == 0, no contribution.
    bool step_term(int i, double *gterm, double *wterm)
    {
        const double s = sigma[i];
        if (s == 0) { ycur[i] = y[i]; return false; }
        double u = g[i];
        const double v = fabs(g[i]) * s + 0.5 * rho;
        const double s2 = s * s;
        u *= s2;
        const double r = u / (v * s);
        double dy = (u / v) / (-1 - sqrt(fabs(1 - r * r)));
        double yc = y[i] + dy;
        if (yc > hi[i]) yc = hi[i];
        else if (yc < lo[i]) yc = lo[i];
        if (yc > y[i] + 0.9 * s) yc = y[i] + 0.9 * s;
        else if (yc < y[i] - 0.9 * s) yc = y[i] - 0.9 * s;
        ycur[i] = yc;
        dy = yc - y[i];
        const double dy2 = dy * dy, dinv = 1.0 / (s2 - dy2), c = s2 * dy;
        *gterm = (g[i] * c + (fabs(g[i]) * s + 0.5 * rho) * dy2) * dinv;
        *wterm = 0.5 * dy2 * dinv;
        return true;
    }

    // gval / wval as at mma.c:123-125: the terms added in index order
    void step_sum(const double *gterm, const double *wterm, const int *has)
    {
        double gs = fbase, ws = 0;
        for (int i = 0; i < m; ++i)
            if (has[i]) { gs += gterm[i]; ws += wterm[i]; }
        gval = gs;
        wval = ws;
    }

private:
    bool limits_hit(double elapsed)
    {
        if (st.maxeval > 0 && nevals >= st.maxeval) ret = kRetMaxeval;       // stopval is -inf: never reached
        else if (st.maxtime > 0 && elapsed >= st.maxtime) ret = kRetMaxtime;
        return ret != kRetSuccess;
    }

    bool outer_top(double elapsed)                 // mma.c:255-265
    {
        fprev = fcur;
        if (limits_hit(elapsed)) return true;
        if (++k > 1)
            for (int i = 0; i < m; ++i) yprevprev[i] = yprev[i];
        for (int i = 0; i < m; ++i) yprev[i] = ycur[i];
        return false;
    }

    bool outer_end()                               // mma.c:418-446
    {
        if (rel_stop(fprev, fcur, st.ftol_rel, st.ftol_abs)) ret = kRetFtol;
        if (x_converged()) ret = kRetXtol;
        if (ret != kRetSuccess) return true;
        rho = 0.1 * rho > 1e-5 ? 0.1 * rho : 1e-5;
        if (k > 1)
            for (int i = 0; i < m; ++i) {
                const double osc = (ycur[i] - yprev[i]) * (yprev[i] - yprevprev[i]);
                double s = sigma[i] * (osc < 0 ? 0.7 : (osc > 0 ? 1.2 : 1));
                if (!nl_isinf(hi[i]) && !nl_isinf(lo[i])) {
                    const double top = 10 * (hi[i] - lo[i]), bot = 0.01 * (hi[i] - lo[i]);
                    s = s < top ? s : top;
                    s = s > bot ? s : bot;
                }
                sigma[i] = s > 0.0 ? s : 0.0;            // sigma_min = 0
            }
        return false;
    }

    void step()
    {
        double gs = fbase, ws = 0;
        for (int i = 0; i < m; ++i) {
            double gt, wt;
            if (step_term(i, &gt, &wt)) { gs += gt; ws += wt; }
        }
        gval = gs;
        wval = ws;
    }

    // nlopt_stop_x on (ycur, yprev) with unit weights and a uniform xtol_abs (stop.c:98-108).
    // The dual object always carries an xtol_abs array (nlopt_set_xtol_abs1, optimize.c:825).
    bool x_converged() const
    {
        double dn = 0, xn = 0;
        for (int i = 0; i < m; ++i) dn += fabs(ycur[i] - yprev[i]);
        for (int i = 0; i < m; ++i) xn += fabs(ycur[i]);
        if (dn < st.xtol_rel * xn) return true;
        for (int i = 0; i < m; ++i)
            if (fabs(ycur[i] - yprev[i]) >= st.xtol_abs) return false;
        return true;
    }
};

// Host-driven use: one call per dual solve, `eval` is called once per dual evaluation.
class DualMMA {
public:
    explicit DualMMA(unsigned m) : m_(m), grad_(m ? m : 1) {}

    // Minimise F over the box [lo, hi]^m starting from (and returning in) y.
    // eval(y, grad, &ok) -> F(y), fills grad[m]; `ok` false aborts.
    template <class Eval>
    int solve(Eval &&eval, double *y, const double *lo, const double *hi, const DualStop &st,
              double *fmin_out, long *nevals_out)
    {
        const double t0 = wall_seconds();
        int rc = mach_.start((int) m_, y, lo, hi, st);
        if (rc != kRetSuccess) return rc;
        for (;;) {
            bool ok = true;
            const double F = eval(mach_.trial(), grad_.data(), &ok);
            if (!ok) return kRetFailure;
            if (mach_.feed(F, grad_.data(), wall_seconds() - t0)) break;
        }
        for (unsigned i = 0; i < m_; ++i) y[i] = mach_.y[i];
        *fmin_out = mach_.fmin;
        *nevals_out = mach_.nevals;
        return mach_.ret;
    }

private:
    unsigned m_;
    std::vector<double> grad_;
    DualMachine mach_;
};

}  // namespace nb200
