// ccsa_driver.cpp -- the CCSA trust-region loop, host side, on scalars only.
//
// Restates the control flow of the reference's mma_minimize / ccsa_quadratic_minimize
// (src/algs/mma/mma.c:145-452, src/algs/mma/ccsa_quadratic.c:211-606, pre == NULL branch).
// The two reference files differ only in (i) the dual evaluation formula, (ii) MMA's
// "NaN constraint value = inactive constraint" rule and (iii) the lower sigma clamp; here one
// loop serves both and the differences are `variant` tests.  Everything O(n) is a Backend call:
// per inner iteration the device sees K dual-kernel launches (K chosen by the m-dimensional
// DualMMA below), one user evaluation and, on acceptance, pointer swaps.
#include "ccsa_driver.hpp"

#include <cmath>
#include <cstdio>

#include "dual_mma.hpp"

namespace nb200 {

namespace {

constexpr double kRhoFloor = 1e-5;   // MMA_RHOMIN (mma.c:41) == CCSA_RHOMIN (ccsa_quadratic.c:58)

enum {
    R_FAILURE = -1, R_INVALID = -2, R_FORCED = -5,
    R_SUCCESS = 1, R_STOPVAL = 2, R_FTOL = 3, R_XTOL = 4, R_MAXEVAL = 5, R_MAXTIME = 6
};

struct Loop {
    Variant variant;
    Backend &be;
    const std::vector<double> &tol;
    const StopCriteria &stop;
    const CcsaParams &prm;
    DriverStats *stats;
    std::string *err;
    double start;
    unsigned m;

    bool forced() const { return stop.force_stop && *stop.force_stop; }
    bool evals_out() const { return stop.maxeval > 0 && *stop.nevals_p >= stop.maxeval; }
    // Several ranks: every rank must take the same branch, or one returns MAXTIME while its peers wait in the next
    // exchange.  The backend turns the local clock test into a collective one (any rank over the limit => all stop).
    bool timed_out() const
    {
        if (!(stop.maxtime > 0)) return false;
        return be.agree_any(wall_seconds() - start >= stop.maxtime);
    }
    // MMA only: a NaN constraint value means "constraint switched off" (mma.c:141-143)
    bool off(double c) const { return variant == kMMA && std::isnan(c); }

    int fail(const char *what)
    {
        if (err) *err = std::string(what) + ": " + be.error();
        return R_FAILURE;
    }

    // termination tests shared by the top of the outer loop and the end of each inner
    // iteration (mma.c:258-262, :394-399)
    int poll(bool feasible, double minf) const
    {
        if (forced()) return R_FORCED;
        if (evals_out()) return R_MAXEVAL;
        if (timed_out()) return R_MAXTIME;
        if (feasible && minf < stop.minf_max) return R_STOPVAL;
        return R_SUCCESS;
    }

    // all constraint objects at one slot; values into c[0..m)
    int eval_constraints(Slot slot, bool want_grad, double *c)
    {
        unsigned row = 0;
        for (unsigned ic = 0; ic < be.num_constraint_objects(); ++ic) {
            if (!be.eval_constraint(slot, ic, row, want_grad, c + row)) return fail("constraint evaluation");
            row += be.constraint_dim(ic);
            if (forced()) return R_FORCED;
        }
        return R_SUCCESS;
    }
};

}  // namespace

int ccsa_minimize(Variant variant, Backend &be, const std::vector<double> &tol, double *minf,
                  const StopCriteria &stop, const CcsaParams &prm, DriverStats *stats, std::string *errmsg)
{
    const unsigned m = be.m();
    Loop L{variant, be, tol, stop, prm, stats, errmsg, stop.start >= 0 ? stop.start : wall_seconds(), m};
    const bool is_mma = variant == kMMA;
    const char *tag = is_mma ? "MMA" : "CCSA";

    std::vector<double> c(m), c_cur(m), rhoc(m, prm.rho_init), gc(m), sums(m), y(m, 0.0), ylo(m, 0.0),
        yhi(m, HUGE_VAL);
    DualMMA dual(m);
    double rho = prm.rho_init;
    int ret = R_SUCCESS;

    if (!be.init_sigma(prm.sigma_min)) return L.fail("sigma initialisation");

    // ---- first evaluation at the starting point, with gradients (mma.c:218-233) ----
    double fbase, fcur;
    if (!be.eval_objective(kBase, true, &fbase)) return L.fail("objective evaluation");
    ++*stop.nevals_p;
    if (L.forced()) return R_FORCED;
    if ((ret = L.eval_constraints(kBase, true, c.data())) != R_SUCCESS) return ret;
    if (!be.finish_evals(&fbase, c.data())) return L.fail("function value exchange");
    fcur = *minf = fbase;
    bool feasible = true;
    double infeas = 0;
    for (unsigned i = 0; i < m; ++i) {
        feasible = feasible && (c[i] <= 0 || L.off(c[i]));
        if (c[i] > infeas) infeas = c[i];
    }
    if (!feasible)                                   // mma.c:245-246: finite cap on the multipliers
        for (unsigned i = 0; i < m; ++i) yhi[i] = 1e40;

    // ---- one dual evaluation = one kernel launch + the O(m) constants added on the host ----
    DualScalars sc;
    sc.fcval = c.data();
    sc.rhoc = rhoc.data();
    DualSums raw;
    raw.gc = sums.data();
    double g0 = 0, w = 0;            // approximant values at the latest x*(y)
    long long launches = 0;
    // the O(m) constants around the n-term sums of one evaluation, in the reference's order
    auto assemble = [&](const double *yy, double *grad) -> double {
        double val = fbase;                                    // mma.c:75-78
        for (unsigned i = 0; i < m; ++i) {
            const double ci = L.off(c[i]) ? 0.0 : c[i];
            val += yy[i] * ci;
            gc[i] = ci + raw.gc[i];
        }
        val += raw.val;
        g0 = fbase + raw.gval;
        w = raw.wval;
        if (grad)
            for (unsigned i = 0; i < m; ++i) grad[i] = -gc[i];  // mma.c:135
        return -val;
    };
    auto dual_value = [&](const double *yy, double *grad, bool materialize, bool *ok) -> double {
        sc.fval = fbase;
        sc.rho = rho;
        if (!be.dual_eval(yy, sc, materialize, &raw)) { *ok = false; return 0.0; }
        ++launches;
        return assemble(yy, grad);
    };
    bool fused = prm.fused_solve && m > 0 && be.supports_dual_solve();
    const bool model = variant == kCCSAQ && be.solves_model();     // preconditioned CCSAQ: a model solve per inner iteration

    if (!be.first_outer()) return L.fail("state rotation");
    unsigned k = 0;
    for (;;) {                                       // ---- outer iterations (mma.c:255) ----
        const double fprev = fcur;
        if ((ret = L.poll(feasible, *minf)) != R_SUCCESS) return ret;
        ++k;
        if (stats) ++stats->outer_iters;
        int inner_nevals = 0;

        for (;;) {                                   // ---- inner iterations (mma.c:267) ----
            // dual solve, warm-started from the previous multipliers (mma.c:275-288)
            launches = 0;
            bool ok = true;
            const double t_dual0 = wall_seconds();
            if (model) {
                // the nested solve of the preconditioned model (ccsa_quadratic.c:441-467); its result as on :455-463
                Backend::ModelStop ms;
                ms.ftol_rel = prm.dual_ftol_rel;
                ms.ftol_abs = prm.dual_ftol_abs;
                ms.maxeval = prm.dual_maxeval;
                if (stop.maxtime > 0) {
                    const double left = stop.maxtime - (wall_seconds() - L.start);
                    ms.maxtime = left > 0 ? left : 1e-9;
                }
                ms.force_stop = stop.force_stop;
                sc.fval = fbase;
                sc.rho = rho;
                int reti = 0;
                if (!be.model_solve(sc, ms, &g0, gc.data(), &w, &reti, &launches)) return L.fail("model solve");
                if (reti < 0 || reti == R_MAXTIME) {
                    if (reti < 0 && errmsg) *errmsg = "nested model solve: " + be.error();
                    return L.forced() ? R_FORCED : reti;
                }
            } else if (fused) {
                // the whole dual solve + final evaluation as one persistent kernel (SURVEY.md 8(f)-1)
                const double stop6[6] = {prm.dual_ftol_rel, prm.dual_ftol_abs, prm.dual_xtol_rel, prm.dual_xtol_abs,
                                         (double) prm.dual_maxeval, stop.maxtime - (wall_seconds() - L.start)};
                sc.fval = fbase;
                sc.rho = rho;
                int reti = 0;
                long dn = 0;
                if (!be.dual_solve(y.data(), ylo.data(), yhi.data(), stop6, sc, &raw, &reti, &dn)) {
                    if (be.supports_dual_solve()) return L.fail("dual solve");
                    fused = false;                                // persistent kernel unavailable: host-driven from now on
                    continue;                                     // redo this inner iteration's dual solve
                }
                if (reti < 0 || reti == R_MAXTIME) {              // mma.c:283-286
                    if (reti == kRetInvalid && errmsg) *errmsg = "dual variables left their box";
                    if (reti == kRetFailure) return L.fail("dual solve");
                    return reti;
                }
                launches = dn + 1;
                assemble(y.data(), nullptr);
            } else if (m > 0) {
                DualStop ds;
                ds.ftol_rel = prm.dual_ftol_rel;
                ds.ftol_abs = prm.dual_ftol_abs;
                ds.xtol_rel = prm.dual_xtol_rel;
                ds.xtol_abs = prm.dual_xtol_abs;
                ds.maxeval = prm.dual_maxeval;
                ds.maxtime = stop.maxtime - (wall_seconds() - L.start);   // mma.c:278-281
                double dmin;
                long dn;
                const int reti = dual.solve(
                    [&](const double *yy, double *grad, bool *okp) { return dual_value(yy, grad, false, okp); },
                    y.data(), ylo.data(), yhi.data(), ds, &dmin, &dn);
                if (reti < 0 || reti == R_MAXTIME) {              // mma.c:283-286
                    if (reti == kRetFailure) return L.fail("dual evaluation");
                    if (reti == kRetInvalid && errmsg) *errmsg = "dual variables left their box";
                    return reti;
                }
            }
            if (!fused && !model) {
                dual_value(y.data(), nullptr, true, &ok);         // mma.c:288: x*(y), g, w at the solution
                if (!ok) return L.fail("dual evaluation");
            }
            if (stats) {
                stats->dual_evals += launches;
                ++stats->dual_solves;
                stats->seconds_dual += wall_seconds() - t_dual0;
            }
            const double t_eval0 = wall_seconds();
            if (prm.verbosity) {
                std::printf("%s dual converged in %lld iterations to g=%g:\n", tag, launches, g0);
                for (unsigned i = 0; i < m && i < (unsigned) prm.verbosity && !model; ++i)
                    std::printf("    %s y[%u]=%g, gc[%u]=%g\n", tag, i, y[i], i, gc[i]);
            }

            // candidate evaluation (mma.c:297-326)
            if (!be.eval_objective(kCandidate, prm.inner_gradients != 0, &fcur)) return L.fail("objective evaluation");
            ++*stop.nevals_p;
            ++inner_nevals;
            if (L.forced()) return R_FORCED;
            if ((ret = L.eval_constraints(kCandidate, prm.inner_gradients != 0, c_cur.data())) != R_SUCCESS) return ret;
            if (!be.finish_evals(&fcur, c_cur.data())) return L.fail("function value exchange");
            if (stats) stats->seconds_eval += wall_seconds() - t_eval0;
            bool feasible_cur = true, inner_done = g0 >= fcur, new_infeasible = false;
            double infeas_cur = 0;
            auto classify = [&](bool touch_inner_done) {
                feasible_cur = true;
                infeas_cur = 0;
                new_infeasible = false;
                for (unsigned i = 0; i < m; ++i) {
                    if (L.off(c_cur[i])) continue;
                    feasible_cur = feasible_cur && c_cur[i] <= tol[i];
                    if (!L.off(c[i])) {
                        if (touch_inner_done) inner_done = inner_done && gc[i] >= c_cur[i];
                    } else if (c_cur[i] > 0)
                        new_infeasible = true;                    // mma.c:321-322 (MMA only)
                    if (c_cur[i] > infeas_cur) infeas_cur = c_cur[i];
                }
            };
            classify(true);
            inner_done = inner_done || (prm.inner_maxeval > 0 && inner_nevals == prm.inner_maxeval);

            // acceptance (mma.c:334-392)
            const bool take = prm.always_improve
                ? ((fcur < *minf && (inner_done || feasible_cur || !feasible)) || (!feasible && infeas_cur < infeas))
                : inner_done;
            if (take) {
                if (prm.verbosity && !feasible_cur) std::printf("%s - using infeasible point?\n", tag);
                if (!prm.inner_gradients) {
                    // gradients are needed now; evaluation count is left alone (mma.c:339-370)
                    if (!be.eval_objective(kCandidate, true, &fcur)) return L.fail("objective evaluation");
                    if (!be.finish_evals(&fcur, nullptr)) return L.fail("function value exchange");
                    if (L.forced()) return R_FORCED;
                    if (is_mma) inner_done = g0 >= fcur;          // mma.c:346 (absent in ccsa_quadratic.c)
                    if ((ret = L.eval_constraints(kCandidate, true, c_cur.data())) != R_SUCCESS) return ret;
                    if (!be.finish_evals(nullptr, c_cur.data())) return L.fail("function value exchange");
                    classify(false);
                }
                fbase = *minf = fcur;
                infeas = infeas_cur;
                c = c_cur;
                be.accept_candidate();
                if (infeas_cur == 0) {                            // mma.c:384-390
                    if (!feasible) yhi.assign(m, HUGE_VAL);
                    feasible = true;
                } else if (new_infeasible)
                    feasible = false;
            }
            if ((ret = L.poll(feasible, *minf)) != R_SUCCESS) return ret;
            if (inner_done) break;

            // the approximants were not conservative: raise the penalties (mma.c:403-410)
            if (fcur > g0) {
                const double a = 10 * rho, b = 1.1 * (rho + (fcur - g0) / w);
                rho = a < b ? a : b;
            }
            for (unsigned i = 0; i < m; ++i)
                if (!L.off(c_cur[i]) && c_cur[i] > gc[i]) {
                    const double a = 10 * rhoc[i], b = 1.1 * (rhoc[i] + (c_cur[i] - gc[i]) / w);
                    rhoc[i] = a < b ? a : b;
                }
            if (prm.verbosity) {
                std::printf("%s inner iteration: rho -> %g\n", tag, rho);
                for (unsigned i = 0; i < m && i < (unsigned) prm.verbosity; ++i)
                    std::printf("                 %s rhoc[%u] -> %g\n", tag, i, rhoc[i]);
            }
        }

        // convergence tests; the x test wins when both fire (mma.c:418-422).  The fused
        // end-of-iteration pass also prepares sigma / xprev / xprevprev for iteration k+1.
        double dnorm, xnorm;
        bool below_abs;
        const double t_glue0 = wall_seconds();
        if (!be.end_outer(k, prm.sigma_min, &dnorm, &xnorm, &below_abs)) return L.fail("end-of-iteration pass");
        if (stats) stats->seconds_glue += wall_seconds() - t_glue0;
        if (rel_stop(fprev, fcur, stop.ftol_rel, stop.ftol_abs)) ret = R_FTOL;
        if (dnorm < stop.xtol_rel * xnorm || (stop.has_xtol_abs && below_abs)) ret = R_XTOL;   // stop.c:98-108
        if (ret != R_SUCCESS) return ret;

        rho = 0.1 * rho > kRhoFloor ? 0.1 * rho : kRhoFloor;      // mma.c:425-429
        for (unsigned i = 0; i < m; ++i) rhoc[i] = 0.1 * rhoc[i] > kRhoFloor ? 0.1 * rhoc[i] : kRhoFloor;
        if (prm.verbosity) std::printf("%s outer iteration: rho -> %g\n", tag, rho);
    }
}

}  // namespace nb200
