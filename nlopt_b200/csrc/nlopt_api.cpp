// nlopt_api.cpp -- the NLopt object API (C ABI) of libnlopt_b200.so.
//
// Same names, arguments, return codes and side effects as the reference's
// src/api/options.c, src/api/general.c and the MMA/CCSAQ slice of src/api/optimize.c
// (cited per function).  The object is a C++ struct of our own; only two algorithms run.
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>

#include "backend_factory.hpp"
#include "ccsa_driver.hpp"
#include "dual_mma.hpp"
#include "nlopt_object.hpp"

using nb200::ConstraintRec;
using nb200::FuncSpec;
using nb200::NamedParam;

namespace {
/* process-wide defaults of the deprecated API (deprecated.c:27-29, :48) */
nlopt_algorithm g_local_deriv = NLOPT_LD_MMA, g_local_nonderiv = NLOPT_LN_COBYLA;
int g_local_maxeval = -1;
int g_stochastic_population = 0;
}  // namespace

namespace {

const double kInf = HUGE_VAL;

void set_err(nlopt_opt opt, const char *fmt, ...)
{
    if (!opt) return;
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    std::vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    opt->errmsg = buf;
    opt->has_errmsg = true;
}

void clear_err(nlopt_opt opt)
{
    if (opt) { opt->errmsg.clear(); opt->has_errmsg = false; }
}

// nlopt_istiny (stop.c:230-245): zero or subnormal
bool is_tiny(double x) { return x == 0.0 || std::fpclassify(x) == FP_SUBNORMAL; }

// options.c:375-377 / :429-431: a subnormally thin interval is snapped shut
void snap_lower(nlopt_opt o, unsigned i)
{
    if (o->lb[i] < o->ub[i] && is_tiny(o->ub[i] - o->lb[i])) o->lb[i] = o->ub[i];
}
void snap_upper(nlopt_opt o, unsigned i)
{
    if (o->lb[i] < o->ub[i] && is_tiny(o->ub[i] - o->lb[i])) o->ub[i] = o->lb[i];
}

// device mode: the bounds live in opt->dbounds (nlopt_b200_set_*_bounds_device)
bool device_mode(const nlopt_opt o) { return o->dbounds != nullptr; }

// Every host reader of the bounds goes through here: in device mode one download of both arrays into lb / ub, which
// stay valid until a device setter changes the device arrays; false (with a message) when the download fails.
bool host_bounds(nlopt_opt o)
{
    if (!device_mode(o) || o->lb_ub_mirror) return true;
    std::string err;
    if (!o->dbounds->download(o->lb.data(), o->ub.data(), &err)) {
        set_err(o, "%s", err.c_str());
        return false;
    }
    o->lb_ub_mirror = true;
    return true;
}

// a host setter: the device values come down, and the object continues on host arrays
bool leave_device_mode(nlopt_opt o)
{
    if (!host_bounds(o)) return false;
    delete o->dbounds;
    o->dbounds = nullptr;
    o->lb_ub_mirror = false;
    return true;
}

// a run in device mode: one rank, on the device that holds the arrays
bool device_mode_runs_here(nlopt_opt o)
{
    std::string err;
    if (o->dbounds->runs_here(&err)) return true;
    set_err(o, "%s", err.c_str());
    return false;
}

// Every host reader of a per-variable option (xtol_abs, x_weights, dx) goes through here: in device mode one download
// into the option's host vector, which stays valid until a device setter replaces the device values; false (with a
// message) when the download fails.
bool host_option(nlopt_opt o, nb200::DeviceOption &d, std::vector<double> &v)
{
    if (!d.dev || d.mirror) return true;
    v.resize(o->n);
    std::string err;
    if (!d.dev->download(v.data(), &err)) {
        set_err(o, "%s", err.c_str());
        return false;
    }
    d.mirror = true;
    return true;
}

bool host_options(nlopt_opt o)
{
    return host_option(o, o->xtol_abs_dev, o->xtol_abs) && host_option(o, o->x_weights_dev, o->x_weights) &&
           host_option(o, o->dx_dev, o->dx);
}

// a host setter of the option: the device copy goes
void leave_device_option(nb200::DeviceOption &d)
{
    delete d.dev;
    d = nb200::DeviceOption();
}

// a run with device options: one rank, on the device that holds them
bool device_options_run_here(nlopt_opt o)
{
    std::string err;
    for (const nb200::DeviceOption *d : {&o->xtol_abs_dev, &o->x_weights_dev, &o->dx_dev})
        if (d->dev && !d->dev->runs_here(&err)) {
            set_err(o, "%s", err.c_str());
            return false;
        }
    return true;
}

// to (an option of another object) <- from, device to device; `to` is then in device mode
bool copy_device_option(nlopt_opt o, const nb200::DeviceOption &from, nb200::DeviceOption &to, bool &to_has)
{
    std::string err;
    if (!from.dev->copy_into(&to.dev, &err)) {
        set_err(o, "%s", err.c_str());
        return false;
    }
    to.mirror = false;
    to_has = true;
    return true;
}

bool is_auglag(nlopt_algorithm a)
{
    return a == NLOPT_AUGLAG || a == NLOPT_AUGLAG_EQ || a == NLOPT_LN_AUGLAG || a == NLOPT_LN_AUGLAG_EQ
        || a == NLOPT_LD_AUGLAG || a == NLOPT_LD_AUGLAG_EQ;
}
// options.c:549-554
bool inequality_ok(nlopt_algorithm a)
{
    return a == NLOPT_LD_MMA || a == NLOPT_LD_CCSAQ || a == NLOPT_LD_SLSQP || a == NLOPT_LN_COBYLA || is_auglag(a)
        || a == NLOPT_GN_ISRES || a == NLOPT_GN_ORIG_DIRECT || a == NLOPT_GN_ORIG_DIRECT_L || a == NLOPT_GN_AGS;
}
// options.c:617-622
bool equality_ok(nlopt_algorithm a)
{
    return is_auglag(a) || a == NLOPT_LD_SLSQP || a == NLOPT_GN_ISRES || a == NLOPT_LN_COBYLA;
}

void munge_all(nlopt_opt o, std::vector<ConstraintRec> &v)
{
    if (o->munge_on_destroy)
        for (auto &c : v) o->munge_on_destroy(c.fn.data);
}

// options.c:504-547
nlopt_result add_constraint(nlopt_opt opt, std::vector<ConstraintRec> &list, const FuncSpec &fn, const double *tol)
{
    if (fn.empty()) return NLOPT_INVALID_ARGS;
    if (tol)
        for (unsigned i = 0; i < fn.m; ++i)
            if (tol[i] < 0) { set_err(opt, "negative constraint tolerance"); return NLOPT_INVALID_ARGS; }
    ConstraintRec r{fn, std::vector<double>(fn.m, 0.0)};
    if (tol) r.tol.assign(tol, tol + fn.m);
    try { list.push_back(r); } catch (const std::bad_alloc &) { return NLOPT_OUT_OF_MEMORY; }
    return NLOPT_SUCCESS;
}

// the record of each registration form
FuncSpec host_spec(nlopt_func f, nlopt_precond pre, void *data) { FuncSpec s; s.f = f; s.pre = pre; s.data = data; return s; }
FuncSpec host_mspec(unsigned m, nlopt_mfunc mf, void *data) { FuncSpec s; s.m = m; s.mf = mf; s.data = data; return s; }
FuncSpec device_spec(nlopt_b200_dfunc df, void *data) { FuncSpec s; s.df = df; s.data = data; return s; }
FuncSpec sharded_spec(nlopt_b200_sfunc sf, void *data) { FuncSpec s; s.sf = sf; s.data = data; return s; }
FuncSpec device2_spec(unsigned m, nlopt_b200_dfunc2 f, nlopt_b200_dmfunc2 mf, nlopt_b200_dfinish fin, nlopt_b200_dmfinish mfin,
                      void *data, int halo)
{
    FuncSpec s;
    s.m = m; s.df2 = f; s.dmf2 = mf; s.dfin = fin; s.dmfin = mfin; s.data = data; s.halo = halo;
    return s;
}
// per-variable terms: a scalar function finishes in dfin, m rows in dmfin
FuncSpec terms_spec(unsigned m, nlopt_b200_dtfunc f, nlopt_b200_dfinish fin, nlopt_b200_dmfinish mfin, void *data, int halo)
{
    FuncSpec s;
    s.m = m; s.dtf = f; s.dfin = fin; s.dmfin = mfin; s.data = data; s.halo = halo;
    return s;
}

// The argument checks of the asynchronous forms (a callback, its finish, halo 0 or 1) and of the sharded form (a
// callback).  Their entry points make them before anything else: a refusal leaves the error message and the data alone.
bool complete(const FuncSpec &s)
{
    return s.sharded() || (s.async_device() && (s.dfin || s.dmfin) && (s.halo == 0 || s.halo == 1));
}

// nlopt_eval_constraint (stop.c:178-184) of a host function
void eval_host(const FuncSpec &c, unsigned n, const double *x, double *out, double *grad)
{
    if (c.f) out[0] = c.f(n, x, grad, c.data);
    else c.mf(c.m, out, n, x, grad, c.data);
}

struct AlgInfo { const char *id; const char *desc; };
// general.c:39-98 (descriptions) and :112-160 (ids)
const AlgInfo kAlgs[NLOPT_NUM_ALGORITHMS] = {
    {"GN_DIRECT", "DIRECT (global, no-derivative)"},
    {"GN_DIRECT_L", "DIRECT-L (global, no-derivative)"},
    {"GN_DIRECT_L_RAND", "Randomized DIRECT-L (global, no-derivative)"},
    {"GN_DIRECT_NOSCAL", "Unscaled DIRECT (global, no-derivative)"},
    {"GN_DIRECT_L_NOSCAL", "Unscaled DIRECT-L (global, no-derivative)"},
    {"GN_DIRECT_L_RAND_NOSCAL", "Unscaled Randomized DIRECT-L (global, no-derivative)"},
    {"GN_ORIG_DIRECT", "Original DIRECT version (global, no-derivative)"},
    {"GN_ORIG_DIRECT_L", "Original DIRECT-L version (global, no-derivative)"},
    {"GD_STOGO", "StoGO (NOT COMPILED)"},
    {"GD_STOGO_RAND", "StoGO randomized (NOT COMPILED)"},
    {"NLOPT_LD_LBFGS_NOCEDAL", "original L-BFGS code by Nocedal et al. (NOT COMPILED)"},
    {"LD_LBFGS", "Limited-memory BFGS (L-BFGS) (local, derivative-based)"},
    {"LN_PRAXIS", "Principal-axis, praxis (local, no-derivative)"},
    {"LD_VAR1", "Limited-memory variable-metric, rank 1 (local, derivative-based)"},
    {"LD_VAR2", "Limited-memory variable-metric, rank 2 (local, derivative-based)"},
    {"LD_TNEWTON", "Truncated Newton (local, derivative-based)"},
    {"LD_TNEWTON_RESTART", "Truncated Newton with restarting (local, derivative-based)"},
    {"LD_TNEWTON_PRECOND", "Preconditioned truncated Newton (local, derivative-based)"},
    {"LD_TNEWTON_PRECOND_RESTART", "Preconditioned truncated Newton with restarting (local, derivative-based)"},
    {"GN_CRS2_LM", "Controlled random search (CRS2) with local mutation (global, no-derivative)"},
    {"GN_MLSL", "Multi-level single-linkage (MLSL), random (global, no-derivative)"},
    {"GD_MLSL", "Multi-level single-linkage (MLSL), random (global, derivative)"},
    {"GN_MLSL_LDS", "Multi-level single-linkage (MLSL), quasi-random (global, no-derivative)"},
    {"GD_MLSL_LDS", "Multi-level single-linkage (MLSL), quasi-random (global, derivative)"},
    {"LD_MMA", "Method of Moving Asymptotes (MMA) (local, derivative)"},
    {"LN_COBYLA", "COBYLA (Constrained Optimization BY Linear Approximations) (local, no-derivative)"},
    {"LN_NEWUOA", "NEWUOA unconstrained optimization via quadratic models (local, no-derivative)"},
    {"LN_NEWUOA_BOUND", "Bound-constrained optimization via NEWUOA-based quadratic models (local, no-derivative)"},
    {"LN_NELDERMEAD", "Nelder-Mead simplex algorithm (local, no-derivative)"},
    {"LN_SBPLX", "Sbplx variant of Nelder-Mead (re-implementation of Rowan's Subplex) (local, no-derivative)"},
    {"LN_AUGLAG", "Augmented Lagrangian method (local, no-derivative)"},
    {"LD_AUGLAG", "Augmented Lagrangian method (local, derivative)"},
    {"LN_AUGLAG_EQ", "Augmented Lagrangian method for equality constraints (local, no-derivative)"},
    {"LD_AUGLAG_EQ", "Augmented Lagrangian method for equality constraints (local, derivative)"},
    {"LN_BOBYQA", "BOBYQA bound-constrained optimization via quadratic models (local, no-derivative)"},
    {"GN_ISRES", "ISRES evolutionary constrained optimization (global, no-derivative)"},
    {"AUGLAG", "Augmented Lagrangian method (needs sub-algorithm)"},
    {"AUGLAG_EQ", "Augmented Lagrangian method for equality constraints (needs sub-algorithm)"},
    {"G_MLSL", "Multi-level single-linkage (MLSL), random (global, needs sub-algorithm)"},
    {"G_MLSL_LDS", "Multi-level single-linkage (MLSL), quasi-random (global, needs sub-algorithm)"},
    {"LD_SLSQP", "Sequential Quadratic Programming (SQP) (local, derivative)"},
    {"LD_CCSAQ",
     "CCSA (Conservative Convex Separable Approximations) with simple quadratic approximations (local, derivative)"},
    {"GN_ESCH", "ESCH evolutionary strategy"},
    {"GN_AGS", "AGS (NOT COMPILED)"},
};

struct ResName { int code; const char *name; };
const ResName kResults[] = {   // general.c:180-196
    {NLOPT_FAILURE, "FAILURE"}, {NLOPT_INVALID_ARGS, "INVALID_ARGS"}, {NLOPT_OUT_OF_MEMORY, "OUT_OF_MEMORY"},
    {NLOPT_ROUNDOFF_LIMITED, "ROUNDOFF_LIMITED"}, {NLOPT_FORCED_STOP, "FORCED_STOP"}, {NLOPT_SUCCESS, "SUCCESS"},
    {NLOPT_STOPVAL_REACHED, "STOPVAL_REACHED"}, {NLOPT_FTOL_REACHED, "FTOL_REACHED"},
    {NLOPT_XTOL_REACHED, "XTOL_REACHED"}, {NLOPT_MAXEVAL_REACHED, "MAXEVAL_REACHED"},
    {NLOPT_MAXTIME_REACHED, "MAXTIME_REACHED"},
};

// maximisation = minimisation of the negated function (optimize.c:969-989)
struct FlipData { nlopt_func f; void *data; };
double flipped(unsigned n, const double *x, double *grad, void *p)
{
    FlipData *d = static_cast<FlipData *>(p);
    const double v = d->f(n, x, grad, d->data);
    if (grad)
        for (unsigned i = 0; i < n; ++i) grad[i] = -grad[i];
    return -v;
}

nlopt_result run_ccsa(nlopt_opt opt, double *x_host, double *x_dev, double *minf);
nlopt_result run_ccsa_precond(nlopt_opt opt, double *x, double *minf, const nb200::CcsaParams &prm);
nlopt_result run_auglag(nlopt_opt opt, double *x_host, double *x_dev, double *minf);

}  // namespace

extern "C" {

/* ------------------------------------------------------------------ names / version */

const char *nlopt_algorithm_name(nlopt_algorithm a)
{
    if ((int) a < 0 || a >= NLOPT_NUM_ALGORITHMS) return "UNKNOWN";
    return kAlgs[a].desc;
}

const char *nlopt_algorithm_to_string(nlopt_algorithm a)
{
    if ((int) a < 0 || a >= NLOPT_NUM_ALGORITHMS) return nullptr;
    return kAlgs[a].id;
}

nlopt_algorithm nlopt_algorithm_from_string(const char *name)
{
    if (name)
        for (int i = 0; i < NLOPT_NUM_ALGORITHMS; ++i)
            if (!std::strcmp(name, kAlgs[i].id)) return (nlopt_algorithm) i;
    return (nlopt_algorithm) -1;
}

const char *nlopt_result_to_string(nlopt_result r)
{
    for (const ResName &e : kResults)
        if (e.code == (int) r) return e.name;
    return nullptr;
}

nlopt_result nlopt_result_from_string(const char *name)
{
    if (name)
        for (const ResName &e : kResults)
            if (!std::strcmp(name, e.name)) return (nlopt_result) e.code;
    return (nlopt_result) -1;
}

void nlopt_version(int *major, int *minor, int *bugfix)
{
    *major = 2; *minor = 11; *bugfix = 0;   /* ABI level of the reference this library mirrors */
}

void nlopt_srand(unsigned long) {}
void nlopt_srand_time(void) {}

/* ------------------------------------------------------------------ lifetime (options.c:36-265) */

nlopt_opt nlopt_create(nlopt_algorithm algorithm, unsigned n)
{
    if ((int) algorithm < 0 || algorithm >= NLOPT_NUM_ALGORITHMS) return nullptr;
    nlopt_opt o = new (std::nothrow) nlopt_opt_s;
    if (!o) return nullptr;
    o->algorithm = algorithm;
    o->n = n;
    o->stopval = -kInf;
    try {
        o->lb.assign(n, -kInf);
        o->ub.assign(n, +kInf);
    } catch (const std::bad_alloc &) {
        delete o;
        return nullptr;
    }
    return o;
}

void nlopt_destroy(nlopt_opt opt)
{
    if (!opt) return;
    if (opt->munge_on_destroy) {
        opt->munge_on_destroy(opt->objective.data);
        munge_all(opt, opt->fc);
        munge_all(opt, opt->h);
    }
    for (NamedParam *p : opt->params) delete p;
    nlopt_destroy(opt->local_opt);
    delete opt->dbounds;
    for (nb200::DeviceOption *d : {&opt->xtol_abs_dev, &opt->x_weights_dev, &opt->dx_dev}) delete d->dev;
    delete opt;
}

nlopt_opt nlopt_copy(const nlopt_opt opt)
{
    if (!opt) return nullptr;
    nlopt_opt c = new (std::nothrow) nlopt_opt_s(*opt);
    if (!c) return nullptr;
    c->params.clear();
    c->dbounds = nullptr;
    c->xtol_abs_dev.dev = c->x_weights_dev.dev = c->dx_dev.dev = nullptr;
    c->local_opt = nullptr;
    c->force_stop_child = nullptr;
    c->errmsg.clear();
    c->has_errmsg = false;
    for (NamedParam *p : opt->params) c->params.push_back(new NamedParam(*p));
    std::string err;
    bool copied = !device_mode(opt) || opt->dbounds->copy_into(&c->dbounds, &err);
    for (auto slot : {&nlopt_opt_s::xtol_abs_dev, &nlopt_opt_s::x_weights_dev, &nlopt_opt_s::dx_dev})
        copied = copied && (!(opt->*slot).dev || (opt->*slot).dev->copy_into(&(c->*slot).dev, &err));
    if (!copied) {
        c->munge_on_destroy = nullptr;
        nlopt_destroy(c);
        return nullptr;
    }
    if (nlopt_munge mg = c->munge_on_copy) {
        bool bad = false;
        if (c->objective.data && !(c->objective.data = mg(c->objective.data))) bad = true;
        for (auto &r : c->fc) if (!bad && r.fn.data && !(r.fn.data = mg(r.fn.data))) bad = true;
        for (auto &r : c->h) if (!bad && r.fn.data && !(r.fn.data = mg(r.fn.data))) bad = true;
        if (bad) {                       /* options.c:261-263: better to leak than to crash */
            c->munge_on_destroy = nullptr;
            nlopt_destroy(c);
            return nullptr;
        }
    }
    if (opt->local_opt && !(c->local_opt = nlopt_copy(opt->local_opt))) {
        c->munge_on_destroy = nullptr;
        nlopt_destroy(c);
        return nullptr;
    }
    return c;
}

/* ------------------------------------------------------------------ objective (options.c:322-364) */

static nlopt_result set_objective(nlopt_opt opt, const FuncSpec &fn, int maximize)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (opt->munge_on_destroy) opt->munge_on_destroy(opt->objective.data);
    opt->objective = fn;
    opt->maximize = maximize;
    if (nb200::nl_isinf(opt->stopval)) {
        if (!maximize && opt->stopval > 0) opt->stopval = -kInf;
        if (maximize && opt->stopval < 0) opt->stopval = +kInf;
    }
    return NLOPT_SUCCESS;
}
static nlopt_result set_objective_checked(nlopt_opt opt, const FuncSpec &fn, int maximize)
{ return complete(fn) ? set_objective(opt, fn, maximize) : NLOPT_INVALID_ARGS; }

nlopt_result nlopt_set_precond_min_objective(nlopt_opt opt, nlopt_func f, nlopt_precond pre, void *d)
{ return set_objective(opt, host_spec(f, pre, d), 0); }
nlopt_result nlopt_set_min_objective(nlopt_opt opt, nlopt_func f, void *d)
{ return set_objective(opt, host_spec(f, nullptr, d), 0); }
nlopt_result nlopt_set_precond_max_objective(nlopt_opt opt, nlopt_func f, nlopt_precond pre, void *d)
{ return set_objective(opt, host_spec(f, pre, d), 1); }
nlopt_result nlopt_set_max_objective(nlopt_opt opt, nlopt_func f, void *d)
{ return set_objective(opt, host_spec(f, nullptr, d), 1); }
nlopt_result nlopt_b200_set_min_objective_device(nlopt_opt opt, nlopt_b200_dfunc f, void *d)
{ return set_objective(opt, device_spec(f, d), 0); }
nlopt_result nlopt_b200_set_max_objective_device(nlopt_opt opt, nlopt_b200_dfunc f, void *d)
{ return set_objective(opt, device_spec(f, d), 1); }
nlopt_result nlopt_b200_set_min_objective_device2(nlopt_opt opt, nlopt_b200_dfunc2 f, nlopt_b200_dfinish fin, void *d, int halo)
{ return set_objective_checked(opt, device2_spec(1, f, nullptr, fin, nullptr, d, halo), 0); }
nlopt_result nlopt_b200_set_max_objective_device2(nlopt_opt opt, nlopt_b200_dfunc2 f, nlopt_b200_dfinish fin, void *d, int halo)
{ return set_objective_checked(opt, device2_spec(1, f, nullptr, fin, nullptr, d, halo), 1); }
nlopt_result nlopt_b200_set_min_objective_terms(nlopt_opt opt, nlopt_b200_dtfunc f, nlopt_b200_dfinish fin, void *d, int halo)
{ return set_objective_checked(opt, terms_spec(1, f, fin, nullptr, d, halo), 0); }
nlopt_result nlopt_b200_set_max_objective_terms(nlopt_opt opt, nlopt_b200_dtfunc f, nlopt_b200_dfinish fin, void *d, int halo)
{ return set_objective_checked(opt, terms_spec(1, f, fin, nullptr, d, halo), 1); }
nlopt_result nlopt_b200_set_min_objective_sharded(nlopt_opt opt, nlopt_b200_sfunc f, void *d)
{ return set_objective_checked(opt, sharded_spec(f, d), 0); }
nlopt_result nlopt_b200_set_max_objective_sharded(nlopt_opt opt, nlopt_b200_sfunc f, void *d)
{ return set_objective_checked(opt, sharded_spec(f, d), 1); }

/* device preconditioners (nlopt_b200_dprecond): attached to a registered record of one row that has no host one */
static nlopt_result set_dprecond(nlopt_opt opt, FuncSpec &fn, nlopt_b200_dprecond pre, void *pre_data)
{
    if (pre && fn.pre) {
        set_err(opt, "this function has a host preconditioner (nlopt_precond); a function takes one preconditioner");
        return NLOPT_INVALID_ARGS;
    }
    fn.dpre = pre;
    fn.pre_data = pre ? pre_data : nullptr;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_b200_set_objective_precond_device(nlopt_opt opt, nlopt_b200_dprecond pre, void *pre_data)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (opt->objective.empty()) { set_err(opt, "no objective registered"); return NLOPT_INVALID_ARGS; }
    return set_dprecond(opt, opt->objective, pre, pre_data);
}

nlopt_result nlopt_b200_set_constraint_precond_device(nlopt_opt opt, unsigned index, nlopt_b200_dprecond pre, void *pre_data)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (index >= opt->fc.size()) {
        set_err(opt, "inequality constraint index %u out of range (%u records; equality constraints take no preconditioner)",
                index, (unsigned) opt->fc.size());
        return NLOPT_INVALID_ARGS;
    }
    FuncSpec &fn = opt->fc[index].fn;
    if (fn.m != 1) {
        set_err(opt, "inequality constraint %u has %u rows: a vector constraint takes no preconditioner", index, fn.m);
        return NLOPT_INVALID_ARGS;
    }
    return set_dprecond(opt, fn, pre, pre_data);
}

nlopt_algorithm nlopt_get_algorithm(const nlopt_opt opt) { return opt->algorithm; }
unsigned nlopt_get_dimension(const nlopt_opt opt) { return opt->n; }
const char *nlopt_get_errmsg(nlopt_opt opt) { return opt->has_errmsg ? opt->errmsg.c_str() : nullptr; }

/* ------------------------------------------------------------------ named parameters (options.c:268-318) */

nlopt_result nlopt_set_param(nlopt_opt opt, const char *name, double val)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    if (!name) { set_err(opt, "invalid NULL parameter name"); return NLOPT_INVALID_ARGS; }
    if (strnlen(name, 1024) + 1 > 1024) { set_err(opt, "parameter name must be < 1024 bytes"); return NLOPT_INVALID_ARGS; }
    for (NamedParam *p : opt->params)
        if (p->name == name) { p->val = val; return NLOPT_SUCCESS; }
    NamedParam *p = new (std::nothrow) NamedParam{name, val};
    if (!p) return NLOPT_OUT_OF_MEMORY;
    opt->params.push_back(p);
    return NLOPT_SUCCESS;
}

double nlopt_get_param(const nlopt_opt opt, const char *name, double defaultval)
{
    if (!opt || !name || strnlen(name, 1024) == 1024) return defaultval;
    for (NamedParam *p : opt->params)
        if (p->name == name) return p->val;
    return defaultval;
}

int nlopt_has_param(const nlopt_opt opt, const char *name)
{
    if (!opt || !name || strnlen(name, 1024) == 1024) return 0;
    for (NamedParam *p : opt->params)
        if (p->name == name) return 1;
    return 0;
}

unsigned nlopt_num_params(const nlopt_opt opt) { return opt ? (unsigned) opt->params.size() : 0; }

const char *nlopt_nth_param(const nlopt_opt opt, unsigned n)
{
    return opt && n < opt->params.size() ? opt->params[n]->name.c_str() : nullptr;
}

/* ------------------------------------------------------------------ bounds (options.c:368-474) */

nlopt_result nlopt_set_lower_bounds(nlopt_opt opt, const double *lb)
{
    clear_err(opt);
    if (!opt || (opt->n > 0 && !lb)) return NLOPT_INVALID_ARGS;
    if (!leave_device_mode(opt)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) opt->lb[i] = lb[i];
    for (unsigned i = 0; i < opt->n; ++i) snap_lower(opt, i);
    opt->lb_uniform = false;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_lower_bounds1(nlopt_opt opt, double lb)
{
    clear_err(opt);
    if (!opt) return NLOPT_INVALID_ARGS;
    if (!leave_device_mode(opt)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) { opt->lb[i] = lb; snap_lower(opt, i); }
    opt->lb_uniform = true;
    for (unsigned i = 1; i < opt->n && opt->lb_uniform; ++i) opt->lb_uniform = opt->lb[i] == opt->lb[0];   // snapping may differ
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_lower_bound(nlopt_opt opt, int i, double lb)
{
    clear_err(opt);
    if (!opt) return NLOPT_INVALID_ARGS;
    if (i < 0 || i >= (int) opt->n) { set_err(opt, "invalid bound index"); return NLOPT_INVALID_ARGS; }
    if (!leave_device_mode(opt)) return NLOPT_FAILURE;
    opt->lb[i] = lb;
    snap_lower(opt, i);
    opt->lb_uniform = false;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_get_lower_bounds(const nlopt_opt opt, double *lb)
{
    clear_err(opt);
    if (!opt || (opt->n > 0 && !lb)) return NLOPT_INVALID_ARGS;
    if (!host_bounds(opt)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) lb[i] = opt->lb[i];
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_upper_bounds(nlopt_opt opt, const double *ub)
{
    clear_err(opt);
    if (!opt || (opt->n > 0 && !ub)) return NLOPT_INVALID_ARGS;
    if (!leave_device_mode(opt)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) opt->ub[i] = ub[i];
    for (unsigned i = 0; i < opt->n; ++i) snap_upper(opt, i);
    opt->ub_uniform = false;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_upper_bounds1(nlopt_opt opt, double ub)
{
    clear_err(opt);
    if (!opt) return NLOPT_INVALID_ARGS;
    if (!leave_device_mode(opt)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) { opt->ub[i] = ub; snap_upper(opt, i); }
    opt->ub_uniform = true;
    for (unsigned i = 1; i < opt->n && opt->ub_uniform; ++i) opt->ub_uniform = opt->ub[i] == opt->ub[0];
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_upper_bound(nlopt_opt opt, int i, double ub)
{
    clear_err(opt);
    if (!opt) return NLOPT_INVALID_ARGS;
    if (i < 0 || i >= (int) opt->n) { set_err(opt, "invalid bound index"); return NLOPT_INVALID_ARGS; }
    if (!leave_device_mode(opt)) return NLOPT_FAILURE;
    opt->ub[i] = ub;
    snap_upper(opt, i);
    opt->ub_uniform = false;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_get_upper_bounds(const nlopt_opt opt, double *ub)
{
    clear_err(opt);
    if (!opt || (opt->n > 0 && !ub)) return NLOPT_INVALID_ARGS;
    if (!host_bounds(opt)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) ub[i] = opt->ub[i];
    return NLOPT_SUCCESS;
}

/* ------------------------------------------------------------------ constraints (options.c:476-659) */

nlopt_result nlopt_remove_inequality_constraints(nlopt_opt opt)
{
    clear_err(opt);
    if (!opt) return NLOPT_INVALID_ARGS;
    munge_all(opt, opt->fc);
    opt->fc.clear();
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_remove_equality_constraints(nlopt_opt opt)
{
    clear_err(opt);
    if (!opt) return NLOPT_INVALID_ARGS;
    munge_all(opt, opt->h);
    opt->h.clear();
    return NLOPT_SUCCESS;
}

static nlopt_result add_any(nlopt_opt opt, bool equality, const FuncSpec &fn, const double *tol)
{
    nlopt_result ret;
    clear_err(opt);
    if (!fn.m) {                             /* options.c:560-564: an empty vector constraint is fine */
        if (opt && opt->munge_on_destroy) opt->munge_on_destroy(fn.data);
        return NLOPT_SUCCESS;
    }
    if (!opt) ret = NLOPT_INVALID_ARGS;
    else if (!(equality ? equality_ok(opt->algorithm) : inequality_ok(opt->algorithm))) {
        set_err(opt, "invalid algorithm for constraints");
        ret = NLOPT_INVALID_ARGS;
    } else
        ret = add_constraint(opt, equality ? opt->h : opt->fc, fn, tol);
    if (ret < 0 && opt && opt->munge_on_destroy) opt->munge_on_destroy(fn.data);
    return ret;
}
// the vector forms check their arguments only when m > 0 (m == 0 registers nothing)
static nlopt_result add_checked(nlopt_opt opt, bool equality, const FuncSpec &fn, const double *tol)
{ return !fn.m || complete(fn) ? add_any(opt, equality, fn, tol) : NLOPT_INVALID_ARGS; }

nlopt_result nlopt_add_inequality_mconstraint(nlopt_opt opt, unsigned m, nlopt_mfunc fc, void *d, const double *tol)
{ return add_any(opt, false, host_mspec(m, fc, d), tol); }
nlopt_result nlopt_add_precond_inequality_constraint(nlopt_opt opt, nlopt_func fc, nlopt_precond pre, void *d, double tol)
{ return add_any(opt, false, host_spec(fc, pre, d), &tol); }
nlopt_result nlopt_add_inequality_constraint(nlopt_opt opt, nlopt_func fc, void *d, double tol)
{ return add_any(opt, false, host_spec(fc, nullptr, d), &tol); }
nlopt_result nlopt_b200_add_inequality_constraint_device(nlopt_opt opt, nlopt_b200_dfunc fc, void *d, double tol)
{ return add_any(opt, false, device_spec(fc, d), &tol); }
nlopt_result nlopt_b200_add_inequality_constraint_device2(nlopt_opt opt, nlopt_b200_dfunc2 fc, nlopt_b200_dfinish fin, void *d,
                                                          double tol, int halo)
{ return add_checked(opt, false, device2_spec(1, fc, nullptr, fin, nullptr, d, halo), &tol); }
nlopt_result nlopt_b200_add_inequality_constraint_sharded(nlopt_opt opt, nlopt_b200_sfunc fc, void *d, double tol)
{ return add_checked(opt, false, sharded_spec(fc, d), &tol); }
nlopt_result nlopt_add_equality_mconstraint(nlopt_opt opt, unsigned m, nlopt_mfunc h, void *d, const double *tol)
{ return add_any(opt, true, host_mspec(m, h, d), tol); }
nlopt_result nlopt_add_precond_equality_constraint(nlopt_opt opt, nlopt_func h, nlopt_precond pre, void *d, double tol)
{ return add_any(opt, true, host_spec(h, pre, d), &tol); }
nlopt_result nlopt_add_equality_constraint(nlopt_opt opt, nlopt_func h, void *d, double tol)
{ return add_any(opt, true, host_spec(h, nullptr, d), &tol); }
nlopt_result nlopt_b200_add_equality_constraint_device(nlopt_opt opt, nlopt_b200_dfunc h, void *d, double tol)
{ return add_any(opt, true, device_spec(h, d), &tol); }
nlopt_result nlopt_b200_add_equality_constraint_device2(nlopt_opt opt, nlopt_b200_dfunc2 h, nlopt_b200_dfinish fin, void *d,
                                                        double tol, int halo)
{ return add_checked(opt, true, device2_spec(1, h, nullptr, fin, nullptr, d, halo), &tol); }
nlopt_result nlopt_b200_add_inequality_mconstraint_device2(nlopt_opt opt, unsigned m, nlopt_b200_dmfunc2 fc,
                                                           nlopt_b200_dmfinish fin, void *d, const double *tol, int halo)
{ return add_checked(opt, false, device2_spec(m, nullptr, fc, nullptr, fin, d, halo), tol); }
nlopt_result nlopt_b200_add_equality_mconstraint_device2(nlopt_opt opt, unsigned m, nlopt_b200_dmfunc2 h,
                                                         nlopt_b200_dmfinish fin, void *d, const double *tol, int halo)
{ return add_checked(opt, true, device2_spec(m, nullptr, h, nullptr, fin, d, halo), tol); }
nlopt_result nlopt_b200_add_inequality_constraint_terms(nlopt_opt opt, nlopt_b200_dtfunc fc, nlopt_b200_dfinish fin, void *d,
                                                        double tol, int halo)
{ return add_checked(opt, false, terms_spec(1, fc, fin, nullptr, d, halo), &tol); }
nlopt_result nlopt_b200_add_equality_constraint_terms(nlopt_opt opt, nlopt_b200_dtfunc h, nlopt_b200_dfinish fin, void *d,
                                                      double tol, int halo)
{ return add_checked(opt, true, terms_spec(1, h, fin, nullptr, d, halo), &tol); }
nlopt_result nlopt_b200_add_inequality_mconstraint_terms(nlopt_opt opt, unsigned m, nlopt_b200_dtfunc fc,
                                                         nlopt_b200_dmfinish fin, void *d, const double *tol, int halo)
{ return add_checked(opt, false, terms_spec(m, fc, nullptr, fin, d, halo), tol); }
nlopt_result nlopt_b200_add_equality_mconstraint_terms(nlopt_opt opt, unsigned m, nlopt_b200_dtfunc h,
                                                       nlopt_b200_dmfinish fin, void *d, const double *tol, int halo)
{ return add_checked(opt, true, terms_spec(m, h, nullptr, fin, d, halo), tol); }

/* ------------------------------------------------------------------ stopping criteria (options.c:661-816) */

#define NB_SCALAR_ACCESSORS(name, T, field)                                                   \
    T nlopt_get_##name(const nlopt_opt opt) { return opt->field; }                            \
    nlopt_result nlopt_set_##name(nlopt_opt opt, T v)                                         \
    {                                                                                         \
        if (!opt) return NLOPT_INVALID_ARGS;                                                  \
        clear_err(opt);                                                                       \
        opt->field = v;                                                                       \
        return NLOPT_SUCCESS;                                                                 \
    }
NB_SCALAR_ACCESSORS(stopval, double, stopval)
NB_SCALAR_ACCESSORS(ftol_rel, double, ftol_rel)
NB_SCALAR_ACCESSORS(ftol_abs, double, ftol_abs)
NB_SCALAR_ACCESSORS(xtol_rel, double, xtol_rel)
NB_SCALAR_ACCESSORS(maxeval, int, maxeval)
NB_SCALAR_ACCESSORS(maxtime, double, maxtime)
NB_SCALAR_ACCESSORS(population, unsigned, stochastic_population)
NB_SCALAR_ACCESSORS(vector_storage, unsigned, vector_storage)
#undef NB_SCALAR_ACCESSORS

int nlopt_get_numevals(const nlopt_opt opt) { return opt->numevals; }

nlopt_result nlopt_set_xtol_abs(nlopt_opt opt, const double *v)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    leave_device_option(opt->xtol_abs_dev);
    if (!v) { opt->xtol_abs.clear(); opt->has_xtol_abs = false; return NLOPT_SUCCESS; }
    opt->xtol_abs.assign(v, v + opt->n);
    opt->has_xtol_abs = opt->n > 0;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_xtol_abs1(nlopt_opt opt, double v)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    leave_device_option(opt->xtol_abs_dev);
    opt->xtol_abs.assign(opt->n, v);
    opt->has_xtol_abs = opt->n > 0;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_get_xtol_abs(const nlopt_opt opt, double *v)
{
    clear_err(opt);
    if (!opt || (opt->n > 0 && !v)) return NLOPT_INVALID_ARGS;
    if (!host_option(opt, opt->xtol_abs_dev, opt->xtol_abs)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) v[i] = opt->has_xtol_abs ? opt->xtol_abs[i] : 0.0;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_x_weights(nlopt_opt opt, const double *w)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (!w) {
        leave_device_option(opt->x_weights_dev);
        opt->x_weights.clear();
        opt->has_x_weights = false;
        return NLOPT_SUCCESS;
    }
    for (unsigned i = 0; i < opt->n; ++i)
        if (w[i] < 0) { set_err(opt, "invalid negative weight"); return NLOPT_INVALID_ARGS; }
    leave_device_option(opt->x_weights_dev);
    opt->x_weights.assign(w, w + opt->n);
    opt->has_x_weights = opt->n > 0;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_x_weights1(nlopt_opt opt, double w)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    if (w < 0) { set_err(opt, "invalid negative weight"); return NLOPT_INVALID_ARGS; }
    clear_err(opt);
    leave_device_option(opt->x_weights_dev);
    opt->x_weights.assign(opt->n, w);
    opt->has_x_weights = opt->n > 0;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_get_x_weights(const nlopt_opt opt, double *w)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    if (opt->n > 0 && !w) { set_err(opt, "invalid NULL weights"); return NLOPT_INVALID_ARGS; }
    clear_err(opt);
    if (!host_option(opt, opt->x_weights_dev, opt->x_weights)) return NLOPT_FAILURE;
    for (unsigned i = 0; i < opt->n; ++i) w[i] = opt->has_x_weights ? opt->x_weights[i] : 1.0;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_force_stop(nlopt_opt opt, int val)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    opt->force_stop = val;
    if (opt->force_stop_child) return nlopt_set_force_stop(opt->force_stop_child, val);
    return NLOPT_SUCCESS;
}
int nlopt_get_force_stop(const nlopt_opt opt) { return opt->force_stop; }
nlopt_result nlopt_force_stop(nlopt_opt opt) { return nlopt_set_force_stop(opt, 1); }

/* ------------------------------------------------------------------ algorithm-specific (options.c:818-957) */

nlopt_result nlopt_set_local_optimizer(nlopt_opt opt, const nlopt_opt local_opt)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (local_opt && local_opt->n != opt->n) {
        set_err(opt, "dimension mismatch in local optimizer");
        return NLOPT_INVALID_ARGS;
    }
    nlopt_destroy(opt->local_opt);
    opt->local_opt = nlopt_copy(local_opt);
    if (local_opt) {
        if (!opt->local_opt) return NLOPT_OUT_OF_MEMORY;
        nlopt_opt lo = opt->local_opt;
        if (!host_bounds(opt)) return NLOPT_FAILURE;
        nlopt_set_lower_bounds(lo, opt->lb.data());
        nlopt_set_upper_bounds(lo, opt->ub.data());
        nlopt_remove_inequality_constraints(lo);
        nlopt_remove_equality_constraints(lo);
        nlopt_set_min_objective(lo, nullptr, nullptr);
        nlopt_set_munge(lo, nullptr, nullptr);
        lo->force_stop = 0;
    }
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_initial_step1(nlopt_opt opt, double dx)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (dx == 0) { set_err(opt, "zero step size"); return NLOPT_INVALID_ARGS; }
    leave_device_option(opt->dx_dev);
    opt->dx.assign(opt->n, dx);
    opt->has_dx = opt->n > 0;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_set_initial_step(nlopt_opt opt, const double *dx)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (!dx) {
        leave_device_option(opt->dx_dev);
        opt->dx.clear();
        opt->has_dx = false;
        return NLOPT_SUCCESS;
    }
    for (unsigned i = 0; i < opt->n; ++i)
        if (dx[i] == 0) { set_err(opt, "zero step size"); return NLOPT_INVALID_ARGS; }
    leave_device_option(opt->dx_dev);
    opt->dx.assign(dx, dx + opt->n);
    opt->has_dx = opt->n > 0;
    return NLOPT_SUCCESS;
}

/* heuristic step of options.c:903-957 (used by derivative-free algorithms; kept for ABI completeness) */
nlopt_result nlopt_set_default_initial_step(nlopt_opt opt, const double *x)
{
    clear_err(opt);
    if (!opt || !x) return NLOPT_INVALID_ARGS;
    if (!host_bounds(opt)) return NLOPT_FAILURE;
    leave_device_option(opt->dx_dev);
    opt->dx.assign(opt->n, 1.0);
    opt->has_dx = opt->n > 0;
    for (unsigned i = 0; i < opt->n; ++i) {
        const double lo = opt->lb[i], hi = opt->ub[i];
        const bool flo = !nb200::nl_isinf(lo), fhi = !nb200::nl_isinf(hi);
        double step = kInf;
        if (fhi && flo && (hi - lo) * 0.25 < step && hi > lo) step = (hi - lo) * 0.25;
        if (fhi && hi - x[i] < step && hi > x[i]) step = (hi - x[i]) * 0.75;
        if (flo && x[i] - lo < step && x[i] > lo) step = (x[i] - lo) * 0.75;
        if (nb200::nl_isinf(step)) {
            if (fhi && std::fabs(hi - x[i]) < std::fabs(step)) step = (hi - x[i]) * 1.1;
            if (flo && std::fabs(x[i] - lo) < std::fabs(step)) step = (x[i] - lo) * 1.1;
        }
        if (nb200::nl_isinf(step) || is_tiny(step)) step = x[i];
        if (nb200::nl_isinf(step) || step == 0.0) step = 1;
        opt->dx[i] = step;
    }
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_get_initial_step(const nlopt_opt opt, const double *x, double *dx)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    clear_err(opt);
    if (!opt->n) return NLOPT_SUCCESS;
    if (!opt->has_dx) {
        nlopt_result r = nlopt_set_default_initial_step(opt, x);
        if (r != NLOPT_SUCCESS) return r;
        for (unsigned i = 0; i < opt->n; ++i) dx[i] = opt->dx[i];
        opt->dx.clear();                 /* x-dependent: not remembered (options.c:896-898) */
        opt->has_dx = false;
    } else {
        if (!host_option(opt, opt->dx_dev, opt->dx)) return NLOPT_FAILURE;
        for (unsigned i = 0; i < opt->n; ++i) dx[i] = opt->dx[i];
    }
    return NLOPT_SUCCESS;
}

void nlopt_set_munge(nlopt_opt opt, nlopt_munge on_destroy, nlopt_munge on_copy)
{
    if (opt) { opt->munge_on_destroy = on_destroy; opt->munge_on_copy = on_copy; }
}

void nlopt_munge_data(nlopt_opt opt, nlopt_munge2 munge, void *data)
{
    if (!opt || !munge) return;
    opt->objective.data = munge(opt->objective.data, data);
    for (auto &c : opt->fc) c.fn.data = munge(c.fn.data, data);
    for (auto &c : opt->h) c.fn.data = munge(c.fn.data, data);
}

nlopt_result nlopt_b200_get_stats(const nlopt_opt opt, nlopt_b200_stats *out)
{
    if (!opt || !out) return NLOPT_INVALID_ARGS;
    *out = opt->stats;
    return NLOPT_SUCCESS;
}

/* ------------------------------------------------------------------ run (optimize.c:991-1083) */

static nlopt_result optimize_common(nlopt_opt opt, double *x_host, double *x_dev, double *opt_f)
{
    clear_err(opt);
    if (!opt || !opt_f || opt->objective.empty()) {
        set_err(opt, "NULL args to nlopt_optimize");
        return NLOPT_INVALID_ARGS;
    }
    nlopt_set_force_stop(opt, 0);
    opt->force_stop_child = nullptr;

    /* maximisation: minimise the sign-flipped objective, then restore (optimize.c:1014-1024, :1070-1077).  A host
       objective is wrapped in flipped(); a device or sharded objective keeps its callback and the backend negates its
       final value and its gradient (FuncSpec::negate) */
    FuncSpec &obj = opt->objective;
    nlopt_func f0 = obj.f;
    void *d0 = obj.data;
    FlipData flip{f0, d0};
    const int maximize = opt->maximize;
    if (maximize) {
        if (obj.f) {
            obj.f = flipped;
            obj.data = &flip;
        } else
            obj.negate = true;
        opt->stopval = -opt->stopval;
        opt->maximize = 0;
    }
    nlopt_result ret;
    if (is_auglag(opt->algorithm))
        ret = run_auglag(opt, x_host, x_dev, opt_f);
    else
        ret = run_ccsa(opt, x_host, x_dev, opt_f);
    if (maximize) {
        opt->maximize = maximize;
        obj.negate = false;
        opt->stopval = -opt->stopval;
        obj.f = f0;
        obj.data = d0;
        *opt_f = -*opt_f;
    }
    return ret;
}

nlopt_result nlopt_optimize(nlopt_opt opt, double *x, double *opt_f)
{
    return optimize_common(opt, x, nullptr, opt_f);
}

/* ------------------------------------------------------------------ deprecated API (deprecated.c) */

void nlopt_get_local_search_algorithm(nlopt_algorithm *deriv, nlopt_algorithm *nonderiv, int *maxeval)
{
    *deriv = g_local_deriv;
    *nonderiv = g_local_nonderiv;
    *maxeval = g_local_maxeval;
}

void nlopt_set_local_search_algorithm(nlopt_algorithm deriv, nlopt_algorithm nonderiv, int maxeval)
{
    g_local_deriv = deriv;
    g_local_nonderiv = nonderiv;
    g_local_maxeval = maxeval;
}

int nlopt_get_stochastic_population(void) { return g_stochastic_population; }
void nlopt_set_stochastic_population(int pop) { g_stochastic_population = pop <= 0 ? 0 : pop; }

nlopt_result nlopt_minimize_econstrained(nlopt_algorithm algorithm, int n, nlopt_func_old f, void *f_data, int m,
                                         nlopt_func_old fc, void *fc_data, ptrdiff_t fc_datum_size, int p, nlopt_func_old h,
                                         void *h_data, ptrdiff_t h_datum_size, const double *lb, const double *ub, double *x,
                                         double *minf, double minf_max, double ftol_rel, double ftol_abs, double xtol_rel,
                                         const double *xtol_abs, double htol_rel, double htol_abs, int maxeval, double maxtime)
{
    (void) htol_rel;                     /* unused in the reference as well (deprecated.c:97) */
    if (n < 0 || m < 0 || p < 0) return NLOPT_INVALID_ARGS;
    nlopt_opt opt = nlopt_create(algorithm, (unsigned) n);
    if (!opt) return NLOPT_INVALID_ARGS;
    /* the old callback type differs from nlopt_func only in the signedness of n */
    nlopt_result ret = nlopt_set_min_objective(opt, reinterpret_cast<nlopt_func>(f), f_data);
    for (int i = 0; ret == NLOPT_SUCCESS && i < m; ++i)
        ret = nlopt_add_inequality_constraint(opt, reinterpret_cast<nlopt_func>(fc), static_cast<char *>(fc_data) + i * fc_datum_size, 0.0);
    for (int i = 0; ret == NLOPT_SUCCESS && i < p; ++i)
        ret = nlopt_add_equality_constraint(opt, reinterpret_cast<nlopt_func>(h), static_cast<char *>(h_data) + i * h_datum_size, htol_abs);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_lower_bounds(opt, lb);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_upper_bounds(opt, ub);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_stopval(opt, minf_max);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_ftol_rel(opt, ftol_rel);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_ftol_abs(opt, ftol_abs);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_xtol_rel(opt, xtol_rel);
    if (ret == NLOPT_SUCCESS && xtol_abs) ret = nlopt_set_xtol_abs(opt, xtol_abs);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_maxeval(opt, maxeval);
    if (ret == NLOPT_SUCCESS) ret = nlopt_set_maxtime(opt, maxtime);
    if (ret == NLOPT_SUCCESS) ret = nlopt_optimize(opt, x, minf);
    nlopt_destroy(opt);
    return ret;
}

nlopt_result nlopt_minimize_constrained(nlopt_algorithm algorithm, int n, nlopt_func_old f, void *f_data, int m,
                                        nlopt_func_old fc, void *fc_data, ptrdiff_t fc_datum_size, const double *lb,
                                        const double *ub, double *x, double *minf, double minf_max, double ftol_rel,
                                        double ftol_abs, double xtol_rel, const double *xtol_abs, int maxeval, double maxtime)
{
    return nlopt_minimize_econstrained(algorithm, n, f, f_data, m, fc, fc_data, fc_datum_size, 0, nullptr, nullptr, 0, lb, ub,
                                       x, minf, minf_max, ftol_rel, ftol_abs, xtol_rel, xtol_abs, ftol_rel, ftol_abs, maxeval, maxtime);
}

nlopt_result nlopt_minimize(nlopt_algorithm algorithm, int n, nlopt_func_old f, void *f_data, const double *lb,
                            const double *ub, double *x, double *minf, double minf_max, double ftol_rel, double ftol_abs,
                            double xtol_rel, const double *xtol_abs, int maxeval, double maxtime)
{
    return nlopt_minimize_constrained(algorithm, n, f, f_data, 0, nullptr, nullptr, 0, lb, ub, x, minf, minf_max, ftol_rel,
                                      ftol_abs, xtol_rel, xtol_abs, maxeval, maxtime);
}

nlopt_result nlopt_b200_optimize_device(nlopt_opt opt, double *x_dev, double *opt_f)
{
    return optimize_common(opt, nullptr, x_dev, opt_f);
}

}  // extern "C"

namespace {

// nlopt_optimize_ (optimize.c:514-566) + the MMA/CCSAQ case (optimize.c:795-834)
nlopt_result run_ccsa(nlopt_opt opt, double *x_host, double *x_dev, double *minf)
{
    const unsigned n = opt->n;
    if ((!x_host && !x_dev) || opt->maximize) {
        set_err(opt, "NULL args to nlopt_optimize_");
        return NLOPT_INVALID_ARGS;
    }
    if (n == 0) {                                    /* optimize.c:536-539 */
        if (!opt->objective.f) { set_err(opt, "n == 0 needs a host objective"); return NLOPT_INVALID_ARGS; }
        *minf = opt->objective.f(0, x_host, nullptr, opt->objective.data);
        return NLOPT_SUCCESS;
    }
    *minf = HUGE_VAL;

    if (opt->algorithm != NLOPT_LD_MMA && opt->algorithm != NLOPT_LD_CCSAQ) {
        set_err(opt, "algorithm %s is not part of this library (only LD_MMA and LD_CCSAQ are built)",
                nlopt_algorithm_to_string(opt->algorithm));
        return NLOPT_INVALID_ARGS;
    }
    const bool dev_bounds = device_mode(opt);      /* device bounds: the backend checks the start point */
    if (dev_bounds && !device_mode_runs_here(opt)) return NLOPT_INVALID_ARGS;
    if (!device_options_run_here(opt)) return NLOPT_INVALID_ARGS;
    if (x_host && !dev_bounds)                       /* optimize.c:547-551 */
        for (unsigned i = 0; i < n; ++i)
            if (opt->lb[i] > opt->ub[i] || x_host[i] < opt->lb[i] || x_host[i] > opt->ub[i]) {
                set_err(opt, "bounds %d fail %g <= %g <= %g", (int) i, opt->lb[i], x_host[i], opt->ub[i]);
                return NLOPT_INVALID_ARGS;
            }

    /* parameters, optimize.c:798-815 */
    nb200::CcsaParams prm;
    prm.inner_maxeval = (int) nlopt_get_param(opt, "inner_maxeval", 0);
    prm.verbosity = (int) nlopt_get_param(opt, "verbosity", 0);
    prm.rho_init = nlopt_get_param(opt, "rho_init", 1.0);
    prm.inner_gradients = (int) nlopt_get_param(opt, "inner_gradients", 1);
    prm.always_improve = (int) nlopt_get_param(opt, "always_improve", 1);
    prm.sigma_min = nlopt_get_param(opt, "sigma_min", 0.0);
    if (!(prm.rho_init > 0) && !nb200::nl_isinf(prm.rho_init)) {
        set_err(opt, "rho_init must be positive and finite");
        return NLOPT_INVALID_ARGS;
    }
    if (prm.inner_gradients != 0 && prm.inner_gradients != 1) {
        set_err(opt, "inner_gradients must be 0 or 1");
        return NLOPT_INVALID_ARGS;
    }
    if (prm.always_improve != 0 && prm.always_improve != 1) {
        set_err(opt, "always_improve must be 0 or 1");
        return NLOPT_INVALID_ARGS;
    }
    if (prm.sigma_min < 0.0) { set_err(opt, "sigma_min must be non-negative"); return NLOPT_INVALID_ARGS; }
    if (prm.verbosity < 0) prm.verbosity = 0;

    /* the dual optimiser's configuration, optimize.c:817-826.  Precedence: named parameter >
       local optimiser (if one was set) > library default; only MMA exists here for the dual. */
    const nlopt_opt lo = opt->local_opt;
    const int dual_alg = (int) nlopt_get_param(opt, "dual_algorithm", lo ? (double) lo->algorithm : (double) g_local_deriv);
    if (dual_alg != NLOPT_LD_MMA) {
        set_err(opt, "dual_algorithm %d is not part of this library (the dual problem is solved by LD_MMA)", dual_alg);
        return NLOPT_INVALID_ARGS;
    }
    prm.dual_ftol_rel = nlopt_get_param(opt, "dual_ftol_rel", lo ? lo->ftol_rel : 1e-14);
    prm.dual_ftol_abs = nlopt_get_param(opt, "dual_ftol_abs", lo ? lo->ftol_abs : 0.0);
    prm.dual_xtol_rel = nlopt_get_param(opt, "dual_xtol_rel", 0.0);
    prm.dual_xtol_abs = nlopt_get_param(opt, "dual_xtol_abs", 0.0);
    prm.dual_maxeval = (int) nlopt_get_param(opt, "dual_maxeval", lo ? (double) lo->maxeval : 100000.0);

    bool any_pre = opt->objective.pre != nullptr, all_host = opt->objective.host(), any_dpre = opt->objective.dpre != nullptr;
    for (const auto &c : opt->fc) {
        any_pre = any_pre || c.fn.pre != nullptr;
        any_dpre = any_dpre || c.fn.dpre != nullptr;
        all_host = all_host && c.fn.host();
    }
    any_dpre = any_dpre && opt->algorithm == NLOPT_LD_CCSAQ;     /* LD_MMA ignores preconditioners (mma.c) */
    if (any_pre && any_dpre) {
        set_err(opt, "preconditioned CCSAQ takes host preconditioners (nlopt_precond) or device preconditioners "
                     "(nlopt_b200_dprecond), not both in one run");
        return NLOPT_INVALID_ARGS;
    }
    if (any_pre && opt->algorithm == NLOPT_LD_CCSAQ) {          /* ccsa_quadratic.c: the !no_precond branch */
        if (!x_host || !all_host) {
            set_err(opt, "preconditioned CCSAQ takes host x and host callbacks (nlopt_precond is a host function)");
            return NLOPT_INVALID_ARGS;
        }
        if (dev_bounds) {
            set_err(opt, "preconditioned CCSAQ takes host bounds (its model problem is built on the host)");
            return NLOPT_INVALID_ARGS;
        }
        if (!host_options(opt)) return NLOPT_FAILURE;     /* device options: read through their host mirrors */
        return run_ccsa_precond(opt, x_host, minf, prm);
    }

    /* hand the O(n) state to the device */
    nb200::BackendConfig cfg;
    cfg.variant = opt->algorithm == NLOPT_LD_MMA ? nb200::kMMA : nb200::kCCSAQ;
    cfg.n = n;
    cfg.objective = opt->objective;
    cfg.penalty = opt->penalty;
    /* a maximisation reaches here as the minimisation of -f: a host objective wrapped in flipped(), any other form
       with FuncSpec::negate (optimize_common) */
    cfg.maximize = opt->objective.negate || opt->objective.f == flipped;
    std::vector<double> tol;
    for (const auto &c : opt->fc) {
        cfg.constraints.push_back(c.fn);
        tol.insert(tol.end(), c.tol.begin(), c.tol.end());
    }
    cfg.lb = opt->lb.data();
    cfg.ub = opt->ub.data();
    cfg.lb_uniform = opt->lb_uniform && n > 0;
    cfg.ub_uniform = opt->ub_uniform && n > 0;
    nb200::StartCheck start;
    if (dev_bounds) {
        cfg.lb = cfg.ub = nullptr;
        cfg.lb_dev = opt->dbounds->lb();
        cfg.ub_dev = opt->dbounds->ub();
        cfg.start_check = &start;
    }
    cfg.x0_host = x_host;
    cfg.x_dev = x_dev;
    cfg.sigma_init = opt->has_dx ? opt->dx.data() : nullptr;
    cfg.x_weights = opt->has_x_weights ? opt->x_weights.data() : nullptr;
    cfg.xtol_abs = opt->has_xtol_abs ? opt->xtol_abs.data() : nullptr;
    if (const nb200::DeviceVector *d = opt->dx_dev.dev) {       /* device options: read in place */
        cfg.sigma_init = nullptr;
        cfg.sigma_init_dev = d->data();
        cfg.sigma_init_uniform = d->uniform();
        cfg.sigma_init0 = d->lane0();
    }
    if (opt->x_weights_dev.dev) {
        cfg.x_weights = nullptr;
        cfg.x_weights_dev = opt->x_weights_dev.dev->data();
    }
    if (opt->xtol_abs_dev.dev) {
        cfg.xtol_abs = nullptr;
        cfg.xtol_abs_dev = opt->xtol_abs_dev.dev->data();
    }
    opt->stats = nlopt_b200_stats{};
    cfg.stats = &opt->stats;

    const double t0 = nb200::wall_seconds();
    std::string err;
    nb200::Backend *be = nb200::make_backend(cfg, &err);
    if (!be) {
        set_err(opt, "%s", err.c_str());
        return NLOPT_FAILURE;
    }
    if (start.bad >= 0) {                            /* optimize.c:547-551, found on the device */
        delete be;
        set_err(opt, "bounds %d fail %g <= %g <= %g", (int) start.bad, start.lb, start.x, start.ub);
        return NLOPT_INVALID_ARGS;
    }
    if (any_dpre && be->ranks() > 1) {               /* the nested model solve runs on device bounds: one rank */
        delete be;
        set_err(opt, "preconditioned CCSAQ with device preconditioners runs on one GPU in this library");
        return NLOPT_INVALID_ARGS;
    }
    if (any_dpre && !be->solves_model()) {           /* never a silent separable run */
        delete be;
        set_err(opt, "this backend does not solve preconditioned models");
        return NLOPT_FAILURE;
    }
    opt->stats.seconds_setup = nb200::wall_seconds() - t0;

    /* library-specific knobs ride on the named-parameter mechanism (no ABI change) */
    if (nlopt_has_param(opt, "b200_geometry_rule")) be->configure("geometry_rule", (long long) nlopt_get_param(opt, "b200_geometry_rule", 1.0));
    if (nlopt_has_param(opt, "b200_group_min_chunks")) be->configure("group_min_chunks", (long long) nlopt_get_param(opt, "b200_group_min_chunks", 2.0));
    if (nlopt_has_param(opt, "b200_group_base")) be->configure("group_base", (long long) nlopt_get_param(opt, "b200_group_base", 440.0));
    if (nlopt_get_param(opt, "b200_time_kernels", 0.0) != 0.0) be->configure("time_kernels", 1);
    if (nlopt_has_param(opt, "b200_pmax")) be->configure("pmax", (long long) nlopt_get_param(opt, "b200_pmax", 0.0));
    if (nlopt_has_param(opt, "b200_target_chunks"))
        be->configure("target_chunks", (long long) nlopt_get_param(opt, "b200_target_chunks", 0.0));
    prm.fused_solve = (int) nlopt_get_param(opt, "b200_fused_solve", 1.0);
    if (nlopt_has_param(opt, "b200_kernel_cfg")) be->configure("kernel_cfg", (long long) nlopt_get_param(opt, "b200_kernel_cfg", 0.0));
    if (nlopt_has_param(opt, "b200_ctas_per_sm")) be->configure("ctas_per_sm", (long long) nlopt_get_param(opt, "b200_ctas_per_sm", 0.0));
    if (nlopt_has_param(opt, "b200_solve_tma")) be->configure("solve_tma", (long long) nlopt_get_param(opt, "b200_solve_tma", -1.0));
    if (nlopt_has_param(opt, "b200_solve_minb")) be->configure("solve_minb", (long long) nlopt_get_param(opt, "b200_solve_minb", 0.0));
    if (nlopt_has_param(opt, "b200_solve_async")) be->configure("solve_async", (long long) nlopt_get_param(opt, "b200_solve_async", 0.0));
    if (nlopt_has_param(opt, "b200_l2_keep_mb")) be->configure("l2_keep_mb", (long long) nlopt_get_param(opt, "b200_l2_keep_mb", 0.0));

    nb200::StopCriteria st;                          /* optimize.c:553-566 */
    st.minf_max = opt->stopval;
    st.ftol_rel = opt->ftol_rel;
    st.ftol_abs = opt->ftol_abs;
    st.xtol_rel = opt->xtol_rel;
    st.has_xtol_abs = opt->has_xtol_abs;
    opt->numevals = 0;
    st.nevals_p = &opt->numevals;
    st.maxeval = opt->maxeval;
    st.maxtime = opt->maxtime;
    st.start = t0;                                   /* the clock started before the device state was built */
    st.force_stop = &opt->force_stop;

    nb200::DriverStats ds;
    int ret = nb200::ccsa_minimize(cfg.variant, *be, tol, minf, st, prm, &ds, &err);
    if (ret == NLOPT_FAILURE && !err.empty()) set_err(opt, "%s", err.c_str());
    if (ret == NLOPT_INVALID_ARGS && !err.empty()) set_err(opt, "%s", err.c_str());
    const double t_fetch0 = nb200::wall_seconds();
    if (!be->fetch_x(x_host ? x_host : x_dev) && ret > 0) {
        set_err(opt, "copying the result back failed: %s", be->error().c_str());
        ret = NLOPT_FAILURE;
    }
    opt->stats.dual_evals = ds.dual_evals;
    opt->stats.dual_solves = ds.dual_solves;
    opt->stats.outer_iters = ds.outer_iters;
    opt->stats.seconds_callbacks = be->seconds_in_callbacks();
    opt->stats.seconds_dual_wall = ds.seconds_dual;
    opt->stats.seconds_eval_wall = ds.seconds_eval;
    opt->stats.seconds_glue_wall = ds.seconds_glue + (nb200::wall_seconds() - t_fetch0);
    delete be;
    opt->stats.seconds_total = nb200::wall_seconds() - t0;
    return (nlopt_result) ret;
}

// ---- NLOPT_AUGLAG / AUGLAG_EQ / LD_AUGLAG / LD_AUGLAG_EQ (optimize.c:907-939, src/algs/auglag/auglag.c:69-300) ----
// The outer loop (multiplier and penalty updates: scalars) runs here; the sub-problems go to LD_MMA / LD_CCSAQ on
// the device, whose objective is the augmented Lagrangian evaluated by the backend (PenaltySpec).
bool rel_stop_host(double vold, double vnew, double reltol, double abstol)      // stop.c:81-86
{
    if (nb200::nl_isinf(vold)) return false;
    const double d = std::fabs(vnew - vold);
    return d < abstol || d < reltol * (std::fabs(vnew) + std::fabs(vold)) * 0.5 || (reltol > 0 && vnew == vold);
}

// ---- preconditioned CCSAQ (ccsa_quadratic.c:153-206, :299-324, :415-441) ------------------------------------------
// With a preconditioner H (user function v -> H(x0) v, nlopt.h:70) on the objective and/or on constraints, the
// convex model around x0 is no longer separable:
//     g(x) = f(x0) + grad f . dx + rho/2 sum_j (dx_j / sigma_j)^2 + 1/2 dx^T H dx        (gfunc, :153-181)
// so there is no closed-form dual.  The reference solves the model problem  min g0  s.t.  gi <= 0  in the trust box
// max(lb, x0 - sigma) <= x <= min(ub, x0 + sigma) with a nested n-dimensional optimiser -- the dual optimiser's
// algorithm and tolerances, i.e. LD_MMA by default (:299-324) -- and keeps the CCSA outer / inner logic unchanged.
// Here the nested problem is an ordinary LD_MMA run of THIS library: its dual evaluations over the n variables are
// the CUDA kernels; g0 / gi are host callbacks because nlopt_precond is a host function (they see x on the host like
// any nlopt_func).  The O(n) glue of this outer loop (sigma update, stop norms) stays on the host: each inner
// iteration is dominated by a whole nested solve.
// One deliberate difference: the reference never assigns dd.wval on this branch (it reads an uninitialised stack
// slot in the rho updates at :550-556); here w = 1/2 sum (dx_j / sigma_j)^2, the value the separable branch uses.
struct PrecondModel {
    unsigned n = 0, m = 0;
    const double *x0 = nullptr, *sigma = nullptr, *dfdx = nullptr, *dfcdx = nullptr;
    double fval = 0, rho = 0;
    const double *fcval = nullptr, *rhoc = nullptr;
    const FuncSpec *obj = nullptr;           // the preconditioners (and their data) of the objective ...
    std::vector<const FuncSpec *> prec;      // ... and of each constraint row
    std::vector<double> scratch;             // dx | H dx
    long count = 0;
};

double precond_gfunc(PrecondModel &d, double f, const double *dfdx, double rho, const FuncSpec &fn, const double *x,
                     double *grad)                                     // ccsa_quadratic.c:153-181
{
    const unsigned n = d.n;
    double *dx = d.scratch.data(), *Hdx = dx + n;
    double val = f;
    for (unsigned j = 0; j < n; ++j) {
        const double sigma2inv = 1.0 / (d.sigma[j] * d.sigma[j]);
        dx[j] = x[j] - d.x0[j];
        val += dfdx[j] * dx[j] + (0.5 * rho) * (dx[j] * dx[j]) * sigma2inv;
        if (grad) grad[j] = dfdx[j] + rho * dx[j] * sigma2inv;
    }
    if (fn.pre) {
        fn.pre(n, d.x0, dx, Hdx, fn.data);
        for (unsigned j = 0; j < n; ++j) val += 0.5 * dx[j] * Hdx[j];
        if (grad)
            for (unsigned j = 0; j < n; ++j) grad[j] += Hdx[j];
    }
    return val;
}

double precond_g0(unsigned, const double *x, double *grad, void *dp)     // :183-191
{
    PrecondModel &d = *static_cast<PrecondModel *>(dp);
    ++d.count;
    return precond_gfunc(d, d.fval, d.dfdx, d.rho, *d.obj, x, grad);
}

void precond_gi(unsigned m, double *result, unsigned n, const double *x, double *grad, void *dp)      // :194-206
{
    PrecondModel &d = *static_cast<PrecondModel *>(dp);
    for (unsigned i = 0; i < m; ++i)
        result[i] = precond_gfunc(d, d.fcval[i], d.dfcdx + (size_t) i * n, d.rhoc[i], *d.prec[i], x,
                                  grad ? grad + (size_t) i * n : nullptr);
}

nlopt_result run_ccsa_precond(nlopt_opt opt, double *x, double *minf, const nb200::CcsaParams &prm)
{
    const unsigned n = opt->n;
    unsigned m = 0;
    for (const auto &c : opt->fc) m += c.fn.m;
    const double t_start = nb200::wall_seconds();
    opt->stats = nlopt_b200_stats{};
    opt->numevals = 0;
    auto forced = [&]() { return opt->force_stop != 0; };
    auto evals_out = [&]() { return opt->maxeval > 0 && opt->numevals >= opt->maxeval; };
    auto timed_out = [&]() { return opt->maxtime > 0 && nb200::wall_seconds() - t_start >= opt->maxtime; };

    std::vector<double> sigma(n), dfdx(n), dfdx_cur(n), xcur(n), xprev(n), xprevprev(n), pre_lb(n), pre_ub(n);
    std::vector<double> dfcdx((size_t) m * n), dfcdx_cur((size_t) m * n), fcval(m), fcval_cur(m), rhoc(m, prm.rho_init), gcval(m), tol;
    for (const auto &c : opt->fc) tol.insert(tol.end(), c.tol.begin(), c.tol.end());
    PrecondModel dd;
    dd.n = n; dd.m = m;
    dd.x0 = x; dd.sigma = sigma.data(); dd.dfdx = dfdx.data(); dd.dfcdx = dfcdx.data();
    dd.fcval = fcval.data(); dd.rhoc = rhoc.data();
    dd.obj = &opt->objective;
    for (const auto &c : opt->fc)
        for (unsigned k = 0; k < c.fn.m; ++k) dd.prec.push_back(&c.fn);
    dd.scratch.assign(2 * (size_t) n, 0.0);

    // the nested optimiser (ccsa_quadratic.c:299-324): dual algorithm and tolerances, objective g0, constraints gi
    nlopt_opt pre_opt = nlopt_create(NLOPT_LD_MMA, n);
    if (!pre_opt) { set_err(opt, "failure creating precond. optimizer"); return NLOPT_FAILURE; }
    struct Guard { nlopt_opt o; ~Guard() { nlopt_destroy(o); } } guard{pre_opt};
    nlopt_result ret = nlopt_set_min_objective(pre_opt, precond_g0, &dd);
    if (ret >= 0 && m) ret = nlopt_add_inequality_mconstraint(pre_opt, m, precond_gi, &dd, nullptr);
    if (ret >= 0) ret = nlopt_set_ftol_rel(pre_opt, prm.dual_ftol_rel);
    if (ret >= 0) ret = nlopt_set_ftol_abs(pre_opt, prm.dual_ftol_abs);
    if (ret >= 0) ret = nlopt_set_maxeval(pre_opt, prm.dual_maxeval);
    if (ret < 0) return ret;
    opt->force_stop_child = pre_opt;                  // nlopt_force_stop on the outer object reaches the nested run

    for (unsigned j = 0; j < n; ++j) {                // :324-332
        if (opt->has_dx && opt->dx[j] > 0) sigma[j] = opt->dx[j];
        else if (nb200::nl_isinf(opt->ub[j]) || nb200::nl_isinf(opt->lb[j])) sigma[j] = 1.0;
        else sigma[j] = 0.5 * (opt->ub[j] - opt->lb[j]);
        sigma[j] = sigma[j] > prm.sigma_min ? sigma[j] : prm.sigma_min;
    }
    double rho = prm.rho_init, fcur;
    const FuncSpec &obj = opt->objective;
    auto eval_f = [&](const double *xx, double *g) { ++opt->numevals; return obj.f(n, xx, g, obj.data); };
    auto eval_c = [&](const double *xx, double *vals, double *grads) -> bool {
        unsigned i = 0;
        for (const auto &c : opt->fc) {
            eval_host(c.fn, n, xx, vals + i, grads ? grads + (size_t) i * n : nullptr);
            i += c.fn.m;
            if (forced()) return false;
        }
        return true;
    };
    dd.fval = fcur = *minf = eval_f(x, dfdx.data());
    xcur.assign(x, x + n);
    if (forced()) return NLOPT_FORCED_STOP;
    if (!eval_c(x, fcval.data(), dfcdx.data())) return NLOPT_FORCED_STOP;
    bool feasible = true;
    double infeasibility = 0;
    for (unsigned i = 0; i < m; ++i) {
        feasible = feasible && fcval[i] <= 0;
        if (fcval[i] > infeasibility) infeasibility = fcval[i];
    }
    auto check_stop = [&]() -> nlopt_result {
        if (forced()) return NLOPT_FORCED_STOP;
        if (evals_out()) return NLOPT_MAXEVAL_REACHED;
        if (timed_out()) return NLOPT_MAXTIME_REACHED;
        if (feasible && *minf < opt->stopval) return NLOPT_STOPVAL_REACHED;
        return NLOPT_SUCCESS;
    };
    unsigned k = 0;
    for (;;) {                                        // outer iterations (:404)
        const double fprev = fcur;
        if ((ret = check_stop()) != NLOPT_SUCCESS) return ret;
        if (++k > 1) xprevprev = xprev;
        xprev = xcur;
        int inner_nevals = 0;
        for (;;) {                                    // inner iterations (:417)
            for (unsigned j = 0; j < n; ++j) {        // :441-446
                pre_lb[j] = opt->lb[j] > x[j] - sigma[j] ? opt->lb[j] : x[j] - sigma[j];
                pre_ub[j] = opt->ub[j] < x[j] + sigma[j] ? opt->ub[j] : x[j] + sigma[j];
                xcur[j] = x[j];
            }
            nlopt_set_lower_bounds(pre_opt, pre_lb.data());
            nlopt_set_upper_bounds(pre_opt, pre_ub.data());
            dd.rho = rho; dd.count = 0;
            if (opt->maxtime > 0) {
                const double left = opt->maxtime - (nb200::wall_seconds() - t_start);
                nlopt_set_maxtime(pre_opt, left > 0 ? left : 1e-9);
            }
            double pre_min;
            const nlopt_result reti = nlopt_optimize(pre_opt, xcur.data(), &pre_min);
            opt->stats.dual_evals += pre_opt->stats.dual_evals;
            opt->stats.kernel_launches += pre_opt->stats.kernel_launches;
            opt->stats.dual_operand_bytes += pre_opt->stats.dual_operand_bytes;
            ++opt->stats.dual_solves;
            if (reti < 0 || reti == NLOPT_MAXTIME_REACHED) {
                if (reti < 0 && nlopt_get_errmsg(pre_opt)) set_err(opt, "nested model solve: %s", nlopt_get_errmsg(pre_opt));
                return forced() ? NLOPT_FORCED_STOP : reti;
            }
            const double gval = precond_g0(n, xcur.data(), nullptr, &dd);       // :465-467
            if (m) precond_gi(m, gcval.data(), n, xcur.data(), nullptr, &dd);
            double wval = 0;
            for (unsigned j = 0; j < n; ++j) { const double q = (xcur[j] - x[j]) / sigma[j]; wval += 0.5 * q * q; }
            if (prm.verbosity) std::printf("CCSA dual converged in %ld iters to g=%g:\n", dd.count, gval);

            fcur = eval_f(xcur.data(), prm.inner_gradients ? dfdx_cur.data() : nullptr);
            ++inner_nevals;
            if (forced()) return NLOPT_FORCED_STOP;
            bool feasible_cur = true, inner_done = gval >= fcur;
            double infeasibility_cur = 0;
            if (!eval_c(xcur.data(), fcval_cur.data(), prm.inner_gradients ? dfcdx_cur.data() : nullptr)) return NLOPT_FORCED_STOP;
            for (unsigned i = 0; i < m; ++i) {
                feasible_cur = feasible_cur && fcval_cur[i] <= tol[i];
                inner_done = inner_done && gcval[i] >= fcval_cur[i];
                if (fcval_cur[i] > infeasibility_cur) infeasibility_cur = fcval_cur[i];
            }
            inner_done = inner_done || (prm.inner_maxeval > 0 && inner_nevals == prm.inner_maxeval);
            const bool take = prm.always_improve
                ? ((fcur < *minf && (inner_done || feasible_cur || !feasible)) || (!feasible && infeasibility_cur < infeasibility))
                : inner_done;
            if (take) {                               // :500-545
                if (!prm.inner_gradients) {
                    fcur = obj.f(n, xcur.data(), dfdx_cur.data(), obj.data);
                    if (forced()) return NLOPT_FORCED_STOP;
                    if (!eval_c(xcur.data(), fcval_cur.data(), dfcdx_cur.data())) return NLOPT_FORCED_STOP;
                }
                dd.fval = *minf = fcur;
                infeasibility = infeasibility_cur;
                fcval = fcval_cur;
                std::copy(xcur.begin(), xcur.end(), x);
                dfdx = dfdx_cur;
                dfcdx = dfcdx_cur;
                dd.dfdx = dfdx.data(); dd.dfcdx = dfcdx.data(); dd.fcval = fcval.data();
                if (infeasibility_cur == 0) feasible = true;
            }
            if ((ret = check_stop()) != NLOPT_SUCCESS) return ret;
            if (inner_done) break;
            if (fcur > gval) {                        // :550-556
                const double a = 10 * rho, b = 1.1 * (rho + (fcur - gval) / wval);
                rho = a < b ? a : b;
            }
            for (unsigned i = 0; i < m; ++i)
                if (fcval_cur[i] > gcval[i]) {
                    const double a = 10 * rhoc[i], b = 1.1 * (rhoc[i] + (fcval_cur[i] - gcval[i]) / wval);
                    rhoc[i] = a < b ? a : b;
                }
        }
        ret = NLOPT_SUCCESS;                          // :566-570: nlopt_stop_ftol, nlopt_stop_x
        if (rel_stop_host(fprev, fcur, opt->ftol_rel, opt->ftol_abs)) ret = NLOPT_FTOL_REACHED;
        {
            double dn = 0, xn = 0;
            bool below = opt->has_xtol_abs;
            for (unsigned j = 0; j < n; ++j) {
                const double w = opt->has_x_weights ? opt->x_weights[j] : 1.0;
                dn += w * std::fabs(xcur[j] - xprev[j]);
                xn += w * std::fabs(xcur[j]);
                if (opt->has_xtol_abs && std::fabs(xcur[j] - xprev[j]) >= opt->xtol_abs[j]) below = false;
            }
            if (dn < opt->xtol_rel * xn || below) ret = NLOPT_XTOL_REACHED;
        }
        if (ret != NLOPT_SUCCESS) return ret;
        rho = 0.1 * rho > 1e-5 ? 0.1 * rho : 1e-5;   // :573-590
        for (unsigned i = 0; i < m; ++i) rhoc[i] = 0.1 * rhoc[i] > 1e-5 ? 0.1 * rhoc[i] : 1e-5;
        if (k > 1)
            for (unsigned j = 0; j < n; ++j) {
                const double dx2 = (xcur[j] - xprev[j]) * (xprev[j] - xprevprev[j]);
                sigma[j] *= dx2 < 0 ? 0.7 : (dx2 > 0 ? 1.2 : 1.0);
                if (!nb200::nl_isinf(opt->ub[j]) && !nb200::nl_isinf(opt->lb[j])) {
                    const double r = opt->ub[j] - opt->lb[j];
                    sigma[j] = sigma[j] < 10 * r ? sigma[j] : 10 * r;
                    sigma[j] = sigma[j] > 1e-8 * r ? sigma[j] : 1e-8 * r;
                }
                sigma[j] = sigma[j] > prm.sigma_min ? sigma[j] : prm.sigma_min;
            }
    }
}

bool stop_x_host(const nlopt_opt opt, const double *x, const double *oldx)      // nlopt_stop_x, stop.c:98-108
{
    const unsigned n = opt->n;
    const double *w = opt->has_x_weights ? opt->x_weights.data() : nullptr;
    double dn = 0, xn = 0;
    if (w) {
        for (unsigned i = 0; i < n; ++i) dn += w[i] * std::fabs(x[i] - oldx[i]);
        for (unsigned i = 0; i < n; ++i) xn += w[i] * std::fabs(x[i]);
    } else {
        for (unsigned i = 0; i < n; ++i) dn += std::fabs(x[i] - oldx[i]);
        for (unsigned i = 0; i < n; ++i) xn += std::fabs(x[i]);
    }
    if (dn < opt->xtol_rel * xn) return true;
    if (!opt->has_xtol_abs) return false;
    for (unsigned i = 0; i < n; ++i)
        if (std::fabs(x[i] - oldx[i]) >= opt->xtol_abs[i]) return false;
    return true;
}

// x_dev: the sub-problem starts from (and returns into) this device array instead of host x
nlopt_result optimize_limited(nlopt_opt sub, double *x, double *x_dev, double *minf, int maxeval, double maxtime)   // optimize.c:1087-1113
{
    const int save_maxeval = sub->maxeval;
    const double save_maxtime = sub->maxtime;
    if (save_maxeval <= 0 || (maxeval > 0 && maxeval < save_maxeval)) sub->maxeval = maxeval;
    if (save_maxtime <= 0 || (maxtime > 0 && maxtime < save_maxtime)) sub->maxtime = maxtime;
    const nlopt_result ret = x_dev ? nlopt_b200_optimize_device(sub, x_dev, minf) : nlopt_optimize(sub, x, minf);
    sub->maxeval = save_maxeval;
    sub->maxtime = save_maxtime;
    return ret;
}

// A run whose x is on the device (x_dev, nlopt_b200_optimize_device) or that has a device callback takes the device
// outer loop: xcur and the best x live in HBM in a values-only backend, each sub-problem is nlopt_b200_optimize_device on
// xcur, and f, h and c are evaluated at xcur as values only, settled with one host synchronisation (host callbacks of a
// mixed run see x copied down once per evaluation).  Host x is uploaded once and downloaded once.  Both loops share the
// scalar logic below.
nlopt_result run_auglag(nlopt_opt opt, double *x, double *x_dev, double *minf)
{
    const unsigned n = opt->n;
    const nlopt_algorithm alg = opt->algorithm;
    if (opt->maximize || (!x && !x_dev)) { set_err(opt, "NULL args to nlopt_optimize_"); return NLOPT_INVALID_ARGS; }
    bool dev = x_dev != nullptr || !opt->objective.host(), sharded = opt->objective.sharded();
    for (const auto *list : {&opt->fc, &opt->h})
        for (const auto &c : *list) {
            dev = dev || !c.fn.host();
            sharded = sharded || c.fn.sharded();
        }
    if (sharded) {
        set_err(opt, "NLOPT_AUGLAG* does not take sharded host callbacks (nlopt_b200_sfunc) in this library");
        return NLOPT_INVALID_ARGS;
    }
    const bool dev_bounds = device_mode(opt);
    if (dev_bounds) {                                /* optimize.c:547-551 on the device, host x or device x */
        if (!device_mode_runs_here(opt)) return NLOPT_INVALID_ARGS;
        nb200::StartCheck start;
        std::string err;
        if (!opt->dbounds->check(x, x ? nullptr : x_dev, &start, &err)) {
            set_err(opt, "%s", err.c_str());
            return NLOPT_FAILURE;
        }
        if (start.bad >= 0) {
            set_err(opt, "bounds %d fail %g <= %g <= %g", (int) start.bad, start.lb, start.x, start.ub);
            return NLOPT_INVALID_ARGS;
        }
    } else if (x)
        for (unsigned i = 0; i < n; ++i)             /* optimize.c:547-551 */
            if (opt->lb[i] > opt->ub[i] || x[i] < opt->lb[i] || x[i] > opt->ub[i]) {
                set_err(opt, "bounds %d fail %g <= %g <= %g", (int) i, opt->lb[i], x[i], opt->ub[i]);
                return NLOPT_INVALID_ARGS;
            }
    if (!device_options_run_here(opt)) return NLOPT_INVALID_ARGS;
    if ((alg == NLOPT_AUGLAG || alg == NLOPT_AUGLAG_EQ) && !opt->local_opt) {
        set_err(opt, "local optimizer must be specified for AUGLAG");
        return NLOPT_INVALID_ARGS;
    }
    nlopt_opt sub = opt->local_opt;
    const bool own_sub = !sub;
    if (!sub) {                                      /* optimize.c:919-928 */
        if (alg == NLOPT_LN_AUGLAG || alg == NLOPT_LN_AUGLAG_EQ) {
            set_err(opt, "the default derivative-free local optimizer is not part of this library; set LD_MMA or LD_CCSAQ with nlopt_set_local_optimizer");
            return NLOPT_INVALID_ARGS;
        }
        sub = nlopt_create(g_local_deriv, n);          /* nlopt_local_search_alg_deriv: LD_MMA unless changed */
        if (!sub) { set_err(opt, "failed to create local_opt"); return NLOPT_FAILURE; }
        nlopt_set_ftol_rel(sub, opt->ftol_rel);
        nlopt_set_ftol_abs(sub, opt->ftol_abs);
        nlopt_set_xtol_rel(sub, opt->xtol_rel);
        nlopt_set_maxeval(sub, g_local_maxeval);
    }
    struct Cleanup {
        nlopt_opt opt, sub;
        bool own;
        ~Cleanup()
        {
            sub->penalty = nullptr;
            sub->objective.negate = false;
            opt->force_stop_child = nullptr;
            if (own) nlopt_destroy(sub);
        }
    } cleanup{opt, sub, own_sub};
    if (sub->algorithm != NLOPT_LD_MMA && sub->algorithm != NLOPT_LD_CCSAQ) {
        set_err(opt, "local optimizer %s is not part of this library (only LD_MMA and LD_CCSAQ are built)",
                nlopt_algorithm_to_string(sub->algorithm));
        return NLOPT_INVALID_ARGS;
    }
    if (own_sub && opt->has_xtol_abs) {            /* device options go device to device */
        if (!opt->xtol_abs_dev.dev) nlopt_set_xtol_abs(sub, opt->xtol_abs.data());
        else if (!copy_device_option(opt, opt->xtol_abs_dev, sub->xtol_abs_dev, sub->has_xtol_abs)) return NLOPT_FAILURE;
    }
    if (opt->has_dx) {
        if (!opt->dx_dev.dev) nlopt_set_initial_step(sub, opt->dx.data());
        else if (!copy_device_option(opt, opt->dx_dev, sub->dx_dev, sub->has_dx)) return NLOPT_FAILURE;
    }
    opt->force_stop_child = sub;

    const bool sub_has_fc = alg == NLOPT_AUGLAG_EQ || alg == NLOPT_LN_AUGLAG_EQ || alg == NLOPT_LD_AUGLAG_EQ;
    const std::vector<nb200::ConstraintRec> none;
    const std::vector<nb200::ConstraintRec> &pen_fc = sub_has_fc ? none : opt->fc;     /* auglag.c:98-101 */
    const std::vector<nb200::ConstraintRec> &sub_fc = sub_has_fc ? opt->fc : none;
    unsigned mm = 0, pp = 0;
    for (const auto &c : pen_fc) mm += c.fn.m;
    for (const auto &c : opt->h) pp += c.fn.m;

    nb200::PenaltySpec pen;
    std::vector<double> lambda(pp ? pp : 1, 0.0), mu(mm ? mm : 1, 0.0);
    for (const auto &c : opt->h) pen.eq.push_back(c.fn);
    for (const auto &c : pen_fc) pen.ineq.push_back(c.fn);
    pen.lambda = lambda.data();
    pen.mu = mu.data();
    opt->numevals = 0;
    pen.nevals_p = &opt->numevals;
    pen.force_stop = &opt->force_stop;

    /* configure the sub-optimiser (auglag.c:107-137).  Its objective is f + penalties: f goes in as its plain
       objective, the rest as the penalty spec */
    sub->objective = opt->objective;    /* negate too: a maximised device objective's sub-problem L starts from -f */
    sub->objective.pre = nullptr;       /* auglag.c:109-135: the sub-problem takes no preconditioner */
    sub->objective.dpre = nullptr;
    sub->maximize = 0;
    if (dev_bounds) {                                /* D2D into the sub-optimiser, which is then in device mode */
        std::string err;
        if (!opt->dbounds->copy_into(&sub->dbounds, &err)) {
            set_err(opt, "%s", err.c_str());
            return NLOPT_FAILURE;
        }
        sub->lb_ub_mirror = false;
    } else {
        nlopt_set_lower_bounds(sub, opt->lb.data());
        nlopt_set_upper_bounds(sub, opt->ub.data());
    }
    sub->lb_uniform = opt->lb_uniform;
    sub->ub_uniform = opt->ub_uniform;
    nlopt_set_stopval(sub, (mm == 0 && pp == 0) ? opt->stopval : -kInf);
    if (mm != 0 || pp != 0)
        if (sub->xtol_rel <= 0 && sub->ftol_rel <= 0) nlopt_set_xtol_rel(sub, opt->xtol_rel > 0 ? opt->xtol_rel : 1e-8);
    {   /* the sub-optimiser borrows the callbacks: its munge hooks must not touch the user's data */
        const nlopt_munge md = sub->munge_on_destroy, mc = sub->munge_on_copy;
        sub->munge_on_destroy = sub->munge_on_copy = nullptr;
        nlopt_remove_inequality_constraints(sub);
        nlopt_remove_equality_constraints(sub);
        sub->munge_on_destroy = md;
        sub->munge_on_copy = mc;
    }
    for (const auto &c : sub_fc) {
        FuncSpec fn = c.fn;
        fn.pre = nullptr;                   /* as the objective's */
        fn.dpre = nullptr;
        const nlopt_result r = add_any(sub, false, fn, c.tol.data());
        if (r < 0) return r;
    }
    sub->penalty = &pen;

    /* the device outer loop's xcur, best x and callback workspace: objective, then h, then the penalty inequalities */
    std::unique_ptr<nb200::Backend> ev;
    nlopt_b200_stats ev_stats{};
    if (dev) {
        nb200::BackendConfig vc;
        vc.values_only = true;
        vc.n = n;
        vc.objective = opt->objective;
        for (const auto &c : opt->h) vc.constraints.push_back(c.fn);
        for (const auto &c : pen_fc) vc.constraints.push_back(c.fn);
        vc.lb = opt->lb.data();
        vc.ub = opt->ub.data();
        vc.x0_host = x;
        vc.x_dev = x_dev;
        vc.x_weights = opt->has_x_weights && !opt->x_weights_dev.dev ? opt->x_weights.data() : nullptr;
        vc.xtol_abs = opt->has_xtol_abs && !opt->xtol_abs_dev.dev ? opt->xtol_abs.data() : nullptr;
        vc.x_weights_dev = opt->x_weights_dev.dev ? opt->x_weights_dev.dev->data() : nullptr;
        vc.xtol_abs_dev = opt->xtol_abs_dev.dev ? opt->xtol_abs_dev.dev->data() : nullptr;
        vc.stats = &ev_stats;
        std::string err;
        ev.reset(nb200::make_backend(vc, &err));
        if (!ev) { set_err(opt, "%s", err.c_str()); return NLOPT_FAILURE; }
        if (ev->ranks() > 1) {   /* DESIGN.md section 8 */
            set_err(opt, "NLOPT_AUGLAG* with device callbacks or device x runs on one GPU in this library");
            return NLOPT_INVALID_ARGS;
        }
    } else if (!host_option(opt, opt->x_weights_dev, opt->x_weights) || !host_option(opt, opt->xtol_abs_dev, opt->xtol_abs))
        return NLOPT_FAILURE;                        /* stop_x_host reads device options through their host mirrors */

    const double t_start = nb200::wall_seconds();
    auto forced = [&] { return opt->force_stop != 0; };
    std::vector<double> xcur, hv(pp ? pp : 1), cv(mm ? mm : 1), dv(pp + mm + 1);
    if (!dev) xcur.assign(x, x + n);

    // f, h and c at xcur (auglag.c:159-170, :212-240), values only; NLOPT_FORCED_STOP as soon as a callback asks for it
    auto eval_point = [&](double *f) -> nlopt_result {
        ++opt->numevals;
        if (!dev) {
            *f = opt->objective.f(n, xcur.data(), nullptr, opt->objective.data);
            if (forced()) return NLOPT_FORCED_STOP;
            unsigned i = 0;
            for (const auto &c : opt->h) {
                eval_host(c.fn, n, xcur.data(), hv.data() + i, nullptr);
                i += c.fn.m;
                if (forced()) return NLOPT_FORCED_STOP;
            }
            i = 0;
            for (const auto &c : pen_fc) {
                eval_host(c.fn, n, xcur.data(), cv.data() + i, nullptr);
                i += c.fn.m;
                if (forced()) return NLOPT_FORCED_STOP;
            }
            return NLOPT_SUCCESS;
        }
        bool ok = ev->eval_objective(nb200::kBase, false, f);
        if (ok && forced()) return NLOPT_FORCED_STOP;
        for (unsigned ic = 0, row = 0; ok && ic < ev->num_constraint_objects(); row += ev->constraint_dim(ic++)) {
            ok = ev->eval_constraint(nb200::kBase, ic, row, false, dv.data() + row);
            if (ok && forced()) return NLOPT_FORCED_STOP;
        }
        if (!ok || !ev->finish_evals(f, dv.data())) {
            set_err(opt, "outer evaluation: %s", ev->error().c_str());
            return NLOPT_FAILURE;
        }
        std::copy(dv.begin(), dv.begin() + pp, hv.begin());
        std::copy(dv.begin() + pp, dv.begin() + pp + mm, cv.begin());
        return NLOPT_SUCCESS;
    };
    // nlopt_stop_x(xcur, x) (stop.c:98-108), then x <- xcur
    auto keep_xcur = [&](bool *stop_x) -> bool {
        if (!dev) {
            *stop_x = stop_x_host(opt, xcur.data(), x);
            std::memcpy(x, xcur.data(), sizeof(double) * n);
            return true;
        }
        double dn, xn;
        bool below;
        if (!ev->stop_x_keep(&dn, &xn, &below)) {
            set_err(opt, "outer stop test: %s", ev->error().c_str());
            return false;
        }
        *stop_x = dn < opt->xtol_rel * xn || (opt->has_xtol_abs && below);
        return true;
    };

    /* magic parameters from Birgin & Martinez (auglag.c:85-87) */
    const double tau = 0.5, gam = 10, lam_min = -1e20, lam_max = 1e20, mu_max = 1e20;
    double ICM = HUGE_VAL, minf_penalty = HUGE_VAL, penalty = 0, fcur = 0;
    int feasible = 0, minf_feasible = 0;
    *minf = HUGE_VAL;

    const int verbose = (int) nlopt_get_param(opt, "verbosity", 0);
    int iters = 0;
    auto outer = [&]() -> nlopt_result {
        nlopt_result ret = NLOPT_SUCCESS;
        if (pp > 0 || mm > 0) {                      /* starting rho, auglag.c:155-190 */
            double con2 = 0;
            if ((ret = eval_point(&fcur)) != NLOPT_SUCCESS) return ret;
            penalty = 0;
            feasible = 1;
            unsigned ii = 0;
            for (const auto &c : opt->h)
                for (unsigned k = 0; k < c.fn.m; ++k) {
                    const double hi = hv[ii++];
                    penalty += std::fabs(hi);
                    feasible = feasible && std::fabs(hi) <= c.tol[k];
                    con2 += hi * hi;
                }
            ii = 0;
            for (const auto &c : pen_fc)
                for (unsigned k = 0; k < c.fn.m; ++k) {
                    const double fci = cv[ii++];
                    penalty += fci > 0 ? fci : 0;
                    feasible = feasible && fci <= c.tol[k];
                    if (fci > 0) con2 += fci * fci;
                }
            *minf = fcur;
            minf_penalty = penalty;
            minf_feasible = feasible;
            const double r0 = 2 * std::fabs(*minf) / con2;
            pen.rho = con2 > 0 ? std::max(1e-6, std::min(10.0, r0)) : 10;
        } else
            pen.rho = 1;

        do {                                         /* auglag.c:204-296 */
            const double prev_ICM = ICM;
            ret = optimize_limited(sub, xcur.data(), dev ? ev->point_device() : nullptr, &fcur, opt->maxeval - opt->numevals,
                                   opt->maxtime - (nb200::wall_seconds() - t_start));
            if (ret < 0) {
                if (sub->has_errmsg) set_err(opt, "%s", sub->errmsg.c_str());
                break;
            }
            if (dev) ev->point_moved();
            if ((ret = eval_point(&fcur)) != NLOPT_SUCCESS) return ret;
            ICM = 0;
            penalty = 0;
            feasible = 1;
            unsigned ii = 0;
            for (const auto &c : opt->h)
                for (unsigned k = 0; k < c.fn.m; ++k) {
                    const double hi = hv[ii];
                    const double newlam = lambda[ii] + pen.rho * hi;
                    penalty += std::fabs(hi);
                    feasible = feasible && std::fabs(hi) <= c.tol[k];
                    ICM = std::max(ICM, std::fabs(hi));
                    lambda[ii++] = std::min(std::max(lam_min, newlam), lam_max);
                }
            ii = 0;
            for (const auto &c : pen_fc)
                for (unsigned k = 0; k < c.fn.m; ++k) {
                    const double fci = cv[ii];
                    const double newmu = mu[ii] + pen.rho * fci;
                    penalty += fci > 0 ? fci : 0;
                    feasible = feasible && fci <= c.tol[k];
                    ICM = std::max(ICM, std::fabs(std::max(fci, -mu[ii] / pen.rho)));
                    mu[ii++] = std::min(std::max(0.0, newmu), mu_max);
                }
            if (ICM > tau * prev_ICM) pen.rho *= gam;
            ++iters;
            if (verbose)
                std::printf("auglag %d: ICM=%g (%sfeasible), rho=%g, fcur=%g\n", iters, ICM, feasible ? "" : "not ", pen.rho, fcur);

            if ((feasible && (!minf_feasible || penalty < minf_penalty || fcur < *minf)) || (!minf_feasible && penalty < minf_penalty)) {
                bool stop_x = false;
                if (!keep_xcur(&stop_x)) return NLOPT_FAILURE;          /* nlopt_stop_x(xcur, x), x <- xcur */
                ret = NLOPT_SUCCESS;
                if (feasible) {
                    if (fcur < opt->stopval) ret = NLOPT_STOPVAL_REACHED;
                    else if (rel_stop_host(*minf, fcur, opt->ftol_rel, opt->ftol_abs)) ret = NLOPT_FTOL_REACHED;
                    else if (stop_x) ret = NLOPT_XTOL_REACHED;
                }
                *minf = fcur;
                minf_penalty = penalty;
                minf_feasible = feasible;
                if (ret != NLOPT_SUCCESS) break;
            }
            if (forced()) { ret = NLOPT_FORCED_STOP; break; }
            if (opt->maxeval > 0 && opt->numevals >= opt->maxeval) { ret = NLOPT_MAXEVAL_REACHED; break; }
            if (opt->maxtime > 0 && nb200::wall_seconds() - t_start >= opt->maxtime) { ret = NLOPT_MAXTIME_REACHED; break; }
            if (ICM == 0) { ret = NLOPT_FTOL_REACHED; break; }
        } while (true);
        opt->stats = sub->stats;
        return ret;
    };
    nlopt_result ret = outer();
    if (dev && !ev->fetch_x(x ? x : x_dev) && ret > 0) {          /* the best x, once */
        set_err(opt, "copying the result back failed: %s", ev->error().c_str());
        ret = NLOPT_FAILURE;
    }
    return ret;
}

}  // namespace
