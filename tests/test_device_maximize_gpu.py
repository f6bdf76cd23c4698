"""Maximisation with __device__ and sharded objectives on the GPU: the bit contract.

The library minimises -f for a maximised device or sharded objective: it negates the final value (after the sum over
ranks and finish) and the gradient (negate_kernel on the library stream).  Negation is exact and a sum of negated
terms in the same tree is the negated sum, so a maximisation of Negated<F> (problems.cu: term -F, gradient -grad F,
finish(s) = -F.finish(-s)) must be the minimisation of F bit for bit: the same result code, evaluation count and
dual-evaluation count, the same bits of x*, and opt_f == -f* bitwise.

The host path of maximisation (nlopt_set_max_objective) is checked against the reference elsewhere
(test_host_driver*.py, test_auglag.py); the last cases tie the device path to it with Python callbacks that return the
device functor's bits (the reduction model of test_device_callbacks_gpu.py).
"""
import numpy as np
import pytest

import nlopt_b200 as nl
from test_auglag_device_gpu import (EPS, SEED, constraint_twin, make_opt, quad_terms, same_bits, solve, twin)

AUGLAG_IDS = {"AUGLAG": nl.AUGLAG, "AUGLAG_EQ": nl.AUGLAG_EQ, "LN_AUGLAG": nl.LN_AUGLAG, "LN_AUGLAG_EQ": nl.LN_AUGLAG_EQ,
              "LD_AUGLAG": nl.LD_AUGLAG, "LD_AUGLAG_EQ": nl.LD_AUGLAG_EQ}
LOCALS = {"MMA": nl.LD_MMA, "CCSAQ": nl.LD_CCSAQ}
FORMS = ("dfunc2", "sync")
ENTRIES = ("host", "device")
SIZES = (20011, 250000)        # one group per virtual shard / many groups per virtual shard
TOL = 1e-6


def _rows(n, m=4):
    from nlopt_b200.problems import linear_weights
    return np.stack([linear_weights(k, n) for k in range(m)]), [0.5 + 0.1 * k for k in range(m)]


# problem -> (lower bound, upper bound, x0(n), maxeval)
PROBLEMS = {
    "quad": (-1.0, 1.0, lambda n: np.full(n, 0.25), 30),              # quadratic + mean(x) + 0.1 <= 0
    "rosen": (-2.0, 2.0, None, 12),                                    # chained Rosenbrock (halo 1) + LinearRowsDev<4>
    "simp_eq": (1e-3, 1.0, lambda n: np.full(n, 0.3), 40),             # SIMP + volume equality (AUGLAG)
    "simp_sharded": (1e-3, 1.0, lambda n: np.full(n, 0.3), 30),        # sharded SIMP + sharded volume inequality
    "simp": (1e-3, 1.0, lambda n: np.full(n, 0.4), 25),                # SIMP alone
}


def register(o, p, prob, form, maximize, n, tol=TOL):
    sync = form == "sync"
    if prob == "quad":
        (p.set_quadratic_device_max if maximize else p.set_quadratic_device)(o, SEED, sync=sync)
        p.add_mean_device(o, 0.1, tol, sync)
    elif prob == "rosen":
        p.set_rosenbrock_device(o, sync=sync, maximize=maximize)
        W, b = _rows(n)
        p.add_linear_rows_device(o, W, b, 1e-8)
    elif prob == "simp_eq":
        (p.set_simp_device_max if maximize else p.set_simp_device)(o, SEED, EPS, sync=sync)
        p.add_mean_device_eq(o, -0.4, tol, sync)
    elif prob == "simp_sharded":
        (p.simp_sharded_max if maximize else p.simp_sharded)(o, SEED, EPS, 0.4, tol)
    else:
        (p.set_simp_device_max if maximize else p.set_simp_device)(o, SEED, EPS, sync=sync)


def run(alg, prob, n, form, entry, maximize, local=None, stopval=None, maxeval=None, x0=None, tol=TOL):
    """((ret, numevals, opt_f, x), dual_evals) of one run"""
    from nlopt_b200.problems import Problem, rosen_x0
    p = Problem()
    lo, hi, x0f, me = PROBLEMS[prob]
    o = nl.opt(alg, n)
    o.set_lower_bounds(lo)
    o.set_upper_bounds(hi)
    o.set_maxeval(maxeval or me)
    o.set_ftol_rel(1e-10)
    if local is not None:
        sub = nl.opt(local, n)
        sub.set_ftol_rel(1e-8)
        o.set_local_optimizer(sub)
    register(o, p, prob, form, maximize, n, tol)
    if stopval is not None:
        o.set_stopval(stopval)
    if x0 is None:
        x0 = rosen_x0(n) if prob == "rosen" else x0f(n)
    r = solve(o, x0, entry)
    assert r[0] > 0, o.get_errmsg()
    return r, o.get_stats()["dual_evals"]


def assert_max_is_min(mx, mn):
    """mx: the max run of Negated<F>, mn: the min run of F"""
    (a, da), (b, db) = mx, mn
    assert a[0] == b[0], (a[0], b[0])
    assert a[1] == b[1], (a[1], b[1])
    assert da == db, (da, db)
    assert same_bits(a[2], -b[2]), (a[2], b[2])
    assert same_bits(a[3], b[3]), np.flatnonzero(a[3] != b[3])[:8]


# ---- LD_MMA / LD_CCSAQ ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("prob", ["quad", "rosen"])
@pytest.mark.parametrize("alg", [nl.LD_MMA, nl.LD_CCSAQ], ids=["MMA", "CCSAQ"])
def test_ccsa_max_equals_min(built, alg, prob, n, form, entry):
    mn = run(alg, prob, n, form, entry, False)
    mx = run(alg, prob, n, form, entry, True)
    assert_max_is_min(mx, mn)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("alg", [nl.LD_MMA, nl.LD_CCSAQ], ids=["MMA", "CCSAQ"])
def test_sharded_max_equals_min(built, alg, n, entry):
    mn = run(alg, "simp_sharded", n, "sharded", entry, False)
    mx = run(alg, "simp_sharded", n, "sharded", entry, True)
    assert_max_is_min(mx, mn)


# ---- the AUGLAG family --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("local", list(LOCALS))
@pytest.mark.parametrize("alg", list(AUGLAG_IDS))
def test_auglag_max_equals_min(built, alg, local, n, form, entry):
    a, lo = AUGLAG_IDS[alg], LOCALS[local]
    mn = run(a, "simp_eq", n, form, entry, False, local=lo)
    mx = run(a, "simp_eq", n, form, entry, True, local=lo)
    assert_max_is_min(mx, mn)


# ---- stopval: S on the max run, -S on the min run ----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["MMA", "CCSAQ", "LD_AUGLAG"])
def test_stopval_stops_both_at_the_same_evaluation(built, case):
    """S = -nextafter(f_K, +inf), f_K the best value of a min run of K evaluations from a feasible start: the min run with
    stopval -S and the max run with stopval S both stop with STOPVAL_REACHED, at the same evaluation.  LD_AUGLAG runs SIMP
    without constraints, whose sub-problem takes the outer stopval (auglag.c), so that the stop is certain to come"""
    n, form, entry = 20011, "dfunc2", "device"
    if case == "LD_AUGLAG":
        kw = dict(alg=nl.LD_AUGLAG, prob="simp", local=nl.LD_MMA)
    else:
        kw = dict(alg=nl.LD_MMA if case == "MMA" else nl.LD_CCSAQ, prob="quad", x0=np.full(n, -0.25))
    alg, prob = kw.pop("alg"), kw.pop("prob")
    (ret_k, evals_k, f_k, _), _ = run(alg, prob, n, form, entry, False, maxeval=25, **kw)
    s_min = float(np.nextafter(f_k, np.inf))
    mn = run(alg, prob, n, form, entry, False, stopval=s_min, **kw)
    mx = run(alg, prob, n, form, entry, True, stopval=-s_min, **kw)
    assert mn[0][0] == nl.STOPVAL_REACHED, (mn[0][0], ret_k, evals_k)
    assert mn[0][1] <= evals_k
    assert_max_is_min(mx, mn)


# ---- registration from Python through exported pointers ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_python_registration_with_exported_pointers(built, form):
    """the pointers the C++ front end registers, handed to opt.set_max_objective_device2 / set_max_objective_device (and
    the min twins): the same runs as nb200p_set_quadratic_device_max / the min registration"""
    from nlopt_b200.problems import Problem
    n = 20011

    def go(maximize, how):
        p = Problem()
        o = nl.opt(nl.LD_MMA, n)
        o.set_lower_bounds(-1.0)
        o.set_upper_bounds(1.0)
        o.set_maxeval(20)
        if how == "front_end":
            (p.set_quadratic_device_max if maximize else p.set_quadratic_device)(o, SEED, sync=form == "sync")
        else:
            fn, fin, data = p.quadratic_pointers(o, SEED, negated=maximize, sync=form == "sync")
            if form == "sync":
                (o.set_max_objective_device if maximize else o.set_min_objective_device)(fn, data)
            else:
                (o.set_max_objective_device2 if maximize else o.set_min_objective_device2)(fn, fin, data, halo=0)
        p.add_mean_device(o, 0.1, TOL)
        r = solve(o, np.full(n, 0.25), "device")
        assert r[0] > 0, o.get_errmsg()
        return r, o.get_stats()["dual_evals"]

    mn_py, mn_fe = go(False, "pointers"), go(False, "front_end")
    mx_py, mx_fe = go(True, "pointers"), go(True, "front_end")
    assert_max_is_min(mx_fe, mn_fe)
    for a, b in ((mn_py, mn_fe), (mx_py, mx_fe)):
        assert a[0][:2] == b[0][:2] and a[1] == b[1]
        assert same_bits(a[0][2], b[0][2]) and same_bits(a[0][3], b[0][3])


# ---- device max against the library's host max path --------------------------------------------------------------------
def neg_quad_terms(x):
    t, g = quad_terms(x)
    return -t, -g


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("alg", ["LD_MMA", "LD_AUGLAG"])
def test_device_max_matches_host_max_path(built, alg, form, entry):
    """Negated<QuadraticDev> maximised on the device against nlopt_set_max_objective with a Python callback that returns
    the same bits (numpy terms, the device reduction model, Negated's finish); constraints likewise.  LD_AUGLAG: sphere
    equality and mean inequality (test_auglag_device_gpu's LD_AUGLAG case), outer xtol_rel = 0."""
    from nlopt_b200.problems import Problem
    n, sync = 20011, form == "sync"
    neg_finish = lambda s: -(0.5 * -s)      # noqa: E731  (Negated<QuadraticDev>::finish)

    def make():
        if alg == "LD_AUGLAG":
            return make_opt("LD_AUGLAG", n)
        o = nl.opt(nl.LD_MMA, n)
        o.set_lower_bounds(-1.0)
        o.set_upper_bounds(1.0)
        o.set_maxeval(30)
        o.set_ftol_rel(1e-10)
        return o

    p = Problem()
    od = make()
    p.set_quadratic_device_max(od, SEED, sync=sync)
    if alg == "LD_AUGLAG":
        p.add_sphere_device_eq(od, 0.2, TOL, sync)
    p.add_mean_device(od, 0.1, TOL, sync)
    got = solve(od, np.full(n, 0.25), entry)

    oh = make()
    oh.set_max_objective(twin(neg_quad_terms, neg_finish, form))
    if alg == "LD_AUGLAG":
        oh.add_equality_constraint(constraint_twin("sphere", 0.2, n, form), TOL)
    oh.add_inequality_constraint(constraint_twin("mean", 0.1, n, form), TOL)
    want = solve(oh, np.full(n, 0.25), "host")

    assert want[0] > 0, oh.get_errmsg()
    assert got[0] == want[0] and got[1] == want[1], (got[:2], want[:2])
    assert same_bits(got[2], want[2]), (got[2], want[2])
    assert same_bits(got[3], want[3]), np.flatnonzero(got[3] != want[3])[:8]
