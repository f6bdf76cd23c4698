"""Vector __device__ constraints on the GPU: the multi-row kernels against the model of the scalar summation order, and
whole runs against twins made of scalar device functors or host callbacks, bit for bit.

Component i of a vector functor is reduced in exactly the order of a scalar functor (test_device_callbacks_gpu.py has
the model), so a run with one LinearRowsDev<m> must be the same run as with m LinearDev rows: same result code,
evaluation count, dual-evaluation count and bits of opt_f and x.
"""
import ctypes as C

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi
from test_auglag_device_gpu import SEED, assert_same_run, same_bits, solve
from test_device_callbacks_gpu import EDGE_SIZES, adversarial_x, hash_terms, model_dfunc2
from test_device_mconstraints import mprobe, mprobe_so  # noqa: F401  (fixtures)

TERM, HASH = 0, 1


class MFunctor:
    """one vector probe functor (ids k_id .. k_id + m - 1) and its witness counters; keep it alive while its opt runs"""

    def __init__(self, L, kind, m, k_id, n, seed=0, offset=0.0):
        import torch
        self.L, self.kind, self.m, self.k_id, self.n = L, kind, m, k_id, n
        self.visits = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        self.counters = torch.zeros(2, dtype=torch.int32, device="cuda")       # errors, calls with a gradient
        cp = self.counters.data_ptr()
        self.h = L.probe_mnew(kind, m, k_id, seed, offset, n, self.visits.data_ptr(), cp, cp + 4)
        assert self.h

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            self.L.probe_mfree(self.kind, self.m, h)

    def register(self, o, equality=False, tol=None):
        t = None if tol is None else np.ascontiguousarray(tol, dtype=np.float64)
        o._check(self.L.probe_mregister(o._h, self.kind, self.m, self.h, int(equality), None if t is None else t.ctypes.data))
        self._tol = t

    def totals(self, i):
        cnt = self.L.probe_mtotals(self.k_id + i, None, 0)
        buf = (C.c_double * max(cnt, 1))()
        self.L.probe_mtotals(self.k_id + i, buf, cnt)
        return [buf[k] for k in range(cnt)]

    def check_witness(self, evals):
        visits = self.visits[:self.n].cpu().numpy()
        errors, grad_calls = self.counters.cpu().tolist()
        bad = np.flatnonzero(visits != evals)
        assert bad.size == 0, f"m {self.m}: {bad.size} variables not visited {evals}x, first {bad[:5]} -> {visits[bad[:5]]}"
        assert errors == 0, f"m {self.m}: {errors} calls with a wrong j, n, n_local or jl"
        assert grad_calls == self.n * evals, (self.m, grad_calls, self.n * evals)


def terms(kind, k_id, x, seed):
    return np.ldexp(x, k_id) if kind == TERM else hash_terms(x.size, k_id, seed)


# ---- 1. totals against the model ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("m", (1, 3, 4, 16))
def test_component_totals_match_the_scalar_model(mprobe, m):
    """every size of EDGE_SIZES: component i's total is model_dfunc2 of its terms, bit for bit; each variable is visited
    once per evaluation (not m times), with the right indices and a gradient pointer"""
    import torch
    from nlopt_b200.problems import Problem
    kind = HASH if m == 3 else TERM
    seed = 0x5EED4321
    for n in EDGE_SIZES:
        mprobe.probe_mreset()
        x = adversarial_x(n)
        f = MFunctor(mprobe, kind, m, 20, n, seed=seed, offset=0.5)
        p = Problem()
        o = nl.opt(nl.LD_MMA, n)
        o.set_maxeval(1)
        p.set_quadratic_device(o)
        f.register(o, tol=np.full(m, 1e-8))
        xd = torch.from_numpy(x.copy()).cuda()
        o.optimize_device(xd.data_ptr())
        torch.cuda.synchronize()
        for i in range(m):
            want = model_dfunc2(terms(kind, 20 + i, x, seed))
            got = f.totals(i)
            assert len(got) == 1 and same_bits(got[0], want), (n, m, i, got, want)
        f.check_witness(1)
        del f, o, xd
        torch.cuda.empty_cache()


# ---- 2. vector = scalar, whole runs ---------------------------------------------------------------------------------
def rosen_run(alg, n, m, form, entry, maxeval=12):
    from nlopt_b200.problems import Problem, rosen_x0
    p = Problem()
    o = nl.opt(alg, n)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_maxeval(maxeval)
    if form == "scalar":
        p.rosenbrock_device(o, m)
    else:
        p.rosenbrock_device_rows(o, m)
    r = solve(o, rosen_x0(n), entry)
    return r, o.get_stats()["dual_evals"]


def assert_same_with_duals(a, b):
    (ra, da), (rb, db) = a, b
    assert_same_run(ra, rb)
    assert da == db, (da, db)


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("n", (20011, 250000, 10**7))
@pytest.mark.parametrize("alg", [nl.LD_MMA, nl.LD_CCSAQ], ids=["MMA", "CCSAQ"])
def test_linear_rows_run_equals_four_linear_functors(built, alg, n, entry):
    want = rosen_run(alg, n, 4, "scalar", entry)
    got = rosen_run(alg, n, 4, "vector", entry)
    assert want[0][0] > 0
    assert_same_with_duals(got, want)


# ---- 3. mixed registration order -------------------------------------------------------------------------------------
def host_rows(W, b):
    """an nlopt_mfunc c = W x - b (the same host function in both runs)"""
    def f(result, x, grad):
        result[:] = W @ x - b
        if grad.size:
            grad[:] = W
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("n", (20011, 250000))
def test_mixed_registration_order(built, n):
    """vector device rows, a host nlopt_mfunc, a scalar device row and a second vector device object, against the
    all-scalar twin: the row offsets of every kind of constraint object line up"""
    from nlopt_b200.problems import Problem, linear_weights, rosen_x0
    W = np.stack([linear_weights(k, n) for k in range(7)])
    b = 0.5 + 0.1 * np.arange(7)

    def run(form):
        p = Problem()
        o = nl.opt(nl.LD_MMA, n)
        o.set_lower_bounds(-2.0)
        o.set_upper_bounds(2.0)
        o.set_maxeval(12)
        o._check(p.L.nb200p_set_rosenbrock_device(p.h, o._h))

        def scalar(k):
            w = np.ascontiguousarray(W[k])
            o._check(p.L.nb200p_add_linear_device(p.h, o._h, w.ctypes.data_as(_capi.c_double_p), b[k], 1e-8))

        if form == "vector":
            p.add_linear_rows_device(o, W[0:2], b[0:2], 1e-8)
        else:
            scalar(0)
            scalar(1)
        o.add_inequality_mconstraint(host_rows(W[2:4], b[2:4]), np.full(2, 1e-8))
        scalar(4)
        if form == "vector":
            p.add_linear_rows_device(o, W[5:7], b[5:7], 1e-8)
        else:
            scalar(5)
            scalar(6)
        r = solve(o, rosen_x0(n), "device")
        return r, o.get_stats()["dual_evals"]

    want, got = run("scalar"), run("vector")
    assert want[0][0] > 0
    assert_same_with_duals(got, want)


# ---- 4. more than 16 rows ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", (20011, 250000))
def test_twenty_rows_wide_kernel(built, n):
    """LinearRowsDev<16> + LinearRowsDev<4>: 20 rows, past the fused solve (wide kernel, host dual optimiser)"""
    from nlopt_b200.problems import Problem, linear_weights, rosen_x0

    def run(form):
        p = Problem()
        o = nl.opt(nl.LD_MMA, n)
        o.set_lower_bounds(-2.0)
        o.set_upper_bounds(2.0)
        o.set_maxeval(8)
        if form == "scalar":
            p.rosenbrock_device(o, 20)
        else:
            o._check(p.L.nb200p_set_rosenbrock_device(p.h, o._h))
            W = np.stack([linear_weights(k, n) for k in range(20)])
            b = 0.5 + 0.1 * np.arange(20)
            p.add_linear_rows_device(o, W[:16], b[:16], 1e-8)
            p.add_linear_rows_device(o, W[16:], b[16:], 1e-8)
        r = solve(o, rosen_x0(n), "device")
        return r, o.get_stats()["dual_evals"]

    want, got = run("scalar"), run("vector")
    assert want[0][0] > 0
    assert_same_with_duals(got, want)


# ---- 5. AUGLAG ----------------------------------------------------------------------------------------------------------
def block_mean_twin(n, targets):
    """the host nlopt_mfunc of BlockMeanDev<M>: model totals of x inside block i (+0.0 outside), then s / |block| - t_i"""
    M = len(targets)
    edge = [i * n // M for i in range(M + 1)]
    inv_len = [1.0 / (edge[i + 1] - edge[i]) for i in range(M)]

    def h(result, x, grad):
        for i in range(M):
            t = np.zeros(n)
            t[edge[i]:edge[i + 1]] = x[edge[i]:edge[i + 1]]
            result[i] = model_dfunc2(t) * inv_len[i] - targets[i]
        if grad.size:
            grad[:] = 0.0
            for i in range(M):
                grad[i, edge[i]:edge[i + 1]] = inv_len[i]
    return h


AUG_CASES = {"LD_AUGLAG": nl.LD_AUGLAG, "LD_AUGLAG_EQ": nl.LD_AUGLAG_EQ}


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("n", (20011, 250000))
@pytest.mark.parametrize("case", list(AUG_CASES))
def test_auglag_vector_equality_and_inequality(built, case, n, entry):
    """quadratic objective, BlockMeanDev<4> equalities and LinearRowsDev<2> inequalities, against a twin with a host
    nlopt_mfunc of the model values for the equalities and two scalar LinearDev for the inequalities.  LD_AUGLAG_EQ
    hands the inequalities to its sub-problem"""
    from nlopt_b200.problems import Problem, linear_weights
    targets = [0.2, 0.25, 0.3, 0.22]
    W = np.stack([linear_weights(k, n) for k in range(2)])
    b = np.array([0.1, 0.05])

    def run(form):
        p = Problem()
        o = nl.opt(AUG_CASES[case], n)
        o.set_lower_bounds(-1.0)
        o.set_upper_bounds(1.0)
        o.set_maxeval(40)
        o.set_ftol_rel(1e-10)
        p.set_quadratic_device(o, SEED)
        if form == "vector":
            p.add_block_mean_device_eq(o, targets, 1e-6)
            p.add_linear_rows_device(o, W, b, 1e-6)
        else:
            o.add_equality_mconstraint(block_mean_twin(n, targets), np.full(4, 1e-6))
            for k in range(2):
                w = np.ascontiguousarray(W[k])
                o._check(p.L.nb200p_add_linear_device(p.h, o._h, w.ctypes.data_as(_capi.c_double_p), b[k], 1e-6))
        return solve(o, np.full(n, 0.25), entry)

    want, got = run("scalar"), run("vector")
    assert want[0] > 0, want[0]
    assert_same_run(got, want)


# ---- 6. Python registration through function pointers -------------------------------------------------------------
@pytest.mark.gpu
def test_python_registration_with_exported_pointers(mprobe):
    """opt.add_inequality_mconstraint_device with the probe's exported nlopt_b200_dmfunc2 / dmfinish pair gives the same
    totals and opt_f as the template front end"""
    import torch
    from nlopt_b200.problems import Problem
    n, m = 100003, 4
    x = adversarial_x(n)

    def run(how):
        mprobe.probe_mreset()
        f = MFunctor(mprobe, TERM, m, 40, n, offset=0.5)
        p = Problem()
        o = nl.opt(nl.LD_MMA, n)
        o.set_maxeval(1)
        p.set_quadratic_device(o)
        if how == "python":
            o.add_inequality_mconstraint_device(mprobe.probe_mfunc_ptr(TERM, m), mprobe.probe_mfinish_ptr(TERM, m), f.h,
                                                np.full(m, 1e-8))
        else:
            f.register(o, tol=np.full(m, 1e-8))
        xd = torch.from_numpy(x.copy()).cuda()
        o.optimize_device(xd.data_ptr())
        torch.cuda.synchronize()
        f.check_witness(1)
        return o.last_optimum_value(), [f.totals(i) for i in range(m)]

    a, b = run("python"), run("template")
    assert same_bits(a[0], b[0])
    for i in range(m):
        want = model_dfunc2(np.ldexp(x, 40 + i))
        assert len(a[1][i]) == 1 and same_bits(a[1][i][0], want), (i, a[1][i], want)
        assert same_bits(a[1][i][0], b[1][i][0])
