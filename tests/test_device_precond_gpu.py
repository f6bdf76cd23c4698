"""Preconditioned CCSAQ with device preconditioners (nlopt_b200_dprecond), on the H100.

The problem is test_host_driver.py's precond_problem, f(x) = 1/2 x^T A x - b^T x with A = tridiag(-1, d_j, -1) and H = A,
plus one linear constraint, written here with PyTorch terms callbacks and a PyTorch preconditioner.  The device path
(nested LD_MMA on the model, everything in HBM) is checked against the library's host path (nlopt_precond, numpy) at
the optimum, which test_host_driver.py pins to the reference; maximisation and the runs that ignore preconditioners are
checked bit for bit.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import dual_sums_model as dsm
import nlopt_b200 as nl
import outer_model as om
from nlopt_b200 import _capi
from nlopt_b200 import problems as nlp

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_SRC = os.path.join(ROOT, "tests", "cpp", "precond_model_probe.cu")
PROBE_SO = os.path.join(ROOT, "tests", "_build", "libprecond_model_probe.so")
EDGE_SIZES = (1, 255, 256, 257, 511, 512, 513, 4095, 4097, 100003, 10**7)


@pytest.fixture(scope="session")
def probe(built):
    """tests/cpp/precond_model_probe.cu -> tests/_build/: the library's precond.cu kernels and terms reduction"""
    g = built
    deps = [PROBE_SRC, g.LIB, os.path.join(ROOT, "nlopt_b200", "csrc", "precond.cu"),
            os.path.join(ROOT, "nlopt_b200", "csrc", "terms_kernels.cuh")]
    if not os.path.exists(PROBE_SO) or any(os.path.getmtime(d) > os.path.getmtime(PROBE_SO) for d in deps):
        os.makedirs(os.path.dirname(PROBE_SO), exist_ok=True)
        tmp = PROBE_SO + f".{os.getpid()}.tmp"
        r = subprocess.run([g.NVCC, *g.ARCH, *g.NVCC_FLAGS, "-shared", PROBE_SRC, "-o", tmp, "-cudart", "shared",
                            "-L" + os.path.dirname(g.LIB), "-lnlopt_b200", "-Xlinker", "-rpath=$ORIGIN/../../nlopt_b200"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        os.replace(tmp, PROBE_SO)
    L = C.CDLL(PROBE_SO, mode=C.RTLD_LOCAL)
    P, U, D = C.c_void_p, C.c_ulonglong, C.c_double
    L.probe_box.argtypes = [U, P, P, D, D, P, P, P, P, P]
    L.probe_dx.argtypes = [U, P, P, P]
    L.probe_model.argtypes = [U, P, P, P, P, D, P, P, P]
    L.probe_w.argtypes = [U, P, P, P, P]
    L.probe_sum.argtypes = [U, P, P]
    return L


def ptr(a):
    return None if a is None else a.ctypes.data


def bits_equal(got, want):
    """bit for bit, NaN for NaN (the payload of a NaN is the hardware's)"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint64), want[~nan].view(np.uint64))


def problem(n, seed=3):
    """the numbers of test_host_driver.py:precond_problem (same generator, same seed)"""
    rng = np.random.default_rng(seed)
    d = 2.5 + rng.random(n)
    b = rng.standard_normal(n)
    w = (1.0 + 0.5 * np.sin(0.37 * np.arange(n))) / n
    return d, b, w


def A_np(d, v):
    out = d * v
    out[:-1] -= v[1:]
    out[1:] -= v[:-1]
    return out


def A_t(d, v):
    out = d * v
    out[:-1] -= v[1:]
    out[1:] -= v[:-1]
    return out


def torch_funcs(n, sign=1.0):
    """objective terms, constraint terms and preconditioner on cuda:0; sign -1: the negated objective and H"""
    d, b, w = (torch.tensor(a, dtype=torch.float64, device="cuda") for a in problem(n))

    def f(x, g):
        Ax = A_t(d, x)
        if g.numel():
            g.copy_(sign * (Ax - b))
        return sign * (0.5 * x * Ax - b * x)

    def c(x, g):
        if g.numel():
            g.copy_(w)
        return w * x

    def pre(x, v, vpre):
        vpre.copy_(sign * A_t(d, v))

    return f, c, pre


def configure(o, n, maxeval=60):
    o.set_lower_bounds(np.full(n, -2.0))
    o.set_upper_bounds(np.full(n, 2.0))
    o.set_xtol_rel(1e-9)
    o.set_maxeval(maxeval)
    o.set_param("dual_ftol_rel", 1e-12)


def run_device(n, with_constraint_pre, alg=nl.LD_CCSAQ, maximize=False, with_pre=True, maxeval=60):
    f, c, pre = torch_funcs(n, -1.0 if maximize else 1.0)
    o = nl.opt(alg, n)
    configure(o, n, maxeval)
    (o.set_max_objective_torch if maximize else o.set_min_objective_torch)(f)
    o.add_inequality_constraint_torch(c, 1e-8, finish=lambda t: t + 0.05)
    if with_pre:
        o.set_objective_precond_torch(pre)
        if with_constraint_pre:
            o.set_constraint_precond_torch(0, lambda x, v, vpre: vpre.zero_())
    x = o.optimize(np.zeros(n))
    return dict(ret=o.last_optimize_result(), x=x, f=o.last_optimum_value(), numevals=o.get_numevals(), stats=o.get_stats())


def run_host(n, with_constraint_pre):
    d, b, w = problem(n)

    def f(x, g):
        Ax = A_np(d, x)
        if g.size:
            g[:] = Ax - b
        return float(0.5 * x @ Ax - b @ x)

    def c(x, g):
        if g.size:
            g[:] = w
        return float(w @ x) + 0.05

    o = nl.opt(nl.LD_CCSAQ, n)
    configure(o, n)
    o.set_precond_min_objective(f, lambda x, v, vpre: vpre.__setitem__(slice(None), A_np(d, v)))
    if with_constraint_pre:
        o.add_precond_inequality_constraint(c, lambda x, v, vpre: vpre.__setitem__(slice(None), 0.0), 1e-8)
    else:
        o.add_inequality_constraint(c, 1e-8)
    x = o.optimize(np.zeros(n))
    return dict(ret=o.last_optimize_result(), x=x, f=o.last_optimum_value())


def kkt_residual(n, x):
    d, b, w = problem(n)
    g = A_np(d, x) - b
    lam = -float(g @ w) / float(w @ w)
    return lam, float(np.max(np.abs(g + lam * w)))


def same_bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


@pytest.mark.parametrize("with_constraint_pre", [False, True])
def test_device_path_reaches_the_host_paths_optimum(with_constraint_pre):
    n = 60
    a = run_device(n, with_constraint_pre)
    h = run_host(n, with_constraint_pre)
    assert a["ret"] > 0 and h["ret"] > 0, (a["ret"], h["ret"])
    assert abs(a["f"] - h["f"]) <= 1e-7 * max(1.0, abs(h["f"]))
    assert np.max(np.abs(a["x"] - h["x"])) <= 1e-5
    lam, res = kkt_residual(n, a["x"])
    assert lam > 0 and res <= 1e-4, (lam, res)
    st = a["stats"]
    assert st["dual_solves"] > 0 and st["dual_evals"] > 0 and st["kernel_launches"] > 0


def test_maximising_the_negation_is_the_same_run():
    n = 60
    mn = run_device(n, True)
    mx = run_device(n, True, maximize=True)
    assert mx["ret"] == mn["ret"] and mx["numevals"] == mn["numevals"]
    assert same_bits(mx["f"], -mn["f"]) and same_bits(mx["x"], mn["x"])


@pytest.mark.parametrize("alg", [nl.LD_MMA, nl.LD_AUGLAG_EQ])
def test_runs_that_ignore_preconditioners_are_unchanged(alg):
    n = 60

    def run(with_pre):
        if alg == nl.LD_MMA:
            return run_device(n, True, alg=alg, with_pre=with_pre)
        f, c, pre = torch_funcs(n)
        o = nl.opt(alg, n)
        configure(o, n, maxeval=200)
        sub = nl.opt(nl.LD_CCSAQ, n)
        sub.set_xtol_rel(1e-7)
        o.set_local_optimizer(sub)
        o.set_min_objective_torch(f)
        o.add_inequality_constraint_torch(c, 1e-8, finish=lambda t: t + 0.05)
        if with_pre:
            o.set_objective_precond_torch(pre)
            o.set_constraint_precond_torch(0, lambda x, v, vpre: vpre.zero_())
        x = o.optimize(np.zeros(n))
        return dict(ret=o.last_optimize_result(), x=x, f=o.last_optimum_value(), numevals=o.get_numevals())

    a, b = run(True), run(False)
    assert a["ret"] == b["ret"] and a["numevals"] == b["numevals"]
    assert same_bits(a["f"], b["f"]) and same_bits(a["x"], b["x"])


def test_a_raising_preconditioner_stops_the_run():
    n = 60
    f, c, _ = torch_funcs(n)
    o = nl.opt(nl.LD_CCSAQ, n)
    configure(o, n)
    o.set_min_objective_torch(f)
    o.add_inequality_constraint_torch(c, 1e-8, finish=lambda t: t + 0.05)

    class Boom(Exception):
        pass

    def pre(x, v, vpre):
        raise Boom("preconditioner failed")

    o.set_objective_precond_torch(pre)
    with pytest.raises(Boom):
        o.optimize(np.zeros(n))
    assert o.last_optimize_result() == nl.FORCED_STOP


def test_large_n_stays_on_the_device():
    """n = 1e6 with device x, device bounds and a torch tridiagonal preconditioner (the exact Hessian, so the model is
    exact): the run converges to the box-constrained minimiser (projected gradient) and moves fewer than 8 n bytes
    between host and device over the whole run"""
    n = 1_000_000
    f, _, pre = torch_funcs(n)
    o = nl.opt(nl.LD_CCSAQ, n)
    o.set_lower_bounds(torch.full((n,), -2.0, dtype=torch.float64, device="cuda"))
    o.set_upper_bounds(torch.full((n,), 2.0, dtype=torch.float64, device="cuda"))
    o.set_xtol_rel(1e-9)
    o.set_maxeval(40)
    o.set_param("dual_ftol_rel", 1e-12)
    o.set_min_objective_torch(f)
    o.set_objective_precond_torch(pre)
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    o.optimize_torch(x)
    st = o.get_stats()
    assert o.last_optimize_result() > 0, o.last_optimize_result()
    assert st["h2d_bytes"] + st["d2h_bytes"] < 8 * n, (st["h2d_bytes"], st["d2h_bytes"])
    d, b, _ = problem(n)
    xh = x.cpu().numpy()
    g = A_np(d, xh) - b
    at_lb, at_ub = xh <= -2.0 + 1e-9, xh >= 2.0 - 1e-9
    pg = np.where(at_lb, np.minimum(g, 0.0), np.where(at_ub, np.maximum(g, 0.0), g))
    assert np.max(np.abs(pg)) <= 1e-4, (np.max(np.abs(pg)), o.get_numevals(), o.last_optimize_result())


# ---- the kernels of precond.cu against a numpy model of ccsa_quadratic.c:153-181 and :441-446, bit for bit ------------
def model_np(dx, sigma, dfdx, hdx, rho):
    """precond_gfunc (nlopt_api.cpp) per variable: numpy float64 elementwise operations round once each, like C"""
    with np.errstate(all="ignore"):
        sigma2inv = 1.0 / (sigma * sigma)
        sterm = dfdx * dx + ((0.5 * rho) * (dx * dx)) * sigma2inv
        grad = dfdx + (rho * dx) * sigma2inv
        qterm = None
        if hdx is not None:
            qterm = (0.5 * dx) * hdx
            grad = grad + hdx
    return sterm, qterm, grad


def edge_inputs(n=4096, seed=11):
    rng = np.random.default_rng(seed)
    dx = rng.standard_normal(n) * np.exp(rng.uniform(-20, 5, n))
    sigma = np.exp(rng.uniform(-10, 3, n))
    dfdx = rng.standard_normal(n) * 1e3
    hdx = rng.standard_normal(n) * np.exp(rng.uniform(-5, 5, n))
    dx[:8] = [0.0, -0.0, 0.0, -0.0, 1e-300, -1e-300, 5e-324, -5e-324]
    sigma[8:12] = [5e-324, 1e-160, 0.0, 0.0]           # sigma^2 subnormal or zero: sigma^-2 = inf; a fixed variable
    dx[10] = 0.0                                        # 0 * inf: NaN, as on the host
    hdx[12:16] = [np.nan, np.inf, -np.inf, -0.0]
    dfdx[16:18] = [np.inf, -0.0]
    return dx, sigma, dfdx, hdx


@pytest.mark.parametrize("rho", [1.0, 1e-5, 37.5])
@pytest.mark.parametrize("with_h", [True, False])
def test_model_kernel_matches_the_host_model_bit_for_bit(probe, rho, with_h):
    dx, sigma, dfdx, hdx = edge_inputs()
    n = dx.size
    h = hdx if with_h else None
    sterm, qterm, grad = np.empty(n), np.empty(n), np.empty(n)
    assert probe.probe_model(n, ptr(dx), ptr(sigma), ptr(dfdx), ptr(h), rho, ptr(sterm), ptr(qterm), ptr(grad)) == 0
    ws, wq, wg = model_np(dx, sigma, dfdx, h, rho)
    assert bits_equal(sterm, ws) and bits_equal(grad, wg)
    if with_h:
        assert bits_equal(qterm, wq)
    sterm2 = np.empty(n)                                # values only: the same terms
    assert probe.probe_model(n, ptr(dx), ptr(sigma), ptr(dfdx), ptr(h), rho, ptr(sterm2), ptr(qterm), None) == 0
    assert bits_equal(sterm2, ws)


def test_dx_and_w_kernels_match_bit_for_bit(probe):
    rng = np.random.default_rng(5)
    n = 3000
    x, x0 = rng.standard_normal(n), rng.standard_normal(n)
    x[:4] = [0.0, -0.0, np.inf, np.nan]
    x0[:4] = [-0.0, -0.0, np.inf, 1.0]
    sigma = np.exp(rng.uniform(-8, 2, n))
    sigma[4:6] = [0.0, 5e-324]
    dx, w = np.empty(n), np.empty(n)
    assert probe.probe_dx(n, ptr(x), ptr(x0), ptr(dx)) == 0
    assert probe.probe_w(n, ptr(x), ptr(x0), ptr(sigma), ptr(w)) == 0
    with np.errstate(all="ignore"):
        assert bits_equal(dx, x - x0)
        q = (x - x0) / sigma
        assert bits_equal(w, (0.5 * q) * q)


@pytest.mark.parametrize("bounds", ["array", "scalar", "infinite", "lower_only", "upper_only"])
def test_box_kernel_matches_the_host_loop_bit_for_bit(probe, bounds):
    rng = np.random.default_rng(7)
    n = 2049
    x = rng.uniform(-3, 3, n)
    sigma = np.exp(rng.uniform(-6, 1, n))
    sigma[:3] = [0.0, np.inf, np.nan]
    lb, ub = rng.uniform(-4, -1, n), rng.uniform(1, 4, n)
    lb0, ub0 = -2.0, 2.5
    if bounds == "infinite":
        lb, ub = np.full(n, -np.inf), np.full(n, np.inf)
    elif bounds == "lower_only":
        ub = np.full(n, np.inf)
    elif bounds == "upper_only":
        lb = np.full(n, -np.inf)
    lbd, ubd = (None, None) if bounds == "scalar" else (lb, ub)
    L, Uu = (np.full(n, lb0), np.full(n, ub0)) if bounds == "scalar" else (lb, ub)
    pl, pu, xc = np.empty(n), np.empty(n), np.empty(n)
    assert probe.probe_box(n, ptr(lbd), ptr(ubd), lb0, ub0, ptr(x), ptr(sigma), ptr(pl), ptr(pu), ptr(xc)) == 0
    with np.errstate(all="ignore"):
        lo, hi = x - sigma, x + sigma
    # nlopt_api.cpp:run_ccsa_precond: lb > x - sigma ? lb : x - sigma (a NaN comparison is false: the second operand)
    assert bits_equal(pl, np.where(L > lo, L, lo)) and bits_equal(pu, np.where(Uu < hi, Uu, hi)) and bits_equal(xc, x)


@pytest.mark.parametrize("n", EDGE_SIZES)
def test_model_sums_lie_within_the_float64_bound_of_fsum(probe, n):
    """the separable, quadratic and w terms of the model through the library's terms reduction: within
    (depth + 1) 2^-53 sum|t| of math.fsum, depth that of the functor / terms fold"""
    rng = np.random.default_rng(n)
    dx = rng.standard_normal(n) * 0.1
    sigma = np.exp(rng.uniform(-3, 1, n))
    dfdx, hdx = rng.standard_normal(n), rng.standard_normal(n)
    sterm, qterm, w = np.empty(n), np.empty(n), np.empty(n)
    assert probe.probe_model(n, ptr(dx), ptr(sigma), ptr(dfdx), ptr(hdx), 0.3, ptr(sterm), ptr(qterm), None) == 0
    x0 = rng.standard_normal(n)
    xc = x0 + dx
    assert probe.probe_w(n, ptr(xc), ptr(x0), ptr(sigma), ptr(w)) == 0
    dep = dsm.depth("eval", om.geometry(n), 1)
    got = []
    for t in (sterm, qterm, w):
        tot = C.c_double()
        assert probe.probe_sum(n, ptr(t), C.byref(tot)) == 0
        got.append(tot.value)
    dsm.check_dual_sums(got, [sterm, qterm, w], dep, what=f"n={n}")


# ---- the callback forms: a C-kernel preconditioner (problems.cu) and a host objective ------------------------------
class TridiagData(C.Structure):
    _fields_ = [("d", C.c_void_p), ("sign", C.c_double)]


def c_precond(n, sign=1.0):
    """problems.cu's tridiagonal preconditioner (an nlopt_b200_dprecond) and its data; keep the returned tuple alive"""
    d = torch.tensor(problem(n)[0], dtype=torch.float64, device="cuda")
    data = TridiagData(d.data_ptr(), sign)
    fn = C.cast(getattr(nlp.lib(), "nb200p_tridiag_precond"), C.c_void_p)
    return fn, C.cast(C.pointer(data), C.c_void_p), (d, data)


def test_c_kernel_and_torch_preconditioners_give_the_same_run():
    n = 60

    def run(form):
        f, c, pre = torch_funcs(n)
        o = nl.opt(nl.LD_CCSAQ, n)
        configure(o, n)
        o.set_min_objective_torch(f)
        o.add_inequality_constraint_torch(c, 1e-8, finish=lambda t: t + 0.05)
        keep = None
        if form == "torch":
            o.set_objective_precond_torch(pre)
        else:
            fn, data, keep = c_precond(n)
            o.set_objective_precond_device(fn, data)
        x = o.optimize(np.zeros(n))
        del keep
        return dict(ret=o.last_optimize_result(), x=x, f=o.last_optimum_value(), numevals=o.get_numevals())

    a, b = run("c"), run("torch")
    assert a["ret"] > 0 and a["ret"] == b["ret"] and a["numevals"] == b["numevals"]
    assert same_bits(a["f"], b["f"]) and same_bits(a["x"], b["x"])
    h = run_host(n, False)
    assert abs(a["f"] - h["f"]) <= 1e-7 * max(1.0, abs(h["f"])) and np.max(np.abs(a["x"] - h["x"])) <= 1e-5


def test_maximising_a_host_objective_applies_minus_h():
    """a host nlopt_func objective maximised with (-F, -H) runs bit for bit like (F, H) minimised"""
    n = 60
    d, b, w = problem(n)

    def run(maximize):
        sign = -1.0 if maximize else 1.0

        def f(x, g):
            Ax = A_np(d, x)
            if g.size:
                g[:] = sign * (Ax - b)
            return sign * float(0.5 * x @ Ax - b @ x)

        _, c, _ = torch_funcs(n)
        o = nl.opt(nl.LD_CCSAQ, n)
        configure(o, n)
        (o.set_max_objective if maximize else o.set_min_objective)(f)
        o.add_inequality_constraint_torch(c, 1e-8, finish=lambda t: t + 0.05)
        fn, data, keep = c_precond(n, sign)
        o.set_objective_precond_device(fn, data)
        x = o.optimize(np.zeros(n))
        del keep
        return dict(ret=o.last_optimize_result(), x=x, f=o.last_optimum_value(), numevals=o.get_numevals())

    mn, mx = run(False), run(True)
    assert mn["ret"] > 0 and mx["ret"] == mn["ret"] and mx["numevals"] == mn["numevals"]
    assert same_bits(mx["f"], -mn["f"]) and same_bits(mx["x"], mn["x"])
