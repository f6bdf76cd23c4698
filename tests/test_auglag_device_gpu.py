"""NLOPT_AUGLAG* with __device__ functors and device-resident x.

The library's host-callback AUGLAG path is checked against the reference (test_auglag.py).  Here every device run is
compared with a twin run of that host path whose Python callbacks return the same bits: numpy terms in the device
functor's order of operations, folded with the model of the device reduction (test_device_callbacks_gpu.py), then the
functor's finish().  Gradients are single IEEE operations on both sides.  Equal bits in, the same trajectory out: the
device run must give the same result code, the same number of evaluations and the same bits of opt_f and x.

Outer xtol_rel = 0 in the bit-for-bit cases: the device outer loop sums the nlopt_stop_x norms in the library's group
order, the host loop sequentially, and a test right at the threshold could then decide differently.  The runs that
end on the x test use a threshold far from either sum (see test_device_stop_pass_matches_host_twin).
"""
import ctypes as C
import shutil
import subprocess

import numpy as np
import pytest

import nlopt_b200 as nl
import synth
from nlopt_b200 import _capi

SEED = 0x5EED0000
EPS = 1e-3
AUGLAG_IDS = (nl.AUGLAG, nl.AUGLAG_EQ, nl.LN_AUGLAG, nl.LN_AUGLAG_EQ, nl.LD_AUGLAG, nl.LD_AUGLAG_EQ)
FORMS = ("dfunc2", "sync")
SIZES = (20011, 250000)        # one group per virtual shard / many groups per virtual shard
DFUNC2 = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
DFINISH = C.CFUNCTYPE(C.c_double, C.c_double, C.c_void_p)


def same_bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


# ---- registration (C ABI; the API layer linked against the CPU test backend) ------------------------------------
@pytest.fixture(scope="module")
def cbs():
    """callables to register: their addresses only; none of them is called"""
    f2 = DFUNC2(lambda *a: None)
    fin = DFINISH(lambda t, d: t)
    f1 = _capi.NLOPT_B200_DFUNC(lambda *a: 0.0)
    return {"f2": C.cast(f2, C.c_void_p), "fin": C.cast(fin, C.c_void_p), "f1": C.cast(f1, C.c_void_p), "_keep": (f2, fin, f1)}


def _eq_device(L, h, cbs, form, tol=0.0, halo=0, fn=True, fin=True):
    if form == "sync":
        return L.dll.nlopt_b200_add_equality_constraint_device(C.c_void_p(h), cbs["f1"] if fn else None, None, C.c_double(tol))
    return L.dll.nlopt_b200_add_equality_constraint_device2(C.c_void_p(h), cbs["f2"] if fn else None, cbs["fin"] if fin else None,
                                                            None, C.c_double(tol), C.c_int(halo))


def _errmsg(L, h):
    L.dll.nlopt_get_errmsg.restype = C.c_char_p
    m = L.dll.nlopt_get_errmsg(C.c_void_p(h))
    return m.decode() if m else None


@pytest.mark.parametrize("form", FORMS)
def test_equality_device_registration_follows_equality_ok(hosttest_lib, cbs, form):
    L = hosttest_lib
    host_h = _capi.NLOPT_FUNC(lambda n, x, g, d: 0.0)
    for alg in (nl.LD_MMA, nl.LD_CCSAQ):
        o1, o2 = L.nlopt_create(alg, 3), L.nlopt_create(alg, 3)
        want = L.nlopt_add_equality_constraint(o1, host_h, None, 0.0)
        got = _eq_device(L, o2, cbs, form)
        assert got == want == nl.INVALID_ARGS
        assert _errmsg(L, o2) == _errmsg(L, o1) == "invalid algorithm for constraints"
        L.nlopt_destroy(o1)
        L.nlopt_destroy(o2)
    for alg in AUGLAG_IDS:
        o = L.nlopt_create(alg, 3)
        assert _eq_device(L, o, cbs, form, tol=1e-6) == nl.SUCCESS
        L.nlopt_destroy(o)


def test_equality_device_argument_checks(hosttest_lib, cbs):
    L = hosttest_lib
    o = L.nlopt_create(nl.LD_AUGLAG, 3)
    assert _eq_device(L, o, cbs, "dfunc2", fn=False) == nl.INVALID_ARGS
    assert _eq_device(L, o, cbs, "dfunc2", fin=False) == nl.INVALID_ARGS
    assert _eq_device(L, o, cbs, "dfunc2", halo=2) == nl.INVALID_ARGS
    assert _eq_device(L, o, cbs, "dfunc2", halo=-1) == nl.INVALID_ARGS
    assert _eq_device(L, o, cbs, "dfunc2", tol=-1e-3) == nl.INVALID_ARGS
    assert _errmsg(L, o) == "negative constraint tolerance"
    assert _eq_device(L, o, cbs, "sync", fn=False) == nl.INVALID_ARGS
    assert _eq_device(L, o, cbs, "sync", tol=-1e-3) == nl.INVALID_ARGS
    assert _eq_device(L, o, cbs, "dfunc2", halo=1) == nl.SUCCESS
    L.nlopt_destroy(o)


def test_remove_equality_constraints_clears_device_equalities(hosttest_lib, cbs):
    """With a device equality left in place the run would take the device outer loop, which the CPU test backend
    cannot evaluate; once removed, the run is the plain host run."""
    def solve(with_device_eq):
        o = nl.opt(nl.LD_AUGLAG, 2, library=hosttest_lib)
        o.set_lower_bounds([-2.0, -2.0])
        o.set_upper_bounds([2.0, 2.0])
        o.set_min_objective(lambda x, g: (g.__setitem__(slice(None), 2 * x) if g.size else None, float(x @ x))[1])
        o.set_maxeval(30)
        o.add_inequality_constraint(lambda x, g: (g.__setitem__(slice(None), -1.0) if g.size else None, 1.0 - x.sum())[1], 1e-8)
        if with_device_eq:
            for form in FORMS:
                assert _eq_device(hosttest_lib, o._h, cbs, form) == nl.SUCCESS
            o.remove_equality_constraints()
        x = o.optimize([1.0, 1.5])
        return o.last_optimize_result(), o.get_numevals(), o.last_optimum_value(), x

    a, b = solve(True), solve(False)
    assert a[0] > 0 and a[:2] == b[:2] and same_bits(a[2], b[2]) and same_bits(a[3], b[3])


def test_problems_library_exports_the_equality_helpers(built):
    """Building problems.cu instantiates add_equality_constraint / add_equality_constraint_sync for its functors."""
    from nlopt_b200 import problems
    L = problems.lib()
    for name in ("nb200p_add_mean_device_eq", "nb200p_add_linear_device_eq", "nb200p_add_sphere_device_eq",
                 "nb200p_set_quadratic_device_sync", "nb200p_set_simp_device_sync", "nb200p_add_mean_device_sync"):
        assert getattr(L, name)


def test_problems_library_finishes_are_not_contracted(built):
    """The twins below compute finish() as separate IEEE operations (MeanDev: s * inv_n + offset, SphereDev:
    s * inv_n - r); the host code of problems.cu must not fuse them into an FMA."""
    from nlopt_b200 import problems
    if not shutil.which("objdump"):
        pytest.skip("objdump not available")
    dis = subprocess.run(["objdump", "-d", "--no-show-raw-insn", problems.LIB_PATH], stdout=subprocess.PIPE, text=True,
                         check=True).stdout
    assert "vfmadd" not in dis and "vfmsub" not in dis and "vfnmadd" not in dis


def test_sharded_callbacks_and_default_ln_local_optimizer_are_refused(built):
    from nlopt_b200.problems import Problem
    p = Problem()
    o = nl.opt(nl.LD_AUGLAG, 1000)
    o.set_lower_bounds(0.0)
    o.set_upper_bounds(1.0)
    p.simp_sharded(o)
    assert o._lib.nlopt_optimize(o._h, np.full(1000, 0.4).ctypes.data_as(_capi.c_double_p), C.byref(C.c_double())) == nl.INVALID_ARGS
    assert "sharded" in o.get_errmsg()
    o2 = nl.opt(nl.LN_AUGLAG, 1000)
    o2.set_lower_bounds(0.0)
    o2.set_upper_bounds(1.0)
    p.simp_device_eq(o2)
    assert o2._lib.nlopt_optimize(o2._h, np.full(1000, 0.4).ctypes.data_as(_capi.c_double_p), C.byref(C.c_double())) == nl.INVALID_ARGS
    assert "derivative-free local optimizer" in o2.get_errmsg()


# ---- host twins of problems.cu's functors ---------------------------------------------------------------------------
_U01 = {}


def u01(k, n):
    if (k, n) not in _U01:
        _U01[(k, n)] = synth.u01(k, n, SEED)
    return _U01[(k, n)]


def quad_terms(x):
    n = x.size
    a = 1.0 + u01(0, n)
    b = 2.0 * u01(1, n) - 1.0
    d = x - b
    ad = a * d
    return ad * d, ad


def simp_terms(x):
    n = x.size
    a = 0.5 + u01(0, n)
    x2 = x * x
    x3 = x2 * x
    ome = 1.0 - EPS
    d = EPS + ome * x3
    return a / d, -(((a * (ome * 3.0)) * x2) / (d * d))


def twin(terms, finish, form):
    """an nlopt_func returning finish(device total) with the device's gradient"""
    from test_device_callbacks_gpu import model_dfunc2, model_sync
    fold = model_dfunc2 if form == "dfunc2" else model_sync

    def f(x, grad):
        t, g = terms(x)
        if grad.size:
            grad[:] = g
        return finish(fold(t))
    return f


def constraint_twin(kind, arg, n, form):
    inv_n = 1.0 / n
    if kind == "mean":
        return twin(lambda x: (x.copy(), np.full(x.size, inv_n)), lambda s: s * inv_n + arg, form)
    if kind == "sphere":
        return twin(lambda x: (x * x, 2.0 * x), lambda s: s * inv_n - arg, form)
    from nlopt_b200.problems import linear_weights
    w = linear_weights(0, n)
    return twin(lambda x: (w * x, w), lambda s: s - arg, form)


# algorithm, local optimiser, objective, bounds, x0, equalities, inequalities ((kind, argument) pairs)
CASES = {
    "LD_AUGLAG": (nl.LD_AUGLAG, None, "quad", (-1.0, 1.0), 0.25, [("sphere", 0.2)], [("mean", 0.1)]),
    "LD_AUGLAG_EQ": (nl.LD_AUGLAG_EQ, None, "quad", (-1.0, 1.0), 0.25, [("linear", -0.05)], [("mean", -0.3)]),
    "AUGLAG_CCSAQ": (nl.AUGLAG, nl.LD_CCSAQ, "simp", (1e-3, 1.0), 0.3, [("mean", -0.4)], []),
    "AUGLAG_EQ_MMA": (nl.AUGLAG_EQ, nl.LD_MMA, "quad", (-1.0, 1.0), 0.25, [("mean", 0.1)], [("mean", -0.5)]),
}


def make_opt(case, n, maxeval=40, xtol_rel=0.0, tol=1e-6):
    alg, local, _, (lo, hi), _, _, _ = CASES[case]
    o = nl.opt(alg, n)
    o.set_lower_bounds(lo)
    o.set_upper_bounds(hi)
    o.set_maxeval(maxeval)
    o.set_ftol_rel(1e-10)
    o.set_xtol_rel(xtol_rel)
    if local is not None:
        lo_ = nl.opt(local, n)
        lo_.set_ftol_rel(1e-8)
        o.set_local_optimizer(lo_)
    return o


def register(o, case, n, how, form, p=None, host_eq=None, tol=1e-6):
    """how: 'device' (problems.cu functors) or 'host' (numpy twins)"""
    from nlopt_b200.problems import linear_weights
    _, _, obj, _, _, eqs, ineqs = CASES[case]
    sync = form == "sync"
    if how == "device":
        (p.set_quadratic_device if obj == "quad" else p.set_simp_device)(o, SEED, **({} if obj == "quad" else {"eps": EPS}), sync=sync)
    else:
        o.set_min_objective(twin(quad_terms, lambda s: 0.5 * s, form) if obj == "quad" else twin(simp_terms, lambda s: s, form))
    for kind, arg in eqs:
        if host_eq is not None:
            o.add_equality_constraint(host_eq, tol)
        elif how == "device":
            if kind == "mean":
                p.add_mean_device_eq(o, arg, tol, sync)
            elif kind == "sphere":
                p.add_sphere_device_eq(o, arg, tol, sync)
            else:
                p.add_linear_device_eq(o, linear_weights(0, n), arg, tol, sync)
        else:
            o.add_equality_constraint(constraint_twin(kind, arg, n, form), tol)
    for kind, arg in ineqs:
        if how == "device":
            p.add_mean_device(o, arg, tol, sync)
        else:
            o.add_inequality_constraint(constraint_twin(kind, arg, n, form), tol)


def solve(o, x0, entry):
    """(ret, numevals, opt_f, x) without raising on negative results"""
    f = C.c_double(0.0)
    if entry == "host":
        x = np.array(x0, dtype=np.float64)
        ret = o._lib.nlopt_optimize(o._h, x.ctypes.data_as(_capi.c_double_p), C.byref(f))
    else:
        import torch
        xd = torch.from_numpy(np.array(x0, dtype=np.float64)).cuda()
        ret = o._lib.nlopt_b200_optimize_device(o._h, C.c_void_p(xd.data_ptr()), C.byref(f))
        torch.cuda.synchronize()
        x = xd.cpu().numpy()
    return ret, o.get_numevals(), f.value, x


_TWINS = {}


def host_twin_run(case, n, form, **kw):
    key = (case, n, form, tuple(sorted(kw.items())))
    if key not in _TWINS:
        o = make_opt(case, n, **kw)
        register(o, case, n, "host", form)
        _TWINS[key] = solve(o, np.full(n, CASES[case][4]), "host")
    return _TWINS[key]


def device_run(case, n, form, entry, **kw):
    from nlopt_b200.problems import Problem
    p = Problem()
    o = make_opt(case, n, **kw)
    register(o, case, n, "device", form, p)
    r = solve(o, np.full(n, CASES[case][4]), entry)
    assert r[0] >= 0, o.get_errmsg()
    return r, o


def assert_same_run(a, b):
    assert a[0] == b[0], (a[0], b[0])
    assert a[1] == b[1], (a[1], b[1])
    assert same_bits(a[2], b[2]), (a[2], b[2])
    assert same_bits(a[3], b[3]), np.flatnonzero(a[3] != b[3])[:8]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("case", list(CASES))
def test_device_run_matches_host_twin(built, case, n, form, entry):
    want = host_twin_run(case, n, form)
    got, _ = device_run(case, n, form, entry)
    assert want[0] > 0
    assert_same_run(got, want)


def _mixed(n, how, stop_at=None, maxeval=40):
    """quadratic objective (device functor or its twin) and a host equality mean(x) = -0.1 (the same host function in
    both runs), LD_AUGLAG over MMA; stop_at: the equality calls nlopt_force_stop at its stop_at-th call"""
    from nlopt_b200.problems import Problem
    p = Problem()
    o = make_opt("LD_AUGLAG", n, maxeval=maxeval)
    calls = [0]

    def h(x, grad):
        calls[0] += 1
        if stop_at is not None and calls[0] == stop_at:
            o.force_stop()
        if grad.size:
            grad[:] = 1.0 / x.size
        return float(np.sum(x)) / x.size + 0.1

    if how == "device":
        p.set_quadratic_device(o, SEED)
    else:
        o.set_min_objective(twin(quad_terms, lambda s: 0.5 * s, "dfunc2"))
    o.add_equality_constraint(h, 1e-6)
    return solve(o, np.full(n, 0.25), "device" if how == "device" else "host"), calls[0]


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_mixed_run_matches_host_twin(built, n):
    (got, calls_d), (want, calls_h) = _mixed(n, "device"), _mixed(n, "host")
    assert want[0] > 0
    assert_same_run(got, want)
    assert calls_d == calls_h


@pytest.mark.gpu
def test_forced_stop_from_host_callback(built):
    (got, _), (want, _) = _mixed(20011, "device", stop_at=9), _mixed(20011, "host", stop_at=9)
    assert got[0] == want[0] == nl.FORCED_STOP
    assert got[1] == want[1]


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_maxeval_stop(built, form):
    want = host_twin_run("LD_AUGLAG", 20011, form, maxeval=7)
    got, _ = device_run("LD_AUGLAG", 20011, form, "device", maxeval=7)
    assert want[0] == nl.MAXEVAL_REACHED
    assert_same_run(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("weights", [False, True])
def test_device_stop_pass_matches_host_twin(built, weights):
    """Runs that end on nlopt_stop_x, evaluated by the device stop pass.  xtol_rel = 1e-3 (and xtol_abs = 1e-3 with
    weights): relative to an L1 norm of 2e4 terms the two summation orders differ by about 1e-12, nine orders below
    the threshold, and the accepted steps of an outer iteration change by far more than that between iterations."""
    n = 20011
    kw = dict(maxeval=400, xtol_rel=1e-3)

    def run(how):
        from nlopt_b200.problems import Problem
        p = Problem()
        o = make_opt("AUGLAG_EQ_MMA", n, **kw)
        o.set_ftol_rel(0.0)
        if weights:
            o.set_x_weights(0.5 + u01(5, n))
            o.set_xtol_abs(1e-3)
        register(o, "AUGLAG_EQ_MMA", n, how, "dfunc2", p, tol=1e-3)
        return solve(o, np.full(n, 0.25), "device" if how == "device" else "host")

    want, got = run("host"), run("device")
    assert want[0] == nl.XTOL_REACHED
    assert_same_run(got, want)


@pytest.mark.gpu
def test_simp_volume_equality_at_scale(built):
    """SIMP with a volume equality at n = 1e7 through optimize_device, against the same run with problems.cu's C host
    callbacks; the bytes the last sub-run moved over PCIe do not grow with n"""
    import torch
    from nlopt_b200.problems import Problem
    tol = 1e-6

    def run(n, how):
        p = Problem()
        o = nl.opt(nl.LD_AUGLAG, n)
        o.set_lower_bounds(1e-3)
        o.set_upper_bounds(1.0)
        o.set_ftol_rel(1e-8)
        o.set_maxeval(120)
        (p.simp_device_eq if how == "device" else p.simp_host_eq)(o, SEED, EPS, 0.4, tol)
        r = solve(o, np.full(n, 0.4), "device" if how == "device" else "host")
        return r, o.get_stats()

    bytes_ = {}
    for n in (10**6, 10**7):
        (ret, evals, f, x), st = run(n, "device")
        assert ret > 0
        bytes_[n] = st["h2d_bytes"] + st["d2h_bytes"]
        if n == 10**7:
            assert abs(np.mean(x) - 0.4) <= tol
            (ret_h, _, f_h, _), _ = run(n, "host")
            assert ret_h > 0
            assert abs(f - f_h) <= 1e-6 * abs(f_h), (f, f_h)
        del x
        torch.cuda.empty_cache()
    assert bytes_[10**6] == bytes_[10**7], bytes_
