"""Maximisation with device and sharded objectives (nlopt_b200_set_max_objective_device / _device2 / _sharded): the API
layer, on the CPU-backed build of the host logic (hosttest_lib), and the sign-flip kernel's build.

The runs themselves, with the bit contract max(Negated<F>) == min(F), are in test_device_maximize_gpu.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi

AUGLAG_IDS = (nl.AUGLAG, nl.AUGLAG_EQ, nl.LN_AUGLAG, nl.LN_AUGLAG_EQ, nl.LD_AUGLAG, nl.LD_AUGLAG_EQ)
DFUNC2 = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
DFINISH = C.CFUNCTYPE(C.c_double, C.c_double, C.c_void_p)
SFUNC = C.CFUNCTYPE(C.c_double, C.c_uint, C.c_ulonglong, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p)
PRECOND_MSG = "preconditioned CCSAQ takes host x and host callbacks (nlopt_precond is a host function)"
BACKEND_MSG = "host test backend needs a host objective"
INF = float("inf")


@pytest.fixture(scope="module")
def cbs():
    """callables to register: their addresses only; none of them is called"""
    f1 = _capi.NLOPT_B200_DFUNC(lambda *a: 0.0)
    f2 = DFUNC2(lambda *a: None)
    fin = DFINISH(lambda t, d: t)
    sf = SFUNC(lambda *a: 0.0)
    keep = (f1, f2, fin, sf)
    return {"f1": C.cast(f1, C.c_void_p), "f2": C.cast(f2, C.c_void_p), "fin": C.cast(fin, C.c_void_p),
            "sf": C.cast(sf, C.c_void_p), "_keep": keep}


def _set(L, h, cbs, form, maximize, fn=True, fin=True, halo=0, data=None):
    """register an objective of the given form; returns the nlopt_result"""
    kind = "max" if maximize else "min"
    h = C.c_void_p(h)
    if form == "sync":
        return getattr(L.dll, f"nlopt_b200_set_{kind}_objective_device")(h, cbs["f1"] if fn else None, C.c_void_p(data))
    if form == "sharded":
        return getattr(L.dll, f"nlopt_b200_set_{kind}_objective_sharded")(h, cbs["sf"] if fn else None, C.c_void_p(data))
    return getattr(L.dll, f"nlopt_b200_set_{kind}_objective_device2")(h, cbs["f2"] if fn else None, cbs["fin"] if fin else None,
                                                                     C.c_void_p(data), C.c_int(halo))


def _errmsg(L, h):
    L.dll.nlopt_get_errmsg.restype = C.c_char_p
    m = L.dll.nlopt_get_errmsg(C.c_void_p(h))
    return m.decode() if m else None


def _optimize(L, h, x0):
    x = np.array(x0, dtype=np.float64)
    f = C.c_double(0.0)
    ret = L.nlopt_optimize(h, x.ctypes.data_as(_capi.c_double_p), C.byref(f))
    return ret, f.value


def test_new_entry_points_are_declared_and_exported(built):
    for name in ("nlopt_b200_set_max_objective_device", "nlopt_b200_set_max_objective_device2",
                 "nlopt_b200_set_max_objective_sharded"):
        assert name in _capi.EXT_SYMBOLS
    nl.opt(nl.LD_MMA, 3)        # the product library resolves every declared symbol


@pytest.mark.parametrize("form", ["sync", "dfunc2", "sharded"])
def test_argument_checks_mirror_the_min_forms(hosttest_lib, cbs, form):
    """every argument combination gives the max form the result code of its min twin; a NULL callback or finish and a halo
    outside {0, 1} are NLOPT_INVALID_ARGS where the min form refuses them"""
    L = hosttest_lib
    combos = [dict(), dict(fn=False)]
    if form == "dfunc2":
        combos += [dict(fin=False), dict(halo=-1), dict(halo=2), dict(halo=1)]
    for kw in combos:
        got, want = [], []
        for maximize, out in ((True, got), (False, want)):
            o = L.nlopt_create(nl.LD_MMA, 4)
            out.append(_set(L, o, cbs, form, maximize, **kw))
            L.nlopt_destroy(o)
        assert got == want, (form, kw, got, want)
        refused = kw.get("halo", 0) not in (0, 1) or not kw.get("fin", True) or (form != "sync" and not kw.get("fn", True))
        assert got[0] == (nl.INVALID_ARGS if refused else nl.SUCCESS), (form, kw, got)
    assert L.dll.nlopt_b200_set_max_objective_device2(None, cbs["f2"], cbs["fin"], None, C.c_int(0)) == nl.INVALID_ARGS


@pytest.mark.parametrize("form", ["sync", "dfunc2", "sharded"])
@pytest.mark.parametrize("stopval", [-INF, INF, -3.5, 2.0])
def test_stopval_after_registration_is_that_of_set_max_objective(hosttest_lib, cbs, form, stopval):
    """the +-inf stopval handling of nlopt_set_max_objective (options.c), and min after max restores it"""
    L = hosttest_lib
    host = _capi.NLOPT_FUNC(lambda n, x, g, d: 0.0)
    o1, o2 = L.nlopt_create(nl.LD_MMA, 4), L.nlopt_create(nl.LD_MMA, 4)
    for o in (o1, o2):
        L.nlopt_set_stopval(o, stopval)
    assert L.nlopt_set_max_objective(o1, host, None) == nl.SUCCESS
    assert _set(L, o2, cbs, form, True) == nl.SUCCESS
    assert L.nlopt_get_stopval(o2) == L.nlopt_get_stopval(o1)
    assert L.nlopt_get_stopval(o2) == (INF if stopval == -INF else stopval)
    assert L.nlopt_set_min_objective(o1, host, None) == nl.SUCCESS
    assert _set(L, o2, cbs, form, False) == nl.SUCCESS
    assert L.nlopt_get_stopval(o2) == L.nlopt_get_stopval(o1)
    L.nlopt_destroy(o1)
    L.nlopt_destroy(o2)


def _quad_opt(L, n=3):
    o = nl.opt(nl.LD_MMA, n, library=L)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_maxeval(20)
    return o


def _host_quad(x, g):
    if g.size:
        g[:] = 2 * (x - 0.5)
    return float((x - 0.5) @ (x - 0.5))


@pytest.mark.parametrize("form", ["sync", "dfunc2", "sharded"])
def test_maximising_device_objective_reaches_the_backend(hosttest_lib, cbs, form):
    """no longer refused by the API layer: the run reaches the backend, which fails with its own message (the CPU test
    backend evaluates host objectives only); opt_f is the maximisation's -HUGE_VAL, as for any failed max run"""
    L = hosttest_lib
    for alg in (nl.LD_MMA, nl.LD_CCSAQ):
        o = L.nlopt_create(alg, 3)
        L.nlopt_set_lower_bounds1(o, -1.0)
        L.nlopt_set_upper_bounds1(o, 1.0)
        assert _set(L, o, cbs, form, True) == nl.SUCCESS
        ret, f = _optimize(L, o, [0.1, 0.2, 0.3])
        assert ret == nl.FAILURE and BACKEND_MSG in _errmsg(L, o), (alg, ret, _errmsg(L, o))
        assert f == -INF
        assert L.nlopt_get_stopval(o) == INF          # restored after the run
        L.nlopt_destroy(o)
    if form != "sharded":
        # the device outer loop of AUGLAG cannot start on the CPU test backend: the max run ends exactly as the min run
        got = []
        for maximize in (True, False):
            o = L.nlopt_create(nl.LD_AUGLAG, 3)
            L.nlopt_set_lower_bounds1(o, -1.0)
            L.nlopt_set_upper_bounds1(o, 1.0)
            assert _set(L, o, cbs, form, maximize) == nl.SUCCESS
            ret, f = _optimize(L, o, [0.1, 0.2, 0.3])
            got.append((ret, _errmsg(L, o), f))
            L.nlopt_destroy(o)
        (rmax, emax, fmax), (rmin, emin, fmin) = got
        assert rmax == rmin < 0 and emax == emin and "maximisation" not in emax
        assert fmax == -fmin


def test_copy_keeps_maximize(hosttest_lib, cbs):
    """nlopt_copy carries the maximisation along: the copy's failed run reports the max run's -HUGE_VAL, where a min
    registration reports +HUGE_VAL"""
    L = hosttest_lib
    for maximize, want in ((True, -INF), (False, INF)):
        o = L.nlopt_create(nl.LD_MMA, 3)
        assert _set(L, o, cbs, "dfunc2", maximize, halo=1) == nl.SUCCESS
        c = L.nlopt_copy(o)
        assert c
        L.nlopt_destroy(o)
        assert L.nlopt_get_stopval(c) == (INF if maximize else -INF)
        ret, f = _optimize(L, c, [0.1, 0.2, 0.3])
        assert ret == nl.FAILURE and BACKEND_MSG in _errmsg(L, c)
        assert f == want
        L.nlopt_destroy(c)


def test_later_set_min_objective_clears_maximize(hosttest_lib, cbs):
    """a device max registration followed by nlopt_set_min_objective is a plain minimisation: the same run as a fresh
    min registration"""
    L = hosttest_lib
    a = _quad_opt(L)
    assert _set(L, a._h, cbs, "dfunc2", True) == nl.SUCCESS
    a.set_min_objective(_host_quad)
    b = _quad_opt(L)
    b.set_min_objective(_host_quad)
    xa, xb = a.optimize([1.5, -1.0, 0.0]), b.optimize([1.5, -1.0, 0.0])
    assert a.last_optimize_result() == b.last_optimize_result() > 0
    assert a.get_numevals() == b.get_numevals()
    assert a.last_optimum_value() == b.last_optimum_value() and np.array_equal(xa, xb)
    assert a.get_stopval() == b.get_stopval() == -INF


def test_existing_refusals_stay(hosttest_lib, cbs):
    L = hosttest_lib
    # preconditioned CCSAQ with a non-host objective (a host preconditioned constraint makes the run take that branch)
    o = nl.opt(nl.LD_CCSAQ, 3, library=L)
    o.set_lower_bounds(-1.0)
    o.set_upper_bounds(1.0)
    o.add_precond_inequality_constraint(lambda x, g: (g.__setitem__(slice(None), -1.0) if g.size else None, 1.0 - x.sum())[1],
                                        lambda x, v, vpre: vpre.__setitem__(slice(None), v), 1e-8)
    assert _set(L, o._h, cbs, "dfunc2", True) == nl.SUCCESS
    assert _optimize(L, o._h, [0.5, 0.5, 0.5])[0] == nl.INVALID_ARGS
    assert o.get_errmsg() == PRECOND_MSG
    # sharded callbacks under AUGLAG
    for alg in AUGLAG_IDS:
        h = L.nlopt_create(alg, 3)
        sub = L.nlopt_create(nl.LD_MMA, 3)
        L.nlopt_set_local_optimizer(h, sub)
        assert _set(L, h, cbs, "sharded", True) == nl.SUCCESS
        assert _optimize(L, h, [0.1, 0.2, 0.3])[0] == nl.INVALID_ARGS
        assert "sharded" in _errmsg(L, h)
        L.nlopt_destroy(sub)
        L.nlopt_destroy(h)
    # n == 0 with a non-host objective
    for form in ("sync", "dfunc2", "sharded"):
        h = L.nlopt_create(nl.LD_MMA, 0)
        assert _set(L, h, cbs, form, True) == nl.SUCCESS
        assert _optimize(L, h, [])[0] == nl.INVALID_ARGS
        assert _errmsg(L, h) == "n == 0 needs a host objective"
        L.nlopt_destroy(h)


def test_problems_library_exports_the_maximisation_helpers(built):
    from nlopt_b200 import problems
    L = problems.lib()
    for name in ("nb200p_set_quadratic_device_max", "nb200p_set_simp_device_max", "nb200p_set_rosenbrock_device_form",
                 "nb200p_quadratic_pointers", "nb200p_simp_sharded_neg"):
        assert getattr(L, name)


def test_negated_sharded_simp_negates_value_and_gradient(built):
    """nb200p_simp_sharded_neg is -nb200p_simp_sharded, value and gradient, bit for bit (host code, no device)"""
    from nlopt_b200 import problems
    L = problems.lib()
    pos = C.cast(L.nb200p_simp_sharded, SFUNC)
    neg = C.cast(L.nb200p_simp_sharded_neg, SFUNC)
    p = L.nb200p_create()
    d = L.nb200p_make_simp_data(p, 0x5EED0000, 1e-3)
    n = 1001
    x = np.linspace(1e-3, 1.0, n)
    g1, g2 = np.empty(n), np.empty(n)
    f1 = pos(n, 7, n + 7, x.ctypes.data, g1.ctypes.data, d)
    f2 = neg(n, 7, n + 7, x.ctypes.data, g2.ctypes.data, d)
    L.nb200p_destroy(p)
    assert np.float64(f2).view(np.uint64) == np.float64(-f1).view(np.uint64)
    assert np.array_equal(g2.view(np.uint64), (-g1).view(np.uint64))


# ---- the sign-flip kernel builds for sm_90a and does not spill --------------------------------------------------------
def test_negate_kernel_is_built_without_local_memory(built):
    """negate_kernel is in the product library for sm_90a; no stack and no local memory (no spills)"""
    cuobjdump = os.path.join(os.path.dirname(built.NVCC), "cuobjdump")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", built.LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True).stdout
    lines = out.splitlines()
    hits = [i for i, line in enumerate(lines) if "negate_kernel" in line]
    assert hits, out[-2000:]
    usage = " ".join(lines[hits[0]:hits[0] + 3])
    assert "STACK:0" in usage and "LOCAL:0" in usage, usage
    elf = subprocess.run([cuobjdump, "--list-elf", built.LIB], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    assert "sm_90a" in elf
