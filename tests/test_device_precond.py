"""Device preconditioners of LD_CCSAQ (nlopt_b200_dprecond): the entry points' argument checks and the run selection,
on the CPU-backed build of the host logic (hosttest_lib).  The runs themselves are in test_device_precond_gpu.py.

Run selection: host preconditioners only keep the host path with its refusals and messages; a run with both kinds is
refused with its own message before any callback runs; a device preconditioner needs a backend that solves the model
(the GPU one), and is never silently dropped.
"""
import ctypes as C

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi

DPRE = _capi.NLOPT_B200_DPRECOND(lambda *a: None)          # registered by address only; never called here
DPRE_P = C.cast(DPRE, C.c_void_p)
MIXED_MSG = ("preconditioned CCSAQ takes host preconditioners (nlopt_precond) or device preconditioners "
             "(nlopt_b200_dprecond), not both in one run")
PRECOND_MSG = "preconditioned CCSAQ takes host x and host callbacks (nlopt_precond is a host function)"


@pytest.fixture(scope="module")
def L(hosttest_lib):
    d = hosttest_lib.dll
    d.nlopt_b200_set_objective_precond_device.restype = C.c_int
    d.nlopt_b200_set_objective_precond_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    d.nlopt_b200_set_constraint_precond_device.restype = C.c_int
    d.nlopt_b200_set_constraint_precond_device.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_void_p]
    d.nlopt_get_errmsg.restype = C.c_char_p
    return hosttest_lib


def set_obj(L, o, pre=DPRE_P, data=None):
    return L.dll.nlopt_b200_set_objective_precond_device(o._h, pre, data)


def set_con(L, o, index, pre=DPRE_P, data=None):
    return L.dll.nlopt_b200_set_constraint_precond_device(o._h, index, pre, data)


def errmsg(L, o):
    m = L.dll.nlopt_get_errmsg(o._h)
    return m.decode() if m else None


class Counted:
    """f(x) = |x|^2, c(x) = sum x - 1, H = 2 I, counting every call"""

    def __init__(self):
        self.calls = 0

    def f(self, x, g):
        self.calls += 1
        if g.size:
            g[:] = 2 * x
        return float(x @ x)

    def c(self, x, g):
        self.calls += 1
        if g.size:
            g[:] = 1.0
        return float(x.sum()) - 1.0

    def pre(self, x, v, vpre):
        self.calls += 1
        vpre[:] = 2 * v


def make(L, alg=nl.LD_CCSAQ, n=4, host_pre_obj=False, host_pre_con=False, cons=1):
    cb = Counted()
    o = nl.opt(alg, n, library=L)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_maxeval(20)
    if host_pre_obj:
        o.set_precond_min_objective(cb.f, cb.pre)
    else:
        o.set_min_objective(cb.f)
    for _ in range(cons):
        if host_pre_con:
            o.add_precond_inequality_constraint(cb.c, cb.pre, 1e-8)
        else:
            o.add_inequality_constraint(cb.c, 1e-8)
    return o, cb


def run(L, o):
    x = np.full(o._n, 0.1)
    f = C.c_double()
    return L.nlopt_optimize(o._h, x.ctypes.data_as(_capi.c_double_p), C.byref(f))


def test_entry_points_are_declared_and_exported(built):
    for name in ("nlopt_b200_set_objective_precond_device", "nlopt_b200_set_constraint_precond_device"):
        assert name in _capi.EXT_SYMBOLS
    nl.opt(nl.LD_CCSAQ, 3)          # the product library resolves every declared symbol


def test_objective_argument_checks(L):
    o = nl.opt(nl.LD_CCSAQ, 4, library=L)
    assert set_obj(L, o) == nl.INVALID_ARGS and errmsg(L, o) == "no objective registered"
    o, _ = make(L, host_pre_obj=True)
    assert set_obj(L, o) == nl.INVALID_ARGS
    assert errmsg(L, o) == "this function has a host preconditioner (nlopt_precond); a function takes one preconditioner"
    assert set_obj(L, o, None) == nl.SUCCESS            # clearing is always allowed
    o, _ = make(L)
    assert set_obj(L, o) == nl.SUCCESS and errmsg(L, o) is None
    assert L.dll.nlopt_b200_set_objective_precond_device(None, DPRE_P, None) == nl.INVALID_ARGS


def test_constraint_argument_checks(L):
    o, _ = make(L, alg=nl.LD_AUGLAG, cons=0)
    o.add_equality_constraint(lambda x, g: 0.0, 1e-8)
    assert set_con(L, o, 0) == nl.INVALID_ARGS
    assert errmsg(L, o) == "inequality constraint index 0 out of range (0 records; equality constraints take no preconditioner)"
    o, _ = make(L, cons=2)
    assert set_con(L, o, 1) == nl.SUCCESS
    assert set_con(L, o, 2) == nl.INVALID_ARGS and "index 2 out of range (2 records" in errmsg(L, o)
    assert set_con(L, o, 2 ** 32 - 1) == nl.INVALID_ARGS
    o.add_inequality_mconstraint(lambda r, x, g: r.fill(-1.0), [0.0, 0.0])
    assert set_con(L, o, 2) == nl.INVALID_ARGS
    assert errmsg(L, o) == "inequality constraint 2 has 2 rows: a vector constraint takes no preconditioner"
    o, _ = make(L, host_pre_con=True)
    assert set_con(L, o, 0) == nl.INVALID_ARGS and "has a host preconditioner" in errmsg(L, o)
    assert set_con(L, o, 0, None) == nl.SUCCESS


@pytest.mark.parametrize("where", ["objective", "constraint"])
def test_mixed_run_is_refused_before_any_callback(L, where):
    """a host preconditioner on one record and a device one on another: NLOPT_INVALID_ARGS with its message, and no
    callback has run"""
    if where == "objective":
        o, cb = make(L, host_pre_con=True)
        assert set_obj(L, o) == nl.SUCCESS
    else:
        o, cb = make(L, host_pre_obj=True)
        assert set_con(L, o, 0) == nl.SUCCESS
    assert run(L, o) == nl.INVALID_ARGS and errmsg(L, o) == MIXED_MSG
    assert cb.calls == 0


def test_clearing_restores_the_host_path(L):
    o, cb = make(L, host_pre_obj=True)
    assert set_con(L, o, 0) == nl.SUCCESS
    assert run(L, o) == nl.INVALID_ARGS and errmsg(L, o) == MIXED_MSG
    assert set_con(L, o, 0, None) == nl.SUCCESS
    assert run(L, o) > 0 and cb.calls > 0               # run_ccsa_precond, unchanged


def test_ld_mma_ignores_device_preconditioners(L):
    """LD_MMA has no preconditioned branch (mma.c): the mixed case is not refused there, and the run is the plain one"""
    o, cb = make(L, alg=nl.LD_MMA, host_pre_obj=True)
    assert set_con(L, o, 0) == nl.SUCCESS
    assert run(L, o) > 0


def test_device_preconditioner_needs_a_model_solving_backend(L):
    """the CPU test backend has no model solve: the run fails with a message instead of dropping the preconditioner"""
    o, cb = make(L)
    assert set_obj(L, o) == nl.SUCCESS
    assert run(L, o) == nl.FAILURE and errmsg(L, o) == "this backend does not solve preconditioned models"


def test_copy_keeps_and_removal_drops_them(L):
    o, _ = make(L, host_pre_obj=True)
    assert set_con(L, o, 0) == nl.SUCCESS
    c = L.nlopt_copy(o._h)
    assert c
    x = np.full(4, 0.1)
    assert L.nlopt_optimize(c, x.ctypes.data_as(_capi.c_double_p), C.byref(C.c_double())) == nl.INVALID_ARGS
    assert L.dll.nlopt_get_errmsg(c).decode() == MIXED_MSG
    L.nlopt_destroy(c)
    o.remove_inequality_constraints()
    o.add_inequality_constraint(Counted().c, 1e-8)
    assert run(L, o) > 0


def test_host_preconditioner_refusals_are_unchanged(L):
    """a host preconditioner with a device-only form still gets today's message"""
    o, _ = make(L, host_pre_obj=True)
    fin = _capi.NLOPT_B200_DFINISH(lambda t, d: t)
    cb = _capi.NLOPT_B200_DTFUNC(lambda *a: None)
    assert L.dll.nlopt_b200_add_inequality_constraint_terms(o._h, C.cast(cb, C.c_void_p), C.cast(fin, C.c_void_p), None,
                                                            C.c_double(0.0), 0) == nl.SUCCESS
    assert run(L, o) == nl.INVALID_ARGS and errmsg(L, o) == PRECOND_MSG


def test_python_validates_the_index(built):
    o = nl.opt(nl.LD_CCSAQ, 3)
    o.set_min_objective(lambda x, g: 0.0)
    o.add_inequality_constraint(lambda x, g: 0.0)
    for bad in (-1, 2 ** 32, 1.0, "0", True):
        with pytest.raises(ValueError):
            o.set_constraint_precond_torch(bad, None)
        with pytest.raises(ValueError):
            o.set_constraint_precond_device(bad, None)
    o.set_constraint_precond_torch(0, None)             # clearing needs no torch
    o.set_objective_precond_torch(None)
    with pytest.raises(ValueError, match="out of range"):
        o.set_constraint_precond_device(1, DPRE_P)
