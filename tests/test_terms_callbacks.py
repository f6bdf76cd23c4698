"""Per-variable terms callbacks (nlopt_b200_dtfunc) and their PyTorch front end: registration, refusals, the reduction
kernel's build and the Python checks that need no device.

The API layer is checked on the CPU-backed build of the host logic (hosttest_lib): every terms entry point gives the
result code and message of its _device2 / _mconstraint_device2 twin on the same inputs, and hands the user's data to the
munge hooks like every other form.  The runs themselves are in test_terms_callbacks_gpu.py.
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUGLAG_IDS = (nl.AUGLAG, nl.AUGLAG_EQ, nl.LN_AUGLAG, nl.LN_AUGLAG_EQ, nl.LD_AUGLAG, nl.LD_AUGLAG_EQ)
ALGS = (nl.LD_MMA, nl.LD_CCSAQ, nl.LD_LBFGS, *AUGLAG_IDS)
DFUNC2 = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
DMFUNC2 = C.CFUNCTYPE(None, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p)
MUNGE = C.CFUNCTYPE(C.c_void_p, C.c_void_p)
PRECOND_MSG = "preconditioned CCSAQ takes host x and host callbacks (nlopt_precond is a host function)"
TERMS_SYMBOLS = ("nlopt_b200_set_min_objective_terms", "nlopt_b200_set_max_objective_terms",
                 "nlopt_b200_add_inequality_constraint_terms", "nlopt_b200_add_equality_constraint_terms",
                 "nlopt_b200_add_inequality_mconstraint_terms", "nlopt_b200_add_equality_mconstraint_terms")


@pytest.fixture(scope="module")
def cbs():
    """callables to register: their addresses only; none of them is called"""
    keep = (_capi.NLOPT_B200_DTFUNC(lambda *a: None), DFUNC2(lambda *a: None), DMFUNC2(lambda *a: None),
            _capi.NLOPT_B200_DFINISH(lambda t, d: t), _capi.NLOPT_B200_DMFINISH(lambda *a: None))
    return dict(zip(("terms", "f2", "mf2", "fin", "mfin"), (C.cast(k, C.c_void_p) for k in keep)), _keep=keep)


def _errmsg(L, h):
    L.dll.nlopt_get_errmsg.restype = C.c_char_p
    m = L.dll.nlopt_get_errmsg(C.c_void_p(h))
    return m.decode() if m else None


def _tolp(tol):
    return None if tol is None else np.ascontiguousarray(tol, dtype=np.float64).ctypes.data_as(_capi.c_double_p)


def _register(L, h, cbs, form, what, fn=True, fin=True, tol=0.0, halo=0, m=3, data=None):
    """one registration through the terms entry point (form "terms") or its asynchronous-functor twin (form "device2")"""
    h, d, hl = C.c_void_p(h), C.c_void_p(data), C.c_int(halo)
    fnp = (cbs["terms"] if form == "terms" else cbs["mf2"] if what.endswith("mconstraint") else cbs["f2"]) if fn else None
    finp = (cbs["mfin"] if what.endswith("mconstraint") else cbs["fin"]) if fin else None
    suffix = "terms" if form == "terms" else "device2"
    if what in ("min", "max"):
        return getattr(L.dll, f"nlopt_b200_set_{what}_objective_{suffix}")(h, fnp, finp, d, hl)
    if what in ("inequality", "equality"):
        return getattr(L.dll, f"nlopt_b200_add_{what}_constraint_{suffix}")(h, fnp, finp, d, C.c_double(tol), hl)
    kind = what.split("_")[0]
    if np.isscalar(tol):
        tol = np.full(max(m, 1), tol)
    return getattr(L.dll, f"nlopt_b200_add_{kind}_mconstraint_{suffix}")(h, C.c_uint(m), fnp, finp, d, _tolp(tol), hl)


def test_entry_points_are_declared_and_exported(built):
    for name in TERMS_SYMBOLS:
        assert name in _capi.EXT_SYMBOLS
    nl.opt(nl.LD_MMA, 3)        # the product library resolves every declared symbol


SCALAR_CASES = [dict(), dict(fn=False), dict(fin=False), dict(halo=-1), dict(halo=2), dict(halo=1), dict(tol=-1e-3),
                dict(tol=1e-6, halo=1)]


@pytest.mark.parametrize("what", ["min", "max", "inequality", "equality"])
def test_scalar_forms_match_their_device2_twins(hosttest_lib, cbs, what):
    """argument and algorithm checks: result code and message of the _device2 twin on the same inputs, on every
    algorithm id the equality / inequality rules tell apart"""
    L = hosttest_lib
    for alg in ALGS:
        for kw in SCALAR_CASES:
            if what in ("min", "max") and "tol" in kw:
                continue
            out = {}
            for form in ("terms", "device2"):
                o = L.nlopt_create(alg, 5)
                out[form] = (_register(L, o, cbs, form, what, **kw), _errmsg(L, o))
                L.nlopt_destroy(o)
            assert out["terms"] == out["device2"], (alg, what, kw, out)
    o = L.nlopt_create(nl.LD_MMA, 5)
    assert _register(L, o, cbs, "terms", "equality") == nl.INVALID_ARGS
    assert _errmsg(L, o) == "invalid algorithm for constraints"
    assert _register(L, o, cbs, "terms", "inequality", tol=-1.0) == nl.INVALID_ARGS
    assert _errmsg(L, o) == "negative constraint tolerance"
    L.nlopt_destroy(o)


@pytest.mark.parametrize("what", ["inequality_mconstraint", "equality_mconstraint"])
def test_vector_forms_match_their_mconstraint_device2_twins(hosttest_lib, cbs, what):
    """m == 0 succeeds and registers nothing, a NULL tol means zeros, a negative entry is refused, and m is not capped
    (the terms have no register-file limit): the same codes and messages as the _mconstraint_device2 twin where both
    take the input"""
    L = hosttest_lib
    cases = [dict(m=0, tol=None, fn=False, fin=False), dict(m=3, tol=None), dict(m=3, tol=[0.0, -1e-3, 0.0]),
             dict(m=3, fn=False), dict(m=3, fin=False), dict(m=3, halo=2), dict(m=3, halo=-1), dict(m=3, halo=1, tol=[1e-6, 0, 2]),
             dict(m=1, tol=[0.5])]
    for alg in ALGS:
        for kw in cases:
            kw = dict(kw)
            kw.setdefault("tol", np.zeros(max(kw["m"], 1)))
            out = {}
            for form in ("terms", "device2"):
                o = L.nlopt_create(alg, 5)
                out[form] = (_register(L, o, cbs, form, what, **kw), _errmsg(L, o))
                L.nlopt_destroy(o)
            assert out["terms"] == out["device2"], (alg, what, kw, out)
    o = L.nlopt_create(nl.LD_AUGLAG, 5)
    assert _register(L, o, cbs, "terms", what, m=40, tol=np.full(40, 1e-8)) == nl.SUCCESS
    assert _register(L, o, cbs, "terms", what, m=0, tol=None, fn=False, fin=False) == nl.SUCCESS
    L.nlopt_destroy(o)


def test_munge_sees_the_users_data(hosttest_lib, cbs):
    """munge_on_destroy gets the data of a refused registration (the algorithm check, like every form) and of an empty
    vector registration; nlopt_copy hands every terms callback's data to munge_on_copy and nlopt_destroy to
    munge_on_destroy"""
    L = hosttest_lib
    destroyed, copied = [], []
    on_destroy = MUNGE(lambda d: destroyed.append(d) or None)
    on_copy = MUNGE(lambda d: copied.append(d) or d)
    o = L.nlopt_create(nl.LD_MMA, 5)
    L.nlopt_set_munge(o, C.cast(on_destroy, C.c_void_p), C.cast(on_copy, C.c_void_p))
    assert _register(L, o, cbs, "terms", "equality", data=0x111) == nl.INVALID_ARGS
    assert _register(L, o, cbs, "terms", "equality_mconstraint", data=0x112) == nl.INVALID_ARGS
    assert _register(L, o, cbs, "terms", "inequality_mconstraint", m=0, tol=None, data=0x113) == nl.SUCCESS
    assert destroyed == [0x111, 0x112, 0x113]
    assert _register(L, o, cbs, "terms", "min", data=0x201) == nl.SUCCESS     # munges the previous objective's NULL data
    assert _register(L, o, cbs, "terms", "inequality", data=0x202) == nl.SUCCESS
    assert _register(L, o, cbs, "terms", "inequality_mconstraint", m=4, tol=None, data=0x203) == nl.SUCCESS
    destroyed.clear()
    c = L.nlopt_copy(o)
    assert c
    assert copied == [0x201, 0x202, 0x203]
    L.nlopt_destroy(o)
    assert destroyed == [0x201, 0x202, 0x203]
    destroyed.clear()
    L.nlopt_destroy(c)
    assert destroyed == [0x201, 0x202, 0x203]


def test_munge_data_reaches_terms_callbacks(hosttest_lib, cbs):
    L = hosttest_lib
    seen = []
    M2 = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_void_p)
    mg = M2(lambda p, d: seen.append(p) or p)
    o = L.nlopt_create(nl.LD_AUGLAG, 5)
    assert _register(L, o, cbs, "terms", "max", data=0x301) == nl.SUCCESS
    assert _register(L, o, cbs, "terms", "equality", data=0x302) == nl.SUCCESS
    assert _register(L, o, cbs, "terms", "equality_mconstraint", m=2, tol=None, data=0x303) == nl.SUCCESS
    L.nlopt_munge_data(o, C.cast(mg, C.c_void_p), None)
    assert seen == [0x301, 0x302, 0x303]
    L.nlopt_destroy(o)


def _precond_opt(L, n=3):
    o = nl.opt(nl.LD_CCSAQ, n, library=L)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_maxeval(30)

    def f(x, g):
        if g.size:
            g[:] = 2 * x
        return float(x @ x)

    o.set_precond_min_objective(f, lambda x, v, vpre: vpre.__setitem__(slice(None), 2 * v))
    return o


@pytest.mark.parametrize("what", ["inequality", "inequality_mconstraint"])
def test_preconditioned_ccsaq_refuses_terms_constraints(hosttest_lib, cbs, what):
    L = hosttest_lib
    o = _precond_opt(L)
    assert _register(L, o._h, cbs, "terms", what, tol=None if what.endswith("mconstraint") else 0.0) == nl.SUCCESS
    x = np.ones(3)
    ret = L.nlopt_optimize(o._h, x.ctypes.data_as(_capi.c_double_p), C.byref(C.c_double()))
    assert ret == nl.INVALID_ARGS and o.get_errmsg() == PRECOND_MSG


def test_terms_objective_reaches_the_backend(hosttest_lib, cbs):
    """the API layer takes a terms objective like a _device2 one: the run reaches the backend (the CPU test backend
    evaluates host objectives only and says so)"""
    L = hosttest_lib
    for form in ("terms", "device2"):
        o = L.nlopt_create(nl.LD_MMA, 3)
        assert _register(L, o, cbs, form, "min") == nl.SUCCESS
        x = np.full(3, 0.1)
        ret = L.nlopt_optimize(o, x.ctypes.data_as(_capi.c_double_p), C.byref(C.c_double()))
        assert ret == nl.FAILURE and "host test backend needs a host objective" in _errmsg(L, o), (form, ret)
        L.nlopt_destroy(o)


def test_no_device_gives_the_usual_failure(built):
    """the product library on a machine without a CUDA device: NLOPT_FAILURE and the message of every other form"""
    if nl.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    L = _capi.default_library()
    fin = _capi.NLOPT_B200_DFINISH(lambda t, d: t)
    cb = _capi.NLOPT_B200_DTFUNC(lambda *a: None)
    msgs = []
    for register in (lambda o: L.nlopt_b200_set_min_objective_terms(o, C.cast(cb, C.c_void_p), C.cast(fin, C.c_void_p), None, 0),
                     lambda o: L.nlopt_b200_set_min_objective_device2(o, C.cast(DFUNC2(lambda *a: None), C.c_void_p),
                                                                      C.cast(fin, C.c_void_p), None, 0)):
        o = L.nlopt_create(nl.LD_MMA, 4)
        assert register(o) == nl.SUCCESS
        x = np.full(4, 0.5)
        assert L.nlopt_optimize(o, x.ctypes.data_as(_capi.c_double_p), C.byref(C.c_double())) == nl.FAILURE
        msgs.append(L.nlopt_get_errmsg(o).decode())
        L.nlopt_destroy(o)
    assert msgs[0] == msgs[1] and "no usable CUDA device" in msgs[0], msgs


# ---- Python --------------------------------------------------------------------------------------------------------
def test_import_stays_torch_free(built):
    code = "import sys, nlopt_b200 as nl; o = nl.opt(nl.LD_MMA, 3); print('torch' in sys.modules)"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "False", r.stdout


def test_optimize_torch_rejects_other_tensors(built):
    import torch
    o = nl.opt(nl.LD_MMA, 5)
    for bad in (torch.zeros(5, dtype=torch.float64), torch.zeros(5, dtype=torch.float32), torch.zeros(4, dtype=torch.float64),
                np.zeros(5)):
        with pytest.raises(ValueError):
            o.optimize_torch(bad)


# ---- the reduction kernel builds for sm_90a without spills ---------------------------------------------------------
def test_terms_kernel_does_not_spill(built, tmp_path):
    src = tmp_path / "terms.cu"
    src.write_text('#include "%s"\n' % os.path.join(ROOT, "nlopt_b200", "csrc", "terms_kernels.cuh"))
    out = subprocess.run([built.NVCC, *built.ARCH, *built.NVCC_FLAGS, "-cubin", str(src), "-o", str(tmp_path / "k.cubin")],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    text = out.stdout
    i = text.index("Function properties for _ZN5nb20018terms_group_kernel")
    block = text[i:i + 400]
    assert re.search(r"0 bytes spill stores, 0 bytes spill loads", block), block
    regs = int(re.search(r"Used (\d+) registers", block).group(1))
    assert regs <= 64, block
