"""Vector __device__ constraints (nlopt_b200_add_*_mconstraint_device2): registration, refusals and the kernels' build.

The API layer is checked on the CPU-backed build of the host logic (hosttest_lib): argument checks and algorithm rules
as nlopt_add_*_mconstraint and the scalar _device2 twins, removal, copying, and the refusal of device constraints under
preconditioned CCSAQ (whose nested model solve works on host arrays).  The probe of tests/cpp/device_mcallback_probe.cu
and problems.cu are compiled for sm_90a; their vector kernels are listed in the binaries and do not spill.  The runs
themselves are in test_device_mconstraints_gpu.py.
"""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MPROBE_SRC = os.path.join(ROOT, "tests", "cpp", "device_mcallback_probe.cu")
MPROBE_SO = os.path.join(ROOT, "tests", "_build", "libdevice_mcallback_probe.so")
PROBLEMS_SRC = os.path.join(ROOT, "nlopt_b200", "csrc", "problems.cu")
AUGLAG_IDS = (nl.AUGLAG, nl.AUGLAG_EQ, nl.LN_AUGLAG, nl.LN_AUGLAG_EQ, nl.LD_AUGLAG, nl.LD_AUGLAG_EQ)
DMFUNC2 = C.CFUNCTYPE(None, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p)
DMFINISH = C.CFUNCTYPE(None, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p)
DFUNC2 = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p)
DFINISH = C.CFUNCTYPE(C.c_double, C.c_double, C.c_void_p)
MUNGE = C.CFUNCTYPE(None, C.c_void_p)
PRECOND_MSG = "preconditioned CCSAQ takes host x and host callbacks (nlopt_precond is a host function)"


# ---- the probe library (shared with the GPU tests) -----------------------------------------------------------------
@pytest.fixture(scope="session")
def mprobe_so(built):
    """tests/cpp/device_mcallback_probe.cu -> tests/_build/, linked against the library that nl.opt loads"""
    g = built
    deps = [MPROBE_SRC, g.LIB, os.path.join(ROOT, "include", "nlopt_b200_device.cuh"),
            os.path.join(ROOT, "include", "nlopt_b200.h"), os.path.join(ROOT, "nlopt_b200", "csrc", "synth.cuh")]
    if not os.path.exists(MPROBE_SO) or any(os.path.getmtime(d) > os.path.getmtime(MPROBE_SO) for d in deps):
        os.makedirs(os.path.dirname(MPROBE_SO), exist_ok=True)
        flags = [f for f in g.NVCC_FLAGS if f != "--fmad=false"] + ["--fmad=false"]
        tmp = MPROBE_SO + f".{os.getpid()}.tmp"
        r = subprocess.run([g.NVCC, *g.ARCH, *flags, "-shared", MPROBE_SRC, "-o", tmp, "-cudart", "shared",
                            "-L" + os.path.dirname(g.LIB), "-lnlopt_b200", "-Xlinker", "-rpath=$ORIGIN/../../nlopt_b200"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        os.replace(tmp, MPROBE_SO)
    return MPROBE_SO


@pytest.fixture(scope="session")
def mprobe(mprobe_so):
    _capi.default_library()
    L = C.CDLL(mprobe_so, mode=C.RTLD_LOCAL)
    L.probe_mnew.restype = C.c_void_p
    L.probe_mnew.argtypes = [C.c_int, C.c_int, C.c_int, C.c_ulonglong, C.c_double, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p]
    L.probe_mfree.argtypes = [C.c_int, C.c_int, C.c_void_p]
    L.probe_mregister.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    L.probe_mfunc_ptr.restype = C.c_void_p
    L.probe_mfunc_ptr.argtypes = [C.c_int, C.c_int]
    L.probe_mfinish_ptr.restype = C.c_void_p
    L.probe_mfinish_ptr.argtypes = [C.c_int, C.c_int]
    L.probe_mtotals.argtypes = [C.c_int, C.POINTER(C.c_double), C.c_int]
    L.probe_mreset.argtypes = []
    return L


# ---- registration on the CPU-backed build ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cbs():
    """callables to register: their addresses only; none of them is called"""
    mf = DMFUNC2(lambda *a: None)
    mfin = DMFINISH(lambda *a: None)
    f2 = DFUNC2(lambda *a: None)
    fin = DFINISH(lambda t, d: t)
    return {"mf": C.cast(mf, C.c_void_p), "mfin": C.cast(mfin, C.c_void_p), "f2": C.cast(f2, C.c_void_p),
            "fin": C.cast(fin, C.c_void_p), "_keep": (mf, mfin, f2, fin)}


def _add(L, h, cbs, equality, m=3, tol="zeros", halo=0, fn=True, fin=True, data=None):
    if isinstance(tol, str):
        tol = np.zeros(max(m, 1))
    tp = None if tol is None else np.ascontiguousarray(tol, dtype=np.float64).ctypes.data_as(_capi.c_double_p)
    name = "nlopt_b200_add_equality_mconstraint_device2" if equality else "nlopt_b200_add_inequality_mconstraint_device2"
    return getattr(L.dll, name)(C.c_void_p(h), C.c_uint(m), cbs["mf"] if fn else None, cbs["mfin"] if fin else None,
                                C.c_void_p(data), tp, C.c_int(halo))


def _errmsg(L, h):
    L.dll.nlopt_get_errmsg.restype = C.c_char_p
    m = L.dll.nlopt_get_errmsg(C.c_void_p(h))
    return m.decode() if m else None


def test_algorithm_rules_follow_the_host_mconstraints(hosttest_lib, cbs):
    """inequalities where nlopt_add_inequality_mconstraint takes them, equalities where nlopt_add_equality_mconstraint
    does (the AUGLAG ids): same result code and message as the host form"""
    L = hosttest_lib
    host = _capi.NLOPT_MFUNC(lambda *a: None)
    tol = np.zeros(3)
    for alg in (nl.LD_MMA, nl.LD_CCSAQ, *AUGLAG_IDS):
        for equality in (False, True):
            o1, o2 = L.nlopt_create(alg, 5), L.nlopt_create(alg, 5)
            add_host = L.nlopt_add_equality_mconstraint if equality else L.nlopt_add_inequality_mconstraint
            want = add_host(o1, 3, host, None, tol.ctypes.data_as(_capi.c_double_p))
            got = _add(L, o2, cbs, equality)
            assert got == want, (alg, equality, got, want)
            assert _errmsg(L, o2) == _errmsg(L, o1)
            if equality and alg in (nl.LD_MMA, nl.LD_CCSAQ):
                assert got == nl.INVALID_ARGS and _errmsg(L, o2) == "invalid algorithm for constraints"
            else:
                assert got == nl.SUCCESS
            L.nlopt_destroy(o1)
            L.nlopt_destroy(o2)


def test_argument_checks(hosttest_lib, cbs):
    L = hosttest_lib
    for equality in (False, True):
        o = L.nlopt_create(nl.LD_AUGLAG, 5)
        assert _add(L, o, cbs, equality, fn=False) == nl.INVALID_ARGS
        assert _add(L, o, cbs, equality, fin=False) == nl.INVALID_ARGS
        assert _add(L, o, cbs, equality, halo=2) == nl.INVALID_ARGS
        assert _add(L, o, cbs, equality, halo=-1) == nl.INVALID_ARGS
        assert _add(L, o, cbs, equality, tol=[0.0, -1e-3, 0.0]) == nl.INVALID_ARGS
        assert _errmsg(L, o) == "negative constraint tolerance"
        assert _add(L, o, cbs, equality, tol=None) == nl.SUCCESS          # NULL tol: zeros
        assert _add(L, o, cbs, equality, halo=1, tol=[1e-6, 0.0, 2.0]) == nl.SUCCESS
        assert _add(L, o, cbs, equality, m=16, tol=np.full(16, 1e-8)) == nl.SUCCESS
        L.nlopt_destroy(o)


def test_empty_vector_constraint_registers_nothing_and_munges(hosttest_lib, cbs):
    """m == 0 succeeds (on any algorithm, as nlopt_add_*_mconstraint), registers nothing and hands the data to the
    munge_on_destroy hook"""
    L = hosttest_lib
    seen = []
    munge = MUNGE(lambda d: seen.append(d))
    for alg, equality in ((nl.LD_MMA, False), (nl.LD_MMA, True), (nl.LD_AUGLAG, True)):
        o = L.nlopt_create(alg, 5)
        L.nlopt_set_munge(o, C.cast(munge, C.c_void_p), None)
        seen.clear()
        assert _add(L, o, cbs, equality, m=0, tol=None, fn=False, fin=False, data=0x1234) == nl.SUCCESS
        assert seen == [0x1234]
        L.nlopt_set_munge(o, None, None)
        L.nlopt_destroy(o)


def _precond_opt(L, n=3):
    """LD_CCSAQ on a host quadratic with a preconditioner and a host constraint sum(x) >= 1: a run of the host path"""
    o = nl.opt(nl.LD_CCSAQ, n, library=L)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_maxeval(30)

    def f(x, g):
        if g.size:
            g[:] = 2 * x
        return float(x @ x)

    def pre(x, v, vpre):
        vpre[:] = 2 * v

    o.set_precond_min_objective(f, pre)
    o.add_inequality_constraint(lambda x, g: (g.__setitem__(slice(None), -1.0) if g.size else None, 1.0 - x.sum())[1], 1e-8)
    return o


def _solve_raw(o, x0):
    x = np.array(x0, dtype=np.float64)
    f = C.c_double(0.0)
    return o._lib.nlopt_optimize(o._h, x.ctypes.data_as(_capi.c_double_p), C.byref(f)), x


@pytest.mark.parametrize("kind", ["scalar", "vector"])
def test_preconditioned_ccsaq_refuses_device_constraints(hosttest_lib, cbs, kind):
    """host objective + preconditioner and one device constraint: NLOPT_INVALID_ARGS with a message, before any
    callback runs (the preconditioned solver only evaluates host functions)"""
    L = hosttest_lib
    o = _precond_opt(L)
    if kind == "scalar":
        r = L.dll.nlopt_b200_add_inequality_constraint_device2(C.c_void_p(o._h), cbs["f2"], cbs["fin"], None, C.c_double(0.0), C.c_int(0))
    else:
        r = _add(L, o._h, cbs, False)
    assert r == nl.SUCCESS
    ret, _ = _solve_raw(o, [1.0, 1.0, 1.0])
    assert ret == nl.INVALID_ARGS
    assert o.get_errmsg() == PRECOND_MSG


def test_copy_keeps_and_remove_drops_vector_constraints(hosttest_lib, cbs):
    """nlopt_copy carries a vector device constraint along (the copy is refused like the original);
    nlopt_remove_inequality_constraints drops it, and the run is then the plain host run"""
    L = hosttest_lib
    o = _precond_opt(L)
    assert _add(L, o._h, cbs, False, m=4, tol=None) == nl.SUCCESS
    c = L.nlopt_copy(o._h)
    assert c
    x = np.ones(3)
    assert L.nlopt_optimize(c, x.ctypes.data_as(_capi.c_double_p), C.byref(C.c_double())) == nl.INVALID_ARGS
    assert _errmsg(L, c) == PRECOND_MSG
    L.nlopt_destroy(c)

    o.remove_inequality_constraints()
    o.add_inequality_constraint(lambda x, g: (g.__setitem__(slice(None), -1.0) if g.size else None, 1.0 - x.sum())[1], 1e-8)
    got = _solve_raw(o, [1.0, 1.0, 1.0])
    want = _solve_raw(_precond_opt(L), [1.0, 1.0, 1.0])
    assert got[0] == want[0] and got[0] > 0
    assert np.array_equal(got[1], want[1])


def test_remove_equality_constraints_drops_vector_equalities(hosttest_lib, cbs):
    """a vector device equality would send LD_AUGLAG to the device outer loop, which the CPU test backend cannot run;
    once removed the run is the plain host run"""
    def solve(with_device_eq):
        o = nl.opt(nl.LD_AUGLAG, 2, library=hosttest_lib)
        o.set_lower_bounds([-2.0, -2.0])
        o.set_upper_bounds([2.0, 2.0])
        o.set_min_objective(lambda x, g: (g.__setitem__(slice(None), 2 * x) if g.size else None, float(x @ x))[1])
        o.set_maxeval(30)
        o.add_inequality_constraint(lambda x, g: (g.__setitem__(slice(None), -1.0) if g.size else None, 1.0 - x.sum())[1], 1e-8)
        if with_device_eq:
            assert _add(hosttest_lib, o._h, cbs, True, m=2) == nl.SUCCESS
            o.remove_equality_constraints()
        x = o.optimize([1.0, 1.5])
        return o.last_optimize_result(), o.get_numevals(), o.last_optimum_value(), x

    a, b = solve(True), solve(False)
    assert a[0] > 0 and a[:3] == b[:3] and np.array_equal(a[3], b[3])


# ---- the kernels build for sm_90a and do not spill ------------------------------------------------------------------
def _cuobjdump(built):
    return os.path.join(os.path.dirname(built.NVCC), "cuobjdump")


def test_probe_lists_the_vector_kernels(built, mprobe_so):
    elf = subprocess.run([_cuobjdump(built), "--list-elf", mprobe_so], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True).stdout
    assert "sm_90a" in elf, elf
    out = subprocess.run([_cuobjdump(built), "--list-text", mprobe_so], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True).stdout
    for name in ("map_group_mkernel", "fold_groups_mkernel", "TermMFILi16E", "HashMFILi3E"):
        assert name in out, name


def test_problems_library_lists_the_vector_kernels(built):
    out = subprocess.run([_cuobjdump(built), "--list-text", built.PROBLEMS_LIB], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True).stdout
    for m in (1, 2, 4, 8, 16):
        for f in ("LinearRowsDev", "BlockMeanDev"):
            assert re.search(rf"map_group_mkernel\w*{f}ILi{m}E", out), (f, m)
    assert "fold_groups_mkernel" in out


def _ptxas(built, src, tmp_path):
    """-Xptxas -v of src compiled to a cubin for sm_90a: {kernel name: (registers, spill stores, spill loads)}"""
    out = subprocess.run([built.NVCC, *built.ARCH, *built.NVCC_FLAGS, "-cubin", src, "-o", str(tmp_path / "k.cubin")],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    res, name = {}, None
    for line in out.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            res[name] = [None, int(m.group(1)), int(m.group(2))]
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and name in res:
            res[name][0] = int(m.group(1))
    return res


@pytest.mark.parametrize("src,functors", [(PROBLEMS_SRC, ("LinearRowsDev", "BlockMeanDev")),
                                          (MPROBE_SRC, ("TermMF", "HashMF"))], ids=["problems", "probe"])
def test_sixteen_row_kernels_do_not_spill(built, tmp_path, src, functors):
    k = _ptxas(built, src, tmp_path)
    for f in functors:
        hits = [v for name, v in k.items() if "map_group_mkernel" in name and f"{f}ILi16E" in name]
        assert hits, (f, sorted(k))
        for regs, st, ld in hits:
            assert st == 0 and ld == 0, (f, regs, st, ld)
            assert regs <= 255
