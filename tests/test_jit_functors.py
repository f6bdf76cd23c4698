"""__device__ functors given as source (nlopt_b200.CudaFunctor, nlopt_b200_jit_* in include/nlopt_b200.h), without a
GPU: NVRTC compiles them for sm_90a, reports m, halo and sizeof, keeps the compiler's log, rejects what the library
cannot run, and the registrations check their arguments before anything touches a device."""
import ctypes as C
import os
import subprocess
import sys

import pytest

import jit_twins
import nlopt_b200 as nl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EM_CUDA = 190


@pytest.fixture(scope="module")
def lib(built):
    return nl.Library()


def test_simp_compiles_to_an_sm_90a_cubin(lib):
    f = nl.CudaFunctor(jit_twins.SOURCE, "twin::SimpDev", library=lib)
    img = f.image()
    assert img[:4] == b"\x7fELF" and img[4] == 2                         # 64-bit ELF
    assert int.from_bytes(img[18:20], "little") == EM_CUDA
    import __graft_entry__ as g
    path = os.path.join(ROOT, "tests", "_build", f"jit_simp.{os.getpid()}.cubin")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(img)
    try:
        out = subprocess.run([os.path.join(os.path.dirname(g.NVCC), "cuobjdump"), "-sass", path],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    finally:
        os.remove(path)
    assert "sm_90a" in out, out[:2000]
    assert "map_group_kernel" in out and "SimpDev" in out, out[:2000]


@pytest.mark.parametrize("name,m,halo,nbytes", [
    ("SimpDev", 0, 0, 16), ("QuadraticDev", 0, 0, 8), ("RosenbrockDev", 0, 1, 1), ("LinearDev", 0, 0, 16),
    ("LinearRowsDev<4>", 4, 0, 48), ("LinearRowsDev<16>", 16, 0, 144), ("BlockMeanDev<4>", 4, 0, 104)])
def test_info_reports_m_halo_and_sizeof(lib, name, m, halo, nbytes):
    f = nl.CudaFunctor(jit_twins.SOURCE, "twin::" + name, library=lib)
    assert (f.m, f.halo, f.param_bytes) == (m, halo, nbytes)


def test_params_of_the_twins_have_the_functors_size(lib):
    assert len(jit_twins.simp(1, 1e-3)) == 16
    assert len(jit_twins.linear_rows(0, 5, [0.0] * 4)) == 48
    assert len(jit_twins.block_means(10, [0.0] * 4)[0]) == 104


def test_a_syntax_error_returns_the_compiler_message(lib):
    src = "struct Bad { __device__ double operator()(unsigned long long j) const { return j +; } };"
    with pytest.raises(nl.CompileError) as e:
        nl.CudaFunctor(src, "Bad", library=lib)
    assert "error" in str(e.value) and "functor.cu" in str(e.value), str(e.value)
    assert "expected an expression" in e.value.log, e.value.log
    h = lib.nlopt_b200_jit_create(src.encode(), b"Bad", None, 0)
    try:
        assert b"expected an expression" in lib.nlopt_b200_jit_errmsg(h)
        assert b"expected an expression" in lib.nlopt_b200_jit_log(h)
        assert lib.nlopt_b200_jit_info(h, None, None, None) == -1
        n = C.c_size_t(7)
        assert not lib.nlopt_b200_jit_image(h, C.byref(n)) and n.value == 0
    finally:
        lib.nlopt_b200_jit_destroy(h)


SCALAR_BODY = ("__device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x, "
               "double *g) const { if (g) *g = 1.0; return x[jl]; }")
VECTOR_BODY = ("__device__ void operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x, "
               "double *t, double *g, long long ld) const { for (int i = 0; i < m; ++i) { t[i] = x[jl]; if (g) g[i * ld] = 1.0; } }")


@pytest.mark.parametrize("src,name,what", [
    ("struct V17 { static constexpr int m = 17; " + VECTOR_BODY + " };", "V17", "m = 17"),
    ("struct H2 { static constexpr int halo = 2; " + SCALAR_BODY + " };", "H2", "halo = 2"),
    ("struct S { " + SCALAR_BODY + " };", "Missing", "Missing"),
])
def test_functors_the_library_cannot_run_are_rejected(lib, src, name, what):
    with pytest.raises(nl.CompileError, match=what):
        nl.CudaFunctor(src, name, library=lib)


def test_caller_options_reach_the_compiler(lib):
    src = "struct S { double k; " + SCALAR_BODY.replace("return x[jl];", "return SCALE * x[jl];") + " };"
    with pytest.raises(nl.CompileError, match="SCALE"):
        nl.CudaFunctor(src, "S", library=lib)
    f = nl.CudaFunctor(src, "S", options=["-DSCALE=2.0"], library=lib)
    assert (f.m, f.param_bytes) == (0, 8)


def test_images_are_cached_per_source_name_and_options(lib):
    a = nl.CudaFunctor(jit_twins.SOURCE, "twin::MeanDev", library=lib)
    b = nl.CudaFunctor(jit_twins.SOURCE, "twin::MeanDev", library=lib)
    c = nl.CudaFunctor(jit_twins.SOURCE, "twin::MeanDev", options=["-DUNUSED=1"], library=lib)
    assert a.image() == b.image() == c.image()
    pa, pb = (lib.nlopt_b200_jit_image(x._h, None) for x in (a, b))
    assert pa == pb                                                     # the same compiled image
    assert lib.nlopt_b200_jit_image(c._h, None) != pa


def _raw(lib, fn, o, f, params, *tail):
    return getattr(lib, fn)(o._h, f._h, params, len(params), None, None, *tail)


def test_registration_argument_checks(lib):
    s = nl.CudaFunctor(jit_twins.SOURCE, "twin::SimpDev", library=lib)
    v = nl.CudaFunctor(jit_twins.SOURCE, "twin::LinearRowsDev<4>", library=lib)
    o = nl.opt(nl.LD_MMA, 10, library=lib)
    good = jit_twins.simp(1, 1e-3)
    assert _raw(lib, "nlopt_b200_jit_set_min_objective", o, s, good[:8]) == nl.INVALID_ARGS
    assert "16" in o.get_errmsg() and "8 bytes" in o.get_errmsg()
    assert _raw(lib, "nlopt_b200_jit_add_inequality_mconstraint", o, s, good, None) == nl.INVALID_ARGS
    assert "scalar functor" in o.get_errmsg()
    vp = jit_twins.linear_rows(0, 10, [0.0] * 4)
    assert _raw(lib, "nlopt_b200_jit_add_inequality_constraint", o, v, vp, 0.0) == nl.INVALID_ARGS
    assert "vector functor" in o.get_errmsg()
    assert _raw(lib, "nlopt_b200_jit_add_inequality_constraint", o, s, good, -1e-8) == nl.INVALID_ARGS
    assert "tolerance" in o.get_errmsg()
    assert _raw(lib, "nlopt_b200_jit_add_inequality_constraint", o, s, good, float("nan")) == nl.INVALID_ARGS
    tol = (C.c_double * 4)(0.0, 1e-8, -1.0, 0.0)
    assert _raw(lib, "nlopt_b200_jit_add_inequality_mconstraint", o, v, vp, tol) == nl.INVALID_ARGS
    assert "tolerance" in o.get_errmsg()
    assert lib.nlopt_b200_jit_set_min_objective(o._h, None, good, len(good), None, None) == nl.INVALID_ARGS
    assert "NULL functor handle" in o.get_errmsg()
    # the algorithm checks of the _device2 twins: no equality constraints under LD_MMA
    assert _raw(lib, "nlopt_b200_jit_add_equality_constraint", o, s, good, 0.0) == nl.INVALID_ARGS
    # and the accepted forms
    assert _raw(lib, "nlopt_b200_jit_set_min_objective", o, s, good) == nl.SUCCESS
    assert _raw(lib, "nlopt_b200_jit_set_max_objective", o, s, good) == nl.SUCCESS
    assert _raw(lib, "nlopt_b200_jit_add_inequality_constraint", o, s, good, 1e-8) == nl.SUCCESS
    assert _raw(lib, "nlopt_b200_jit_add_inequality_mconstraint", o, v, vp, None) == nl.SUCCESS
    a = nl.opt(nl.LD_AUGLAG, 10, library=lib)
    assert _raw(lib, "nlopt_b200_jit_add_equality_constraint", a, s, good, 0.0) == nl.SUCCESS
    assert _raw(lib, "nlopt_b200_jit_add_equality_mconstraint", a, v, vp, None) == nl.SUCCESS


def test_a_failed_handle_is_refused_by_every_registration(lib):
    h = lib.nlopt_b200_jit_create(b"struct A {", b"A", None, 0)
    o = nl.opt(nl.LD_MMA, 10, library=lib)
    try:
        assert lib.nlopt_b200_jit_set_min_objective(o._h, h, b"x", 1, None, None) == nl.INVALID_ARGS
        assert "did not compile" in o.get_errmsg()
        assert lib.nlopt_b200_jit_add_inequality_mconstraint(o._h, h, b"x", 1, None, None, None) == nl.INVALID_ARGS
    finally:
        lib.nlopt_b200_jit_destroy(h)


def test_python_methods_raise_with_the_message(lib):
    s = nl.CudaFunctor(jit_twins.SOURCE, "twin::SimpDev", library=lib)
    v = nl.CudaFunctor(jit_twins.SOURCE, "twin::LinearRowsDev<4>", library=lib)
    o = nl.opt(nl.LD_MMA, 10, library=lib)
    with pytest.raises(ValueError, match="sizeof"):
        o.set_min_objective_cuda(s, b"\0" * 8)
    with pytest.raises(ValueError, match="scalar functor"):
        o.add_inequality_mconstraint_cuda(s, jit_twins.simp(1, 1e-3))
    with pytest.raises(ValueError, match="vector functor"):
        o.add_inequality_constraint_cuda(v, jit_twins.linear_rows(0, 10, [0.0] * 4))
    with pytest.raises(TypeError):
        o.set_min_objective_cuda("twin::SimpDev", b"")
    o.set_min_objective_cuda(s, bytearray(jit_twins.simp(1, 1e-3)), finish=lambda t: t)
    o.add_inequality_mconstraint_cuda(v, jit_twins.linear_rows(0, 10, [0.0] * 4), tol=[1e-8] * 4)


def test_import_and_compile_stay_torch_free(built):
    code = ("import sys, nlopt_b200 as nl, jit_twins\n"
            "f = nl.CudaFunctor(jit_twins.SOURCE, 'twin::MeanDev')\n"
            "assert 'torch' not in sys.modules, 'torch imported'\n")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, "-c", code], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout


def test_device_kernels_header_needs_no_system_header():
    """the header NVRTC sees includes nothing but nlopt_b200.h, whose system include is left out under NVRTC"""
    with open(os.path.join(ROOT, "include", "nlopt_b200_device_kernels.cuh")) as f:
        incs = [ln.strip() for ln in f if ln.startswith("#include")]
    assert incs == ['#include "nlopt_b200.h"']
    with open(os.path.join(ROOT, "include", "nlopt_b200.h")) as f:
        text = f.read()
    assert "#ifndef __CUDACC_RTC__\n#include <stddef.h>" in text
