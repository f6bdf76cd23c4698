"""__device__ functors compiled at run time (nlopt_b200.CudaFunctor) on the GPU, bit for bit against the same functors
built by nvcc.

The source twins (tests/jit_twins.py) of problem_functors.cuh's functors run against the functor registrations of
tests/cpp/terms_callback_probe.cu (form 0), the fixture test_terms_callbacks_gpu.py builds: the result code, the
evaluation and dual-evaluation counts and the bits of f* and x* must be equal.  The reduction alone is checked against
the summation-order model of test_device_callbacks_gpu.py at its geometry edges, and a C program built by gcc alone (no
nvcc, no CUDA header) runs SIMP through the C ABI to the bits of the Python run.
"""
import os
import struct
import subprocess

import numpy as np
import pytest

import jit_twins as T
import nlopt_b200 as nl
from test_device_callbacks_gpu import EDGE_SIZES, adversarial_x, model_dfunc2, same_bits
from test_terms_callbacks_gpu import EPS, SEED, problem, probe, probe_so, rows4, solve  # noqa: F401  (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIN, MAX, INEQ, EQ = range(4)
_SCALAR = {MIN: "set_min_objective_cuda", MAX: "set_max_objective_cuda", INEQ: "add_inequality_constraint_cuda",
           EQ: "add_equality_constraint_cuda"}
_VECTOR = {INEQ: "add_inequality_mconstraint_cuda", EQ: "add_equality_mconstraint_cuda"}


class JitReg:
    """one CudaFunctor registration; keeps its device arrays alive (solve() calls it as reg(opt, form))"""

    def __init__(self, name, role, params, finish=None, tol=None, keep=()):
        self.f, self.role, self.params, self.finish, self.tol, self.keep = T.functor(name), role, params, finish, tol, keep

    def __call__(self, o, form=None):
        if self.f.m:
            getattr(o, _VECTOR[self.role])(self.f, self.params, tol=self.tol, finish=self.finish)
        elif self.role in (MIN, MAX):
            getattr(o, _SCALAR[self.role])(self.f, self.params, finish=self.finish)
        else:
            getattr(o, _SCALAR[self.role])(self.f, self.params, tol=self.tol, finish=self.finish)


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def jit_problem(name, n, maximize, eq_ok):
    """problem() of test_terms_callbacks_gpu.py with the source twins: the same functors, parameters and finishes"""
    obj = MAX if maximize else MIN
    inv_n = 1.0 / float(n)
    if name == "simp":
        w = cuda(np.full(n, 1.0 / n))
        return [JitReg("SimpDev", obj, T.simp(SEED, EPS)),
                JitReg("MeanDev", EQ if eq_ok else INEQ, T.two_doubles(inv_n, -0.4), lambda s: s * inv_n + -0.4, 1e-8),
                JitReg("LinearDev", INEQ, T.linear(w.data_ptr(), 0.45), lambda s: s - 0.45, 1e-8, keep=(w,))]
    if name == "rosen":
        b = np.array([0.1, -0.05, 0.2, 0.0])
        W = cuda(rows4(n))
        return [JitReg("RosenbrockDev", obj, b"\0"),
                JitReg("LinearRowsDev<4>", INEQ, T.linear_rows(W.data_ptr(), n, b), lambda t: t - b, [1e-8] * 4, keep=(W,))]
    target = [0.1, 0.2, 0.0, -0.1]
    params, inv_len = T.block_means(n, target)
    inv_len, tg = np.array(inv_len), np.array(target)
    return [JitReg("QuadraticDev", obj, T.quadratic(SEED), lambda s: 0.5 * s),
            JitReg("SphereDev", EQ if eq_ok else INEQ, T.two_doubles(inv_n, 0.2), lambda s: s * inv_n - 0.2, 1e-8),
            JitReg("BlockMeanDev<4>", EQ if eq_ok else INEQ, params, lambda t: t * inv_len - tg, [1e-8] * 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("alg,sub", [(nl.LD_MMA, None), (nl.LD_CCSAQ, None), (nl.LD_AUGLAG, None), (nl.LD_AUGLAG_EQ, None),
                                     (nl.AUGLAG, nl.LD_CCSAQ)], ids=["MMA", "CCSAQ", "LD_AUGLAG", "LD_AUGLAG_EQ", "AUGLAG-CCSAQ"])
@pytest.mark.parametrize("name", ["simp", "rosen", "quad"])
def test_jit_functors_match_the_nvcc_functors(probe, alg, sub, name):
    eq_ok = alg not in (nl.LD_MMA, nl.LD_CCSAQ)
    try:
        for n in (20011, 250000):
            for maximize in (False, True):
                for device in (False, True):
                    regs, x0, lb, ub = problem(probe, name, n, maximize, eq_ok)
                    kw = dict(sub=sub, maxeval=20 if eq_ok else 12)
                    want = solve(n, regs, 0, alg, device, x0, lb, ub, **kw)
                    got = solve(n, jit_problem(name, n, maximize, eq_ok), None, alg, device, x0, lb, ub, **kw)
                    assert want[0] > 0 and want[1] > 1, (n, maximize, device, want[:3])
                    assert got == want, (n, maximize, device, got[:4], want[:4])
    finally:
        probe.probe_terms_reset()


@pytest.mark.gpu
def test_edge_sizes_match_the_model():
    """terms read from a table (they do not depend on x), objective and three rows, at every geometry edge: the totals
    handed to finish equal the summation-order model bit for bit"""
    import torch
    f, v = T.functor("TableDev"), T.functor("TableRowsDev<3>")
    for n in EDGE_SIZES:
        x = adversarial_x(n)
        rows = np.stack([np.ldexp(x, k) for k in (1, 2, 3)])
        xt, rt = cuda(x), cuda(rows)
        log_f, log_c = [], []
        o = nl.opt(nl.LD_MMA, n)
        o.set_lower_bounds(-1.0)
        o.set_upper_bounds(1.0)
        o.set_maxeval(1)
        o.set_min_objective_cuda(f, struct.pack("<Q", xt.data_ptr()), finish=lambda s: log_f.append(s) or s)
        o.add_inequality_mconstraint_cuda(v, struct.pack("<Qq", rt.data_ptr(), n), tol=[1e-8] * 3,
                                          finish=lambda t: log_c.append(t.copy()) or np.full(3, -1.0))
        o.optimize_torch(torch.zeros(n, dtype=torch.float64, device="cuda"))
        assert len(log_f) == 1 and len(log_c) == 1
        want = [model_dfunc2(x)] + [model_dfunc2(r) for r in rows]
        got = [log_f[0]] + list(log_c[0])
        assert all(same_bits(a, b) for a, b in zip(got, want)), (n, got, want)


@pytest.mark.gpu
def test_identity_finish_is_applied_in_c():
    """finish=None registers no Python finish: the total itself is the value, as with finish=lambda s: s"""
    n = 250000
    runs = []
    for fin in (None, lambda s: s):
        o = nl.opt(nl.LD_MMA, n)
        o.set_lower_bounds(1e-3)
        o.set_upper_bounds(1.0)
        o.set_maxeval(6)
        o.set_min_objective_cuda(T.functor("SimpDev"), T.simp(SEED, EPS), finish=fin)
        x = np.full(n, 0.5)
        o.optimize_inplace(x)
        runs.append((o.last_optimize_result(), o.get_numevals(), np.float64(o.last_optimum_value()).tobytes(), x.tobytes()))
    assert runs[0] == runs[1]


C_N, C_MAXEVAL = 20011, 12


@pytest.mark.gpu
def test_c_program_built_by_gcc_alone_matches_python(built):
    """tests/cpp/jit_simp.c: gcc, the C header and -lnlopt_b200, nothing of CUDA; SIMP + volume under LD_MMA"""
    g = built
    src = os.path.join(ROOT, "tests", "cpp", "jit_simp.c")
    exe = os.path.join(ROOT, "tests", "_build", f"jit_simp.{os.getpid()}")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    libdir = os.path.dirname(g.LIB)
    subprocess.check_call(["gcc", "-std=c99", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L" + libdir, "-lnlopt_b200", "-Wl,-rpath," + libdir])
    try:
        out = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    finally:
        os.remove(exe)
    assert out.returncode == 0, out.stdout
    ret, evals, fbits = out.stdout.split()[:3]

    inv_n = 1.0 / C_N
    o = nl.opt(nl.LD_MMA, C_N)
    o.set_lower_bounds(1e-3)
    o.set_upper_bounds(1.0)
    o.set_maxeval(C_MAXEVAL)
    o.set_min_objective_cuda(T.functor("SimpDev"), T.simp(SEED, EPS))
    o.add_inequality_constraint_cuda(T.functor("MeanDev"), T.two_doubles(inv_n, -0.4), tol=1e-8,
                                     finish=lambda s: s * inv_n + -0.4)
    x = np.full(C_N, 0.5)
    o.optimize_inplace(x)
    assert int(ret) == o.last_optimize_result() > 0
    assert int(evals) == o.get_numevals()
    assert fbits == np.float64(o.last_optimum_value()).tobytes()[::-1].hex(), (out.stdout, o.last_optimum_value())
