"""Per-variable terms callbacks on the GPU: the library's reduction against the summation-order model, and whole runs
with C and PyTorch terms callbacks against the __device__ functors whose terms they reproduce, bit for bit.

The model (model_dfunc2) and the adversarial / hashed terms are those of test_device_callbacks_gpu.py: thread t of a CTA
adds lo + t, lo + t + 256, ... from +0.0, then block_sum's tree, the fold of the P group sums of each virtual shard, and
the 8 shard sums in index order.  tests/cpp/terms_callback_probe.cu registers problems.cu's functors either as functors
or as C terms callbacks that call the same functor once per variable.  The PyTorch twins build every term from one IEEE
operation per torch op, in the functors' order, with a, b and the weights precomputed by numpy (tests/synth.py).
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import nlopt_b200 as nl
import synth
from nlopt_b200 import _capi
from test_device_callbacks_gpu import EDGE_SIZES, adversarial_x, hash_terms, model_dfunc2, same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_SRC = os.path.join(ROOT, "tests", "cpp", "terms_callback_probe.cu")
PROBE_SO = os.path.join(ROOT, "tests", "_build", "libterms_callback_probe.so")
SEED = 0x5EED0000
EPS = 1e-3
SIMP, MEAN, LINEAR, SPHERE, ROSEN, QUAD, ROWS4, BLOCK4 = range(8)
MIN, MAX, INEQ, EQ = range(4)


@pytest.fixture(scope="session")
def probe_so(built):
    """tests/cpp/terms_callback_probe.cu -> tests/_build/, linked against the library that nl.opt loads"""
    g = built
    deps = [PROBE_SRC, g.LIB, os.path.join(ROOT, "include", "nlopt_b200_device.cuh"), os.path.join(ROOT, "include", "nlopt_b200.h"),
            os.path.join(ROOT, "nlopt_b200", "csrc", "problem_functors.cuh"), os.path.join(ROOT, "nlopt_b200", "csrc", "synth.cuh")]
    if not os.path.exists(PROBE_SO) or any(os.path.getmtime(d) > os.path.getmtime(PROBE_SO) for d in deps):
        os.makedirs(os.path.dirname(PROBE_SO), exist_ok=True)
        flags = [f for f in g.NVCC_FLAGS if f != "--fmad=false"] + ["--fmad=false"]
        tmp = PROBE_SO + f".{os.getpid()}.tmp"
        r = subprocess.run([g.NVCC, *g.ARCH, *flags, "-shared", PROBE_SRC, "-o", tmp, "-cudart", "shared",
                            "-L" + os.path.dirname(g.LIB), "-lnlopt_b200", "-Xlinker", "-rpath=$ORIGIN/../../nlopt_b200"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        os.replace(tmp, PROBE_SO)
    return PROBE_SO


@pytest.fixture(scope="session")
def probe(probe_so):
    _capi.default_library()
    L = C.CDLL(probe_so, mode=C.RTLD_LOCAL)
    L.probe_terms_register.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p]
    L.probe_terms_reset.argtypes = []
    return L


def test_probe_compiles_for_sm_90a(probe_so):
    import __graft_entry__ as g
    out = subprocess.run([os.path.join(os.path.dirname(g.NVCC), "cuobjdump"), "--list-elf", probe_so],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    assert "sm_90a" in out, out


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


class Reg:
    """one probe registration; keeps its host arrays alive"""

    def __init__(self, probe, kind, role, p=(), w=None, tol=None):
        self.args = (kind, role, _f64(list(p) or [0.0]), _f64(w), _f64(tol))
        self.probe = probe

    def __call__(self, o, form):
        kind, role, p, w, tol = self.args
        ptr = (lambda a: None if a is None else a.ctypes.data)
        o._check(self.probe.probe_terms_register(o._h, kind, role, form, SEED, ptr(p), ptr(w), ptr(tol)))


def bits(v):
    return np.float64(v).tobytes()


def solve(n, regs, form, alg, device, x0, lb, ub, sub=None, maxeval=12):
    """one run: (result, evaluations, dual evaluations, bits of f*, bits of x*)"""
    import torch
    o = nl.opt(alg, n)
    o.set_lower_bounds(lb)
    o.set_upper_bounds(ub)
    o.set_maxeval(maxeval)
    o.set_xtol_rel(1e-10)
    if sub is not None:
        s = nl.opt(sub, n)
        s.set_maxeval(6)
        s.set_xtol_rel(1e-10)
        o.set_local_optimizer(s)
    for r in regs:
        r(o, form)
    if device:
        xt = torch.full((n,), x0, dtype=torch.float64, device="cuda")
        ret = o.optimize_torch(xt)
        ret, x = o.last_optimize_result(), xt.cpu().numpy()
    else:
        x = np.full(n, x0)
        ret = o.optimize_inplace(x)
    return ret, o.get_numevals(), o.get_stats()["dual_evals"], bits(o.last_optimum_value()), x.tobytes()


def rows4(n):
    return np.stack([synth.u01(50 + i, n, 7) - 0.5 for i in range(4)])


def problem(probe, name, n, maximize, eq_ok):
    """(registrations, x0, lb, ub): SIMP + volume, chained Rosenbrock + 4 linear rows, quadratic + sphere / block means"""
    obj = MAX if maximize else MIN
    if name == "simp":
        return [Reg(probe, SIMP, obj, [EPS]), Reg(probe, MEAN, EQ if eq_ok else INEQ, [-0.4], tol=[1e-8]),
                Reg(probe, LINEAR, INEQ, [0.45], w=np.full(n, 1.0 / n), tol=[1e-8])], 0.5, 1e-3, 1.0
    if name == "rosen":
        return [Reg(probe, ROSEN, obj), Reg(probe, ROWS4, INEQ, [0.1, -0.05, 0.2, 0.0], w=rows4(n), tol=[1e-8] * 4)], 0.3, -2.0, 2.0
    return [Reg(probe, QUAD, obj), Reg(probe, SPHERE, EQ if eq_ok else INEQ, [0.2], tol=[1e-8]),
            Reg(probe, BLOCK4, EQ if eq_ok else INEQ, [0.1, 0.2, 0.0, -0.1], tol=[1e-8] * 4)], 0.3, -1.0, 1.0


# ---- C terms callbacks against the functors ------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("alg,sub", [(nl.LD_MMA, None), (nl.LD_CCSAQ, None), (nl.LD_AUGLAG, None), (nl.LD_AUGLAG_EQ, None),
                                     (nl.AUGLAG, nl.LD_CCSAQ)], ids=["MMA", "CCSAQ", "LD_AUGLAG", "LD_AUGLAG_EQ", "AUGLAG-CCSAQ"])
@pytest.mark.parametrize("name", ["simp", "rosen", "quad"])
def test_c_terms_callbacks_match_the_functors(probe, alg, sub, name):
    eq_ok = alg not in (nl.LD_MMA, nl.LD_CCSAQ)
    try:
        for n in (20011, 250000):
            for maximize in (False, True):
                for device in (False, True):
                    regs, x0, lb, ub = problem(probe, name, n, maximize, eq_ok)
                    kw = dict(sub=sub, maxeval=20 if eq_ok else 12)
                    want = solve(n, regs, 0, alg, device, x0, lb, ub, **kw)
                    got = solve(n, regs, 1, alg, device, x0, lb, ub, **kw)
                    assert want[0] > 0 and want[1] > 1, (n, maximize, device, want[:3])
                    assert got == want, (n, maximize, device, got[:4], want[:4])
    finally:
        probe.probe_terms_reset()


# ---- PyTorch twins of the functors ---------------------------------------------------------------------------------
def twins(n):
    """torch terms callbacks with the functors' operation order, and their finishes"""
    import torch
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()       # noqa: E731
    inv_n = 1.0 / n
    qa, qb = cuda(1.0 + synth.u01(0, n, SEED)), cuda(2.0 * synth.u01(1, n, SEED) - 1.0)
    sa = cuda(0.5 + synth.u01(0, n, SEED))
    w = cuda(np.full(n, 1.0 / n))
    W = cuda(rows4(n))
    ome = 1.0 - EPS

    def quad(x, g):
        d = x - qb
        ad = qa * d
        if g.numel():
            g.copy_(ad)
        return ad * d

    def simp(x, g):
        x2 = x * x
        x3 = x2 * x
        d = EPS + ome * x3
        if g.numel():
            g.copy_(-(((sa * (ome * 3.0)) * x2) / (d * d)))
        return sa / d

    def linear(x, g):
        if g.numel():
            g.copy_(w)
        return w * x

    def sphere(x, g):
        if g.numel():
            g.copy_(2.0 * x)
        return x * x

    def rows(x, g):
        if g.numel():
            g.copy_(W)
        return W * x

    return dict(quad=(quad, lambda s: 0.5 * s), simp=(simp, None), linear=(linear, lambda s: s - 0.45),
                sphere=(sphere, lambda s: s * inv_n - 0.2), rows=(rows, lambda t: t - np.array([0.1, -0.05, 0.2, 0.0])))


class TorchReg:
    def __init__(self, how, fn, fin, tol=1e-8, m=None):
        self.how, self.fn, self.fin, self.tol, self.m = how, fn, fin, tol, m

    def __call__(self, o, form):
        getattr(o, self.how)(self.fn, *(() if self.how.startswith("set_") else ((self.tol if self.m is None else [self.tol] * self.m),)),
                             finish=self.fin)


def torch_case(probe, case, n):
    """(functor registrations, torch registrations, algorithm, x0, lb, ub)"""
    t = twins(n)
    if case == "simp":
        return ([Reg(probe, SIMP, MIN, [EPS]), Reg(probe, LINEAR, INEQ, [0.45], w=np.full(n, 1.0 / n), tol=[1e-8])],
                [TorchReg("set_min_objective_torch", *t["simp"]), TorchReg("add_inequality_constraint_torch", *t["linear"])],
                0.5, 1e-3, 1.0)
    if case == "quad":
        return ([Reg(probe, QUAD, MIN), Reg(probe, SPHERE, INEQ, [0.2], tol=[1e-8])],
                [TorchReg("set_min_objective_torch", *t["quad"]), TorchReg("add_inequality_constraint_torch", *t["sphere"])],
                0.3, -1.0, 1.0)
    if case == "quad-eq":
        return ([Reg(probe, QUAD, MIN), Reg(probe, SPHERE, EQ, [0.2], tol=[1e-8])],
                [TorchReg("set_min_objective_torch", *t["quad"]), TorchReg("add_equality_constraint_torch", *t["sphere"])],
                0.3, -1.0, 1.0)
    if case == "quad-max":
        return ([Reg(probe, QUAD, MAX), Reg(probe, LINEAR, INEQ, [0.45], w=np.full(n, 1.0 / n), tol=[1e-8])],
                [TorchReg("set_max_objective_torch", *t["quad"]), TorchReg("add_inequality_constraint_torch", *t["linear"])],
                0.3, -1.0, 1.0)
    return ([Reg(probe, QUAD, MIN), Reg(probe, ROWS4, INEQ, [0.1, -0.05, 0.2, 0.0], w=rows4(n), tol=[1e-8] * 4)],
            [TorchReg("set_min_objective_torch", *t["quad"]), TorchReg("add_inequality_mconstraint_torch", *t["rows"], m=4)],
            0.3, -1.0, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("case,alg", [("simp", nl.LD_MMA), ("simp", nl.LD_CCSAQ), ("quad", nl.LD_MMA), ("quad", nl.LD_CCSAQ),
                                      ("quad-eq", nl.LD_AUGLAG), ("quad-max", nl.LD_MMA), ("rows", nl.LD_MMA)])
@pytest.mark.parametrize("n", [20011, 10**6])
def test_torch_callbacks_match_the_functors(probe, case, alg, n):
    try:
        freg, treg, x0, lb, ub = torch_case(probe, case, n)
        maxeval = 20 if alg == nl.LD_AUGLAG else 12
        for device in (True, False):
            want = solve(n, freg, 0, alg, device, x0, lb, ub, maxeval=maxeval)
            got = solve(n, treg, None, alg, device, x0, lb, ub, maxeval=maxeval)
            assert want[0] > 0 and want[1] > 1, want[:3]
            assert got == want, (device, got[:4], want[:4])
    finally:
        probe.probe_terms_reset()


@pytest.mark.gpu
def test_torch_callbacks_on_a_non_default_stream(probe):
    """optimize_torch while another torch stream is current: the callbacks still run on the library stream, in order"""
    import torch
    n = 250000
    try:
        freg, treg, x0, lb, ub = torch_case(probe, "simp", n)
        want = solve(n, freg, 0, nl.LD_MMA, True, x0, lb, ub)
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            got = solve(n, treg, None, nl.LD_MMA, True, x0, lb, ub)
        assert got == want, (got[:4], want[:4])
    finally:
        probe.probe_terms_reset()


# ---- the reduction against the model -------------------------------------------------------------------------------
def fixed_run(n, obj_terms, rows, maxeval=1):
    """a torch objective and an m-row torch constraint whose terms do not depend on x: the totals handed to finish at
    every point, [(objective total, row totals)]"""
    import torch
    ot = torch.from_numpy(np.ascontiguousarray(obj_terms)).cuda()
    rt = torch.from_numpy(np.ascontiguousarray(rows)).cuda()
    log_f, log_c = [], []

    def f(x, g):
        if g.numel():
            g.fill_(1.0)
        return ot

    def c(x, g):
        if g.numel():
            g.zero_()
        return rt

    o = nl.opt(nl.LD_MMA, n)
    o.set_lower_bounds(-1.0)
    o.set_upper_bounds(1.0)
    o.set_maxeval(maxeval)
    o.set_min_objective_torch(f, finish=lambda s: log_f.append(s) or s)
    o.add_inequality_mconstraint_torch(c, np.full(rows.shape[0], 1e-8), finish=lambda t: log_c.append(t.copy()) or np.full(t.size, -1.0))
    o.optimize_torch(torch.zeros(n, dtype=torch.float64, device="cuda"))
    return log_f, log_c, o


@pytest.mark.gpu
def test_edge_sizes_ascending_then_descending():
    """every geometry edge of test_device_callbacks_gpu.py, up then down (the terms and group-sum buffers are taken per
    run): objective and three rows of adversarial terms equal the model bit for bit"""
    wants = {}
    for n in (*EDGE_SIZES, *reversed(EDGE_SIZES)):
        x = adversarial_x(n)
        rows = np.stack([np.ldexp(x, k) for k in (1, 2, 3)])
        if n not in wants:
            wants[n] = [model_dfunc2(x)] + [model_dfunc2(r) for r in rows]
        log_f, log_c, _ = fixed_run(n, x, rows)
        assert len(log_f) == 1 and len(log_c) == 1
        got = [log_f[0]] + list(log_c[0])
        assert all(same_bits(a, b) for a, b in zip(got, wants[n])), (n, got, wants[n])


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 3, 4, 16, 17, 40])
def test_rows_of_hashed_terms_match_the_model(m):
    n = 100003
    rows = np.stack([hash_terms(n, 10 + i, SEED) for i in range(m)])
    obj = hash_terms(n, 9, SEED)
    log_f, log_c, _ = fixed_run(n, obj, rows)
    assert same_bits(log_f[0], model_dfunc2(obj))
    for i in range(m):
        assert same_bits(log_c[0][i], model_dfunc2(rows[i])), i


@pytest.mark.gpu
def test_special_terms_match_the_model():
    """cancellation (+-2^53 pairs), signed zeros, subnormals and infinities"""
    n = 300000
    sub = np.ldexp(synth.u01(61, n) - 0.5, -1060)                  # subnormals of both signs
    zeros = np.where(synth.u01(62, n) < 0.5, -0.0, 0.0)
    neg_zeros = np.full(n, -0.0)
    inf = np.zeros(n)
    inf[n // 3] = np.inf
    ninf = adversarial_x(n)
    ninf[7] = -np.inf
    both = np.zeros(n)
    both[1], both[n - 1] = np.inf, -np.inf
    rows = np.stack([adversarial_x(n), sub, zeros, neg_zeros, inf, ninf, both])
    log_f, log_c, _ = fixed_run(n, sub, rows)
    assert same_bits(log_f[0], model_dfunc2(sub))
    for i in range(rows.shape[0] - 1):
        assert same_bits(log_c[0][i], model_dfunc2(rows[i])), (i, log_c[0][i], model_dfunc2(rows[i]))
    assert math.isnan(log_c[0][-1])
    assert log_c[0][4] == np.inf and log_c[0][5] == -np.inf


@pytest.mark.gpu
@pytest.mark.parametrize("n", [513, 1250000])
def test_every_point_starts_from_cleared_sums(n):
    """terms that do not depend on x: the same totals at every point of a run"""
    rows = np.stack([hash_terms(n, 20 + i, SEED) for i in range(3)])
    obj = hash_terms(n, 19, SEED)
    log_f, log_c, o = fixed_run(n, obj, rows, maxeval=3)
    assert o.get_numevals() >= 2 and len(log_f) == o.get_numevals() == len(log_c)
    want_f, want_c = model_dfunc2(obj), [model_dfunc2(r) for r in rows]
    for f, c in zip(log_f, log_c):
        assert same_bits(f, want_f) and all(same_bits(a, b) for a, b in zip(c, want_c))


# ---- run behaviour -------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_exception_in_a_torch_callback_stops_the_run(probe):
    import torch
    n = 20011
    calls = []
    t = twins(n)
    quad, quad_fin = t["quad"]

    def failing(x, g):
        calls.append(1)
        if len(calls) == 2:
            raise KeyError("from the callback")
        return quad(x, g)

    o = nl.opt(nl.LD_MMA, n)
    o.set_lower_bounds(-1.0)
    o.set_upper_bounds(1.0)
    o.set_maxeval(10)
    o.set_min_objective_torch(failing, finish=quad_fin)
    x = torch.full((n,), 0.3, dtype=torch.float64, device="cuda")
    with pytest.raises(KeyError, match="from the callback"):
        o.optimize_torch(x)
    assert o.last_optimize_result() == nl.FORCED_STOP
    x = torch.full((n,), 0.3, dtype=torch.float64, device="cuda")
    o.optimize_torch(x)
    assert o.last_optimize_result() > 0 and len(calls) > 3


@pytest.mark.gpu
def test_kernel_launches_count_the_reductions(probe):
    """two launches (terms_group_kernel + fold) per terms callback and evaluation, on top of the functor run's count
    (the functors' own kernels are user launches, not counted by the library)"""
    n = 250000
    try:
        regs, x0, lb, ub = problem(probe, "simp", n, False, False)
        stats = {}
        for form in (0, 1):
            o = nl.opt(nl.LD_MMA, n)
            o.set_lower_bounds(lb)
            o.set_upper_bounds(ub)
            o.set_maxeval(8)
            for r in regs:
                r(o, form)
            o.optimize_inplace(np.full(n, x0))
            stats[form] = (o.get_numevals(), o.get_stats()["kernel_launches"])
        evals = stats[0][0]
        assert stats[1][0] == evals
        assert stats[1][1] - stats[0][1] == 2 * evals * len(regs), stats
    finally:
        probe.probe_terms_reset()


@pytest.mark.gpu
def test_optimize_torch_rejects_other_cuda_tensors():
    import torch
    o = nl.opt(nl.LD_MMA, 8)
    for bad in (torch.zeros(8, dtype=torch.float32, device="cuda"), torch.zeros(9, dtype=torch.float64, device="cuda"),
                torch.zeros(16, dtype=torch.float64, device="cuda")[::2]):
        with pytest.raises(ValueError):
            o.optimize_torch(bad)
