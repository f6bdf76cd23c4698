"""The map / reduce kernels of include/nlopt_b200_device.cuh against a model of their summation order, bit for bit.

Every __device__ objective and constraint reaches the optimiser through these kernels:
  * dfunc2 form (set_min_objective / add_inequality_constraint): map_group_kernel reduces one group per CTA,
    fold_groups_kernel folds the P group sums of each of the 8 virtual shards, and the library adds the 8 shard sums
    on the host before finish();
  * sync form (the _sync twins): map_reduce_kernel over a fixed 1056-CTA grid, the last CTA folds the partials.

The probe functors of tests/cpp/device_callback_probe.cu have terms that are exact functions of x (TermF) or of the
index alone (HashF), count every visit of every variable on the device and log every total handed to finish().  The
numpy model below follows the kernels' code: thread t of a CTA adds lo + t, lo + t + 256, ... in turn from +0.0, then
block_sum() adds lane ^ 16, 8, 4, 2, 1 inside each warp and thread 0 adds the 8 warp sums from +0.0.  All adds are
float64 round-to-nearest, as __dadd_rn.  With maxeval = 1 the optimiser returns f(x0), so opt_f is finish(total).
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_SRC = os.path.join(ROOT, "tests", "cpp", "device_callback_probe.cu")
PROBE_SO = os.path.join(ROOT, "tests", "_build", "libdevice_callback_probe.so")

THREADS = 256           # kThreads
SYNC_BLOCKS = 1056      # kBlocks
U = 2.0 ** -53
TERM, HASH = 0, 1
FORMS = ("dfunc2", "sync")
EDGE_SIZES = (1, 2, 255, 256, 257, 511, 512, 513, 4095, 4097, 100003, 299999, 300000, 1250000, 2500001, 10**7)


# ---- geometry (include/nlopt_b200.h: nlopt_b200_shard) ------------------------------------------------------------
class ShardGeo(C.Structure):
    _fields_ = [("n", C.c_ulonglong), ("n_local", C.c_ulonglong), ("j0", C.c_ulonglong), ("nchunks", C.c_ulonglong),
                ("chunk0", C.c_ulonglong), ("groups_total", C.c_uint), ("group0", C.c_uint), ("groups_local", C.c_uint),
                ("groups_per_vshard", C.c_uint), ("vshard0", C.c_uint), ("local_vshards", C.c_uint), ("rank", C.c_int),
                ("world", C.c_int)]


def geometry(n, rank=0, world=1):
    g = ShardGeo()
    _capi.default_library().nlopt_b200_shard_geometry(n, rank, world, C.byref(g))
    return g


# ---- the model -----------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def block_sum(acc):
    """block_sum() for each row of 256 thread values: the result thread 0 holds"""
    v = acc.reshape(-1, THREADS // 32, 32)
    lane = np.arange(32)
    for off in (16, 8, 4, 2, 1):
        v = v + v[:, :, lane ^ off]
    s = np.zeros(v.shape[0])
    for w in range(THREADS // 32):
        s = s + v[:, w, 0]
    return s


def segment_sums(t, lo, hi, stride=THREADS):
    """One CTA per segment [lo, hi) of t (empty when hi <= lo): thread k adds t[lo + k], t[lo + k + 256], ... in turn
    from +0.0, then block_sum().  Ragged segments are padded with +0.0, which leaves every partial sum as it is: an
    accumulator that starts at +0.0 never becomes -0.0 under round-to-nearest.  `stride` != 256 models a broken map."""
    lo = np.asarray(lo, dtype=np.int64)
    hi = np.maximum(np.asarray(hi, dtype=np.int64), lo)
    acc = np.zeros((lo.size, THREADS))
    lane = np.arange(THREADS)
    rows = cdiv(int((hi - lo).max()), stride) if lo.size else 0
    for r in range(rows):
        idx = lo[:, None] + r * stride + lane
        acc = acc + np.where(idx < hi[:, None], t[np.minimum(idx, t.size - 1)], 0.0)
    return block_sum(acc)


def group_bounds(g, plus_one=1):
    """variables [lo, hi) of this rank's groups, relative to its j0 (map_group_kernel's c_lo / c_hi)"""
    k = np.arange(g.group0, g.group0 + g.groups_local, dtype=np.int64)
    lo = (k * g.nchunks // g.groups_total - g.chunk0) * 512
    hi = ((k + plus_one) * g.nchunks // g.groups_total - g.chunk0) * 512
    return lo, np.minimum(hi, g.n_local)


def rank_vsums(t_local, g, stride=THREADS, plus_one=1):
    """map_group_kernel + fold_groups_kernel: the sums of this rank's virtual shards"""
    if g.groups_local == 0:
        return np.zeros(g.local_vshards)
    lo, hi = group_bounds(g, plus_one)
    part = segment_sums(t_local, lo, hi, stride)
    P = g.groups_per_vshard
    v = np.arange(g.local_vshards, dtype=np.int64)
    return segment_sums(part, v * P, (v + 1) * P)


def add_in_order(a):
    tot = a[0]
    for v in a[1:]:
        tot = tot + v
    return float(tot)


def model_dfunc2(t, world=1, **mutation):
    """The total the library hands to finish(): every rank writes its virtual-shard slots of the zeroed [8] block (the
    all-reduce over ranks is exact, each slot is non-zero on one rank only), then tot = vs[0]; tot += vs[1..7]."""
    vs = np.zeros(8)
    for rank in range(world):
        g = geometry(t.size, rank, world)
        vs[g.vshard0:g.vshard0 + g.local_vshards] = rank_vsums(t[g.j0:g.j0 + g.n_local], g, **mutation)
    return add_in_order(vs)


def model_sync(t):
    """map_reduce_kernel: 1056 contiguous slices of ceil(n / 1056) variables, then the last CTA folds the partials"""
    n = t.size
    per = cdiv(n, SYNC_BLOCKS)
    b = np.arange(SYNC_BLOCKS, dtype=np.int64)
    part = segment_sums(t, b * per, np.minimum((b + 1) * per, n))
    return float(segment_sums(part, [0], [SYNC_BLOCKS])[0])


def model(form, t):
    return model_dfunc2(t) if form == "dfunc2" else model_sync(t)


def depth(form, n):
    """longest chain of adds from a term to the total: per CTA, a thread's own adds + 5 shuffle steps + 8 warp sums"""
    if form == "dfunc2":
        g = geometry(n)
        lo, hi = group_bounds(g)
        return cdiv(int((hi - lo).max()), THREADS) + 13 + cdiv(g.groups_per_vshard, THREADS) + 13 + 7
    return cdiv(cdiv(n, SYNC_BLOCKS), THREADS) + 13 + cdiv(SYNC_BLOCKS, THREADS) + 13


def check_fsum_bound(form, t, got):
    """the model is a plain float64 summation: within depth * 2^-53 * sum|t| of the correctly rounded sum (+1 for
    fsum's own rounding)"""
    exact = math.fsum(t.tolist())
    scale = math.fsum(np.abs(t).tolist())
    assert abs(got - exact) <= (depth(form, t.size) + 1) * U * scale, (got, exact, scale)


# ---- terms ---------------------------------------------------------------------------------------------------------
def smooth_x(n):
    return 2.0 * synth.u01(31, n) - 1.0


def big_terms(n):
    """+2^53 / -2^53 pairs in neighbouring threads, different groups and different virtual shards, and one
    +-2^(30 + 3 v) in each eighth v of the variables, so that the 8 virtual-shard sums differ widely in size"""
    pairs = [(0, 1), (3, 4100), (300, n // 2 + 7), (n // 8 + 1, n - 2), (n // 3, 7 * n // 8 + 513)]
    cand = [(a, 2.0 ** 53) for a, _ in pairs] + [(b, -(2.0 ** 53)) for _, b in pairs]
    cand += [((2 * v + 1) * n // 16, (-1.0) ** v * 2.0 ** (30 + 3 * v)) for v in range(8)]
    used, out = set(), []
    for j, val in cand:
        if j < n and j not in used:
            used.add(j)
            out.append((j, val))
    return out


def adversarial_x(n):
    """x_j = +-2^e_j with e_j spread over [-40, 40], plus the big terms: nearly every change of summation order changes
    the rounded total"""
    e = np.floor(synth.u01(41, n) * 81.0).astype(np.int64) - 40
    x = np.ldexp(np.where(synth.u01(42, n) < 0.5, -1.0, 1.0), e)
    for j, val in big_terms(n):
        x[j] = val
    return x


def hash_terms(n, k_id, seed):
    """HashF's terms, in the device's operation order"""
    u = synth.u01(k_id, n, seed)
    e = (synth.u01(k_id + 1000, n, seed) * 81.0).astype(np.int64) - 40
    return np.ldexp(2.0 * u - 1.0, e)


# ---- the probe library ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="session")
def probe_so(built):
    """tests/cpp/device_callback_probe.cu -> tests/_build/, linked against the library that nl.opt loads"""
    g = built
    deps = [PROBE_SRC, g.LIB, os.path.join(ROOT, "include", "nlopt_b200_device.cuh"),
            os.path.join(ROOT, "include", "nlopt_b200.h"), os.path.join(ROOT, "nlopt_b200", "csrc", "synth.cuh")]
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
    _capi.default_library()                # libnlopt_b200.so first: the probe resolves against the same copy
    L = C.CDLL(probe_so, mode=C.RTLD_LOCAL)
    L.probe_new.restype = C.c_void_p
    L.probe_new.argtypes = [C.c_int, C.c_int, C.c_ulonglong, C.c_double, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p]
    L.probe_free.argtypes = [C.c_int, C.c_void_p]
    L.probe_register.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double]
    L.probe_totals.argtypes = [C.c_int, C.POINTER(C.c_double), C.c_int]
    L.probe_reset.argtypes = []
    return L


class Functor:
    """one probe functor and its witness counters (torch tensors on the device); keep it alive while its opt runs"""

    def __init__(self, L, kind, k_id, n, seed=0, offset=0.0):
        import torch
        self.L, self.kind, self.k_id, self.n = L, kind, k_id, n
        self.visits = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
        self.counters = torch.zeros(2, dtype=torch.int32, device="cuda")       # errors, calls with a gradient
        cp = self.counters.data_ptr()
        self.h = L.probe_new(kind, k_id, seed, offset, n, self.visits.data_ptr(), cp, cp + 4)
        assert self.h

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            self.L.probe_free(self.kind, h)

    def register(self, o, form, constraint, tol=0.0):
        o._check(self.L.probe_register(o._h, self.kind, self.h, int(form == "sync"), int(constraint), tol))

    def totals(self):
        cnt = self.L.probe_totals(self.k_id, None, 0)
        buf = (C.c_double * max(cnt, 1))()
        self.L.probe_totals(self.k_id, buf, cnt)
        return [buf[i] for i in range(cnt)]

    def check_witness(self, evals):
        """every variable visited once per evaluation, with the right indices, and a gradient pointer on every call"""
        visits = self.visits[:self.n].cpu().numpy()
        errors, grad_calls = self.counters.cpu().tolist()
        bad = np.flatnonzero(visits != evals)
        assert bad.size == 0, f"k_id {self.k_id}: {bad.size} variables not visited {evals}x, first {bad[:5]} -> {visits[bad[:5]]}"
        assert errors == 0, f"k_id {self.k_id}: {errors} calls with a wrong j, n, n_local or jl"
        assert grad_calls == self.n * evals, (self.k_id, grad_calls, self.n * evals)


def run(n, x, funcs, form, alg=nl.LD_MMA, maxeval=1, repeats=1):
    """funcs[0] is the objective, the rest are constraints; returns opt_f of each run"""
    import torch
    o = nl.opt(alg, n)
    o.set_maxeval(maxeval)
    funcs[0].register(o, form, constraint=False)
    for f in funcs[1:]:
        f.register(o, form, constraint=True, tol=1e-8)
    out = []
    for _ in range(repeats):
        xd = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()
        o.optimize_device(xd.data_ptr())
        torch.cuda.synchronize()
        out.append(o.last_optimum_value())
    return out


def same_bits(a, b):
    return np.float64(a).tobytes() == np.float64(b).tobytes()


# ---- CPU: the probe builds, the model does not depend on the number of ranks ---------------------------------------
def test_probe_compiles_for_sm_90a(probe_so):
    """the first instantiation of the _sync templates (map_reduce_kernel) next to the dfunc2 ones"""
    import __graft_entry__ as g
    out = subprocess.run([os.path.join(os.path.dirname(g.NVCC), "cuobjdump"), "--list-elf", probe_so],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout
    assert "sm_90a" in out, out


@pytest.mark.parametrize("n", EDGE_SIZES)
def test_dfunc2_model_is_the_same_for_every_world_size(built, n):
    """nlopt_b200_shard_geometry per rank for 1, 2, 4 and 8 ranks: the same bits (the library's promise that the value
    does not depend on the number of ranks; the GPU tests tie the one-rank model to the kernels)"""
    for t in (adversarial_x(n), smooth_x(n)):
        one = model_dfunc2(t, 1)
        for world in (2, 4, 8):
            assert same_bits(model_dfunc2(t, world), one), (n, world)


@pytest.mark.parametrize("n", (4097, 100003, 2500001, 10**7))
def test_adversarial_terms_tell_summation_orders_apart(built, n):
    """the terms of the bit-for-bit tests separate the kernels' order from nearby wrong ones, so a kernel that adds in
    another order cannot match the model by luck"""
    t = adversarial_x(n)
    want = model_dfunc2(t)
    g = geometry(n)
    others = {
        "sync order": model_sync(t),
        "sequential": add_in_order(t),
        "numpy pairwise": float(np.sum(t)),
        "fsum": math.fsum(t.tolist()),
        "vshards reversed": add_in_order(rank_vsums(t, g)[::-1]),
        "thread stride 128": model_dfunc2(t, stride=THREADS // 2),
        "group bounds without +1": model_dfunc2(t, plus_one=0),
    }
    for name, v in others.items():
        assert not same_bits(v, want), name


# ---- GPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("alg,n", [pytest.param(nl.LD_MMA, 4097, id="MMA-4097"), pytest.param(nl.LD_MMA, 1250000, id="MMA-1250000"),
                                   pytest.param(nl.LD_MMA, 10**7, id="MMA-1e7"), pytest.param(nl.LD_CCSAQ, 10**7, id="CCSAQ-1e7")])
def test_objective_and_three_constraints_match_the_model(probe, form, alg, n):
    """four TermF with k_id 0..3 (terms x_j 2^k_id): each slot's total equals the model bit for bit, twice in a row (the
    sync form's ticket is reset by the last CTA), and opt_f is finish(model)"""
    probe.probe_reset()
    x = smooth_x(n)
    funcs = [Functor(probe, TERM, k, n, offset=0.25 * (k + 1)) for k in range(4)]
    got = run(n, x, funcs, form, alg, repeats=2)
    for f in funcs:
        t = np.ldexp(x, f.k_id)
        want = model(form, t)
        assert [same_bits(v, want) for v in f.totals()] == [True, True], (f.k_id, f.totals(), want)
        f.check_witness(2)
        if f.k_id == 0:
            check_fsum_bound(form, t, want)
            assert all(same_bits(v, want + 0.25) for v in got), (got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("n", (4097, 100003, 2500001, 10**7))
def test_order_sensitive_terms_match_the_model(probe, form, n):
    """+-2^e terms with +-2^53 pairs in different threads, groups and virtual shards; a NaN at j = n - 1 and a +inf at
    j = 0 reach the value"""
    x = adversarial_x(n)
    x_nan, x_inf = x.copy(), x.copy()
    x_nan[-1] = np.nan
    x_inf[0] = np.inf
    for k_id, xs in ((0, x), (1, x_nan), (2, x_inf)):
        probe.probe_reset()
        f = Functor(probe, TERM, k_id, n)
        got = run(n, xs, [f], form)[0]
        logged = f.totals()
        assert len(logged) == 1, logged
        if xs is x:
            want = model(form, np.ldexp(x, k_id))
            assert same_bits(got, want) and same_bits(logged[0], want), (got, logged, want)
        elif xs is x_nan:
            assert math.isnan(got) and math.isnan(logged[0]), (got, logged)
        else:
            assert got == math.inf and logged[0] == math.inf, (got, logged)
        f.check_witness(1)


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
def test_geometry_edge_sizes_ascending_then_descending(probe, form):
    """one process, sizes up then down: the dfunc2 form's group-sum buffer grows while the run goes on and is reused at
    smaller sizes.  The sizes cover fewer chunks than groups (empty groups), the 440-group band of the group rule and
    P > 256 group sums per virtual shard.  n = 1 is accepted and runs like any other size."""
    assert geometry(10**7).groups_per_vshard > THREADS and geometry(300000).groups_total == 440
    assert geometry(4097).groups_total > geometry(4097).nchunks
    wants = {}
    for n in (*EDGE_SIZES, *reversed(EDGE_SIZES)):
        probe.probe_reset()
        x = adversarial_x(n)
        obj, con = Functor(probe, TERM, 4, n), Functor(probe, TERM, 5, n, offset=-1.0)
        got = run(n, x, [obj, con], form)[0]
        if n not in wants:
            wants[n] = (model(form, np.ldexp(x, 4)), model(form, np.ldexp(x, 5)))
        w_obj, w_con = wants[n]
        assert len(obj.totals()) == 1 and same_bits(obj.totals()[0], w_obj), (n, obj.totals(), w_obj)
        assert len(con.totals()) == 1 and same_bits(con.totals()[0], w_con), (n, con.totals(), w_con)
        assert same_bits(got, w_obj), (n, got, w_obj)
        obj.check_witness(1)
        con.check_witness(1)


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("n", (513, 1250000))
def test_every_point_starts_from_cleared_sums(probe, form, n):
    """HashF does not depend on x: the objective and two constraints give the same total at every point of a run"""
    probe.probe_reset()
    seed = 0x5EED1234
    funcs = [Functor(probe, HASH, k, n, seed=seed, offset=1.0) for k in (10, 11, 12)]
    x = smooth_x(n) * 0.5
    o = nl.opt(nl.LD_MMA, n)
    o.set_lower_bounds(-1.0)
    o.set_upper_bounds(1.0)
    o.set_maxeval(3)
    funcs[0].register(o, form, constraint=False)
    for f in funcs[1:]:
        f.register(o, form, constraint=True, tol=1e-8)
    import torch
    xd = torch.from_numpy(x).cuda()
    o.optimize_device(xd.data_ptr())
    evals = o.get_numevals()
    assert evals >= 2, evals
    for f in funcs:
        want = model(form, hash_terms(n, f.k_id, seed))
        assert len(f.totals()) == evals, (f.k_id, f.totals(), evals)
        assert all(same_bits(v, want) for v in f.totals()), (f.k_id, f.totals(), want)
        f.check_witness(evals)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["rosenbrock", "quadratic", "simp"])
def test_bench_functors_at_bench_sizes(built, case):
    """problems.cu's own objectives at the benchmark sizes, m = 0: opt_f is finish(model) of numpy terms written in the
    device's operation order"""
    import torch
    from nlopt_b200.problems import Problem, rosen_x0
    seed = 0x5EED0000
    p = Problem()
    if case == "rosenbrock":
        n = 10**7
        x = rosen_x0(n)
        d = x[1:] - x[:-1] * x[:-1]
        e = 1.0 - x[:-1]
        t = np.append((100.0 * d) * d + e * e, 0.0)
        finish = 1.0
    elif case == "quadratic":
        n = 10**6
        x = np.full(n, -0.5)
        a = 1.0 + synth.u01(0, n, seed)
        b = 2.0 * synth.u01(1, n, seed) - 1.0
        d = x - b
        t = (a * d) * d
        finish = 0.5
    else:
        n = 5 * 10**7
        eps = 1e-3
        x = np.full(n, 0.4)
        a = 0.5 + synth.u01(0, n, seed)
        x2 = x * x
        x3 = x2 * x
        t = a / (eps + (1.0 - eps) * x3)
        finish = 1.0
    want = model_dfunc2(t) * finish
    del t
    o = nl.opt(nl.LD_MMA, n)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_maxeval(1)
    if case == "rosenbrock":
        p.rosenbrock_device(o, 0)
    elif case == "quadratic":
        o._check(p.L.nb200p_set_quadratic_device(p.h, o._h, seed))
    else:
        o._check(p.L.nb200p_set_simp_device(p.h, o._h, seed, eps))
    xd = torch.from_numpy(x).cuda()
    o.optimize_device(xd.data_ptr())
    assert same_bits(o.last_optimum_value(), want), (o.last_optimum_value(), want)
