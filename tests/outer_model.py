"""Plain float64 references of the kernels that run between dual solves (nlopt_b200/csrc/ccsa_kernels.cuh):
sigma_init_kernel, end_outer_kernel (stop sums, xtol_abs count, sigma update, rotation), penalty_axpy_kernel and
negate_kernel; the operand classes the tests mix into their arrays; and the assertions applied to what a kernel
returned.  numpy and math.fsum only: one IEEE operation per numpy operation, in the order of the kernel code.

tests/test_outer_kernels.py pins these models to the oracle port and shows that the assertions reject wrong models;
tests/test_outer_kernels_gpu.py applies the same assertions to the kernels' output.
"""
import ctypes as C
import math

import numpy as np

import synth

U = 2.0 ** -53
MMA, CCSAQ = 0, 1
KAPPA = {MMA: 0.01, CCSAQ: 1e-8}        # mma.c:439, ccsa_quadratic.c:587
CHUNK = 512                             # variables per chunk (geometry.hpp)
THREADS = 256                           # kBlock


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def from_bits(b):
    return np.asarray(b, dtype=np.uint64).view(np.float64)


QNAN = from_bits([0x7FF8DEAD0000BEEF])[0]       # quiet NaN with a payload
SNAN = from_bits([0x7FF4000000001234])[0]       # signalling NaN with a payload
GUARD = from_bits([0x7FF8600D600D600D])[0]      # what the probe buffers hold around a target row


def isinf(v):
    return np.isinf(v)          # dev_isinf: |v| >= HUGE_VAL * 0.99 is |v| == inf in float64


# ---- sigma -----------------------------------------------------------------------------------------------------------
def sigma_init(lb, ub, init, sigma_min):
    """sigma_init_kernel (mma.c:202-210)"""
    with np.errstate(all="ignore"):
        s = np.where(isinf(ub) | isinf(lb), 1.0, 0.5 * (ub - lb))
        if init is not None:
            s = np.where(init > 0, init, s)
        return np.where(s > sigma_min, s, sigma_min)


def sigma_update(variant, xcur, xprev, xprevprev, lb, ub, sigma, sigma_min, kappa=None, one_sided_clamp=False,
                 floor=True):
    """the sigma branch of end_outer_kernel (mma.c:431-442, ccsa_quadratic.c:577-590).  The keyword arguments build
    wrong models for the mutation checks: another kappa, the cap / floor applied unless BOTH bounds are infinite, no
    sigma_min floor."""
    kappa = KAPPA[variant] if kappa is None else kappa
    with np.errstate(all="ignore"):
        osc = (xcur - xprev) * (xprev - xprevprev)
        gam = np.where(osc < 0, 0.7, np.where(osc > 0, 1.2, 1.0))
        s = sigma * gam
        rng = ub - lb
        top, bot = 10.0 * rng, kappa * rng
        clamped = np.where(s < top, s, top)
        clamped = np.where(clamped > bot, clamped, bot)
        free = (isinf(ub) & isinf(lb)) if one_sided_clamp else (isinf(ub) | isinf(lb))
        s = np.where(free, s, clamped)
        return np.where(s > sigma_min, s, sigma_min) if floor else s


# ---- stop sums (stop.c:98-108) ----------------------------------------------------------------------------------------
def stop_terms(xcur, xprev, w=None, xtol_abs=None, strict=False):
    """the correctly rounded per-variable terms w|xc - xp| and w|xc| (without w: |xc - xp| and |xc|) and the number
    of variables with |xc - xp| >= xtol_abs (None without xtol_abs).  strict: `>`, a wrong model."""
    with np.errstate(all="ignore"):
        d = np.abs(xcur - xprev)
        ax = np.abs(xcur)
        td, tx = (d, ax) if w is None else (w * d, w * ax)
        count = None
        if xtol_abs is not None:
            count = int(np.count_nonzero(d > xtol_abs if strict else d >= xtol_abs))
    return td, tx, count


def stop_decision(dn, xn, count, xtol_rel):
    """nlopt_stop_x from the three numbers the kernel returns (ccsa_driver.cpp / stop_x_host): the relative test on
    the sums, else every |dx| below its xtol_abs; a NaN |dx| is never >= anything, so it counts as below"""
    if dn < xtol_rel * xn:
        return True
    return count is not None and count == 0


def exact_sum(t):
    return math.fsum(t.tolist())


# ---- geometry and the depth of the summation tree -----------------------------------------------------------------------
class ShardGeo(C.Structure):            # include/nlopt_b200.h: nlopt_b200_shard
    _fields_ = [("n", C.c_ulonglong), ("n_local", C.c_ulonglong), ("j0", C.c_ulonglong), ("nchunks", C.c_ulonglong),
                ("chunk0", C.c_ulonglong), ("groups_total", C.c_uint), ("group0", C.c_uint), ("groups_local", C.c_uint),
                ("groups_per_vshard", C.c_uint), ("vshard0", C.c_uint), ("local_vshards", C.c_uint), ("rank", C.c_int),
                ("world", C.c_int)]


def geometry(n, rank=0, world=1):
    from nlopt_b200 import _capi
    g = ShardGeo()
    _capi.default_library().nlopt_b200_shard_geometry(n, rank, world, C.byref(g))
    return g


def group_cuts(g):
    """first chunk of every group, and nchunks: group s covers chunks [cuts[s], cuts[s + 1])"""
    s = np.arange(g.groups_total + 1, dtype=np.int64)
    return s * int(g.nchunks) // int(g.groups_total)


def depth(g):
    """The longest chain of adds from a term to a total of end_outer_kernel.  A CTA owns one group: a thread adds its
    two variables of each chunk in turn (from +0.0), block_reduce_to adds 5 shuffle partners and then 7 warp sums;
    the last CTA of a virtual shard adds its share of the P group records (ceil(P / 256) each) and reduces again; the
    8 virtual-shard sums are added in index order (7 adds, in the kernel on one rank, in publish_kernel on several)."""
    chunks = int(np.diff(group_cuts(g)).max())
    return 2 * chunks + 12 + -(-int(g.groups_per_vshard) // THREADS) + 12 + 7


# ---- penalty gradient and negation ------------------------------------------------------------------------------------
def penalty_axpy(g, rows, coefs, row_idx, reverse=False):
    """penalty_axpy_kernel: v = g; for k: v = v + (c_k * rows[row_k]), a rounded multiply then a rounded add
    (auglag.c:47-48, :59-60).  reverse: the rows in the opposite order, a wrong model."""
    order = list(zip(coefs, row_idx))
    v = np.array(g, dtype=np.float64)
    with np.errstate(all="ignore"):
        for c, r in (reversed(order) if reverse else order):
            v = v + np.float64(c) * rows[r]
    return v


def penalty_axpy_fused(g, rows, coefs, row_idx):
    """a wrong model: v = fma(c_k, row_k, v), the exact product and sum rounded once (finite operands only)"""
    from fractions import Fraction
    v = [Fraction(float(x)) for x in g]
    for c, r in zip(coefs, row_idx):
        v = [Fraction(float(Fraction(float(c)) * Fraction(float(x)) + a)) for x, a in zip(rows[r], v)]
    return np.array([float(a) for a in v])


def negate_bits(g):
    return from_bits(bits(g) ^ np.uint64(1 << 63))


# ---- operand classes ---------------------------------------------------------------------------------------------------
OSC = ("osc<0", "osc>0", "osc==0:xc==xp", "osc==0:xp==xpp", "osc underflows to +0", "osc underflows to -0", "NaN in xc")
BND = ("bounds finite", "bounds both infinite", "only lb=-inf", "only ub=+inf", "lb==ub", "bounds +-1.5e308")
SIG = ("sigma ordinary", "sigma on the cap 10*range", "sigma on the floor kappa*range", "sigma below sigma_min")
NCLASS = len(OSC) * len(BND) * len(SIG)
SIGMA_MINS = (0.0, 0.25, 1e3)           # none; above "sigma below sigma_min"; above 10 * range of the finite bounds
INITS = ("absent", "positive", "zero", "negative", "NaN", "mixed")


def class_ids(n, shift=None):
    """class number of every variable: hashed (shift None), or j + shift so that small n enumerate every class"""
    if shift is None:
        c = np.minimum((synth.u01(50, n) * NCLASS).astype(np.int64), NCLASS - 1)
    else:
        c = (np.arange(n, dtype=np.int64) + shift) % NCLASS
    return c % len(OSC), (c // len(OSC)) % len(BND), c // (len(OSC) * len(BND))


def class_name(ids, j):
    return f"{OSC[ids[0][j]]} | {BND[ids[1][j]]} | {SIG[ids[2][j]]}"


def operands(n, variant, shift=None):
    """xcur, xprev, xprevprev, lb, ub, sigma with every class of OSC x BND x SIG, and the class numbers"""
    ids = class_ids(n, shift)
    osc, bnd, sig = ids
    a = 0.01 + 0.1 * synth.u01(52, n)
    b = 0.01 + 0.1 * synth.u01(53, n)
    xp = 2.0 * synth.u01(51, n) - 1.0
    tiny = (osc == 4) | (osc == 5)
    xp[tiny] = 0.0
    xc = xp + a
    xc[osc == 2] = xp[osc == 2]
    xc[tiny] = 1e-200
    xc[osc == 6] = QNAN
    xpp = np.where(osc == 1, xp - b, xp + b)
    xpp[osc == 3] = xp[osc == 3]
    xpp[osc == 4] = -1e-200
    xpp[osc == 5] = 1e-200
    lb = -2.0 - synth.u01(54, n)
    ub = 2.0 + synth.u01(55, n)
    lb[(bnd == 1) | (bnd == 2)] = -np.inf
    ub[(bnd == 1) | (bnd == 3)] = np.inf
    lb[bnd == 4] = ub[bnd == 4] = 0.5
    lb[bnd == 5], ub[bnd == 5] = -1.5e308, 1.5e308
    with np.errstate(all="ignore"):
        rng = np.where(isinf(ub) | isinf(lb) | (bnd == 5), 4.0, ub - lb)
    sigma = (0.05 + 0.95 * synth.u01(56, n)) * 2.0
    sigma = np.where(sig == 1, 10.0 * rng, sigma)
    sigma = np.where(sig == 2, KAPPA[variant] * rng, sigma)
    sigma = np.where(sig == 3, 0.1, sigma)
    return dict(xcur=xc, xprev=xp, xprevprev=xpp, lb=lb, ub=ub, sigma=sigma, ids=ids)


def sigma_init_arg(kind, n):
    if kind == "absent":
        return None
    if kind == "mixed":
        pick = (synth.u01(57, n) * 4).astype(np.int64)
        return np.choose(pick, [0.3 + synth.u01(58, n), np.zeros(n), np.full(n, -1.0), np.full(n, QNAN)])
    return np.full(n, {"positive": 0.3, "zero": 0.0, "negative": -1.0, "NaN": QNAN}[kind])


def weights(n):
    """non-negative x weights with exact zeros and subnormals"""
    w = 0.5 + synth.u01(60, n)
    pick = (synth.u01(61, n) * 16).astype(np.int64)
    w[pick == 0] = 0.0
    w[pick == 1] = 5e-324
    w[pick == 2] = 1e-310
    return w


def xtol_abs_mixed(n, d):
    """per-variable xtol_abs around |dx| = d: 0.0 (never below), inf (always below), d itself, just above, just below"""
    pick = (synth.u01(62, n) * 5).astype(np.int64)
    dd = np.where(np.isnan(d), 1.0, d)
    return np.choose(pick, [np.zeros(n), np.full(n, np.inf), dd, np.nextafter(dd, np.inf), np.nextafter(dd, -np.inf)])


# ---- assertions on what a kernel returned ------------------------------------------------------------------------------
def check_bits(got, want, what, ids=None):
    """uint64 equality of two float64 arrays: signs of zero and NaN payloads count"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(bits(got) != bits(want))
    if bad.size:
        j = int(bad[0])
        cls = f" [{class_name(ids, j)}]" if ids is not None else ""
        raise AssertionError(f"{what}: {bad.size} of {got.size} differ, first at {j}{cls}: got {got[j]!r} "
                             f"({int(bits(got)[j]):#018x}), want {want[j]!r} ({int(bits(want)[j]):#018x})")


def check_bits_or_nan(got, want, what):
    """uint64 equality where the model is a number; NaN where it is NaN (IEEE 754 leaves the payload of a NaN an
    operation produces to the implementation, and the CPU and the GPU choose differently)"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    nan = np.isnan(want)
    bad = np.flatnonzero(np.where(nan, ~np.isnan(got), bits(got) != bits(want)))
    if bad.size:
        j = int(bad[0])
        raise AssertionError(f"{what}: {bad.size} of {got.size} differ, first at {j}: got {got[j]!r} "
                             f"({int(bits(got)[j]):#018x}), want {want[j]!r} ({int(bits(want)[j]):#018x})")


def check_sum(got, terms, dep, what):
    """a float64 summation of `terms` whose longest chain has `dep` adds: within dep * 2^-53 * sum|t| of the exact
    sum (+1 for the rounding of fsum itself); NaN exactly when a term is NaN"""
    if np.isnan(terms).any():
        assert math.isnan(got), f"{what}: a term is NaN, got {got!r}"
        return
    exact = exact_sum(terms)
    scale = exact if not (terms < 0).any() else exact_sum(np.abs(terms))
    assert abs(got - exact) <= (dep + 1) * U * scale, f"{what}: got {got!r}, exact {exact!r}, sum|t| {scale!r}, depth {dep}"


def check_stop(got, xcur, xprev, w, xtol_abs, dep, what):
    """got = (dnorm, xnorm, all_below) of one end_outer / stop pass"""
    td, tx, count = stop_terms(xcur, xprev, w, xtol_abs)
    check_sum(got[0], td, dep, what + ": sum w|xc-xp|")
    check_sum(got[1], tx, dep, what + ": sum w|xc|")
    if xtol_abs is not None:
        assert bool(got[2]) == (count == 0), f"{what}: all below xtol_abs is {got[2]}, {count} variables are not"


def check_one_hot(got, term_d, term_x, below, what):
    """every term but one is +0.0: the sums are that term exactly"""
    check_bits([got[0], got[1]], [term_d, term_x], what + ": one-hot sums")
    if below is not None:
        assert bool(got[2]) == below, f"{what}: all below xtol_abs is {got[2]}, want {below}"


def check_guard(buf, off, n_local, what):
    """a probe buffer pre-filled with GUARD: nothing outside [off, off + n_local) was written"""
    g = bits(buf)
    want = bits(np.array([GUARD]))[0]
    outside = np.concatenate([g[:off], g[off + n_local:]])
    bad = np.flatnonzero(outside != want)
    assert bad.size == 0, f"{what}: {bad.size} entries outside the {n_local} target entries were written"


# ---- the oracle port's sigma functions on an operands() dict -------------------------------------------------------------
def port_sigma_init(lb, ub, init, sigma_min):
    import oracle_bindings as ob
    out = np.zeros(lb.size)
    ob.port().port_sigma_init(lb.size, ob._p(lb), ob._p(ub), ob._p(init), sigma_min, ob._p(out))
    return out


def port_sigma_update(variant, o, sigma_min):
    import oracle_bindings as ob
    out = o["sigma"].copy()
    ob.port().port_sigma_update(variant, out.size, ob._p(o["xcur"]), ob._p(o["xprev"]), ob._p(o["xprevprev"]),
                                ob._p(o["lb"]), ob._p(o["ub"]), sigma_min, ob._p(out))
    return out


def model_sigma_update(variant, o, sigma_min, **mutation):
    return sigma_update(variant, o["xcur"], o["xprev"], o["xprevprev"], o["lb"], o["ub"], o["sigma"], sigma_min,
                        **mutation)


# ---- operands of the penalty gradient and of the negation -----------------------------------------------------------------
PENALTY_ROWS = 20
# (count, kind) of every penalty case the GPU test runs.  "ordinary": coefficients of order 1, every row and its place
# in the order show in the result.  "zeros": 0.0, -0.0 and a subnormal in the first slots, ordinary ones after them.
# "huge", "inf", "nan": that coefficient in the LAST slot, where it cannot absorb the rows before it.
PENALTY_CASES = ([(c, "ordinary") for c in (1, 2, 15, 16)] + [(c, "zeros") for c in (0, 1, 2, 15, 16)] +
                 [(c, k) for k in ("huge", "inf", "nan") for c in (15, 16)])
PENALTY_CASES_LARGE = ((15, "ordinary"), (16, "ordinary"), (16, "zeros"), (16, "huge"))     # n > 100003


def penalty_arrays(n):
    """g and a block of PENALTY_ROWS rows; every tenth variable has zero rows, and -0.0 in g on every other of those
    (-0.0 + (+0.0) is +0.0, as in the host loop)"""
    g = 2.0 * synth.u01(70, n) - 1.0
    rows = np.stack([2.0 * synth.u01(71 + r, n) - 1.0 for r in range(PENALTY_ROWS)])
    rows[:, ::10] = 0.0
    g[::20] = -0.0
    return g, rows


def penalty_coefs(count, kind):
    """`count` coefficients and a non-identity selection of rows out of the block"""
    row_idx = [(7 * k + 3) % PENALTY_ROWS for k in range(count)]
    coefs = [1.37 + 0.37 * k for k in range(count)]
    if kind == "zeros":
        for k, c in zip(range(count), (0.0, -0.0, 5e-324)):
            coefs[k] = c
    elif kind != "ordinary":
        coefs[-1] = {"huge": 1e300, "inf": np.inf, "nan": QNAN}[kind]
    return coefs, row_idx


def penalty_mutations(g, rows, coefs, row_idx):
    """wrong results the penalty assertion has to reject in this case: name -> array"""
    count = len(coefs)
    out = {}
    ordinary = [k for k, c in enumerate(coefs) if 1e-300 < abs(c) < 1e100]
    if not ordinary or len(ordinary) < sum(1 for c in coefs if not abs(c) < 1e-300):
        return out      # only zeros and a subnormal, or a 1e300 / infinite / NaN last row that absorbs the rows before it
    out["last ordinary row dropped"] = penalty_axpy(g, rows, [c for k, c in enumerate(coefs) if k != ordinary[-1]],
                                                    [r for k, r in enumerate(row_idx) if k != ordinary[-1]])
    out["identity row selection"] = penalty_axpy(g, rows, coefs, list(range(count)))
    wrong = list(row_idx)
    wrong[ordinary[len(ordinary) // 2]] = (wrong[ordinary[len(ordinary) // 2]] + 1) % PENALTY_ROWS
    out["one wrong row index"] = penalty_axpy(g, rows, coefs, wrong)
    out["fused multiply-add"] = penalty_axpy_fused(g, rows, coefs, row_idx)
    if len(ordinary) >= 2:
        out["rows in reverse order"] = penalty_axpy(g, rows, coefs, row_idx, reverse=True)
    return out


def negate_values(n):
    v = (2.0 * synth.u01(80, n) - 1.0) * 1e3
    special = np.array([0.0, -0.0, 5e-324, -5e-324, 2.2e-308, np.inf, -np.inf, QNAN, SNAN,
                        negate_bits(np.array([QNAN]))[0], 1.0, -1.5e308])
    pick = (synth.u01(81, n) * 3).astype(np.int64) == 0
    return np.where(pick | (n <= 3), special[(np.arange(n) + n) % special.size], v)


# ---- the probe library -----------------------------------------------------------------------------------------------------
def build_probe(g):
    """tests/cpp/outer_kernels_probe.cu -> tests/_build/ with the library's compiler flags (g = __graft_entry__);
    rebuilt when the probe, any file of nlopt_b200/csrc or the command line changes.  Returns (so, ptxas log)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    csrc = os.path.join(root, "nlopt_b200", "csrc")
    src = os.path.join(root, "tests", "cpp", "outer_kernels_probe.cu")
    so = os.path.join(root, "tests", "_build", "libouter_kernels_probe.so")
    log = so + ".ptxas.log"
    tmp = so + f".{os.getpid()}.tmp"
    cmd = [g.NVCC, *g.ARCH, *g.NVCC_FLAGS, "-I" + csrc, "-shared", src, "-cudart", "shared", "-o"]
    head = " ".join(cmd) + "\n"
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
    fresh = os.path.exists(so) and os.path.exists(log) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps)
    if fresh:
        with open(log) as f:
            fresh = f.readline() == head
    if not fresh:
        os.makedirs(os.path.dirname(so), exist_ok=True)
        r = subprocess.run(cmd + [tmp], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        with open(log, "w") as f:
            f.write(head + r.stdout)
        os.replace(tmp, so)
    with open(log) as f:
        return so, f.read()
