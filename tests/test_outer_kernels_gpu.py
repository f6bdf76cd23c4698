"""The kernels that run between dual solves, against the references of tests/outer_model.py: sigma_init_kernel and
end_outer_kernel through the kernel-level handle (the library's own launch geometry), penalty_axpy_kernel,
negate_kernel, fill_kernel, sigma_init_kernel with a sigma index, end_outer_kernel as one rank of 2, 4 or 8 and
publish_kernel through tests/cpp/outer_kernels_probe.cu, and an AUGLAG run with more penalty rows than one launch takes.

sigma, the rotated points, the penalty gradient and the negation are compared as uint64; the stop sums against
math.fsum within depth * 2^-53 * sum|terms|, and exactly when all terms but one are zero.

The whole file (143 tests) takes 153 s of wall time on one NVIDIA H100 80GB HBM3 at a 700 W power limit, most of it in
the numpy models and math.fsum on the host."""
import ctypes as C

import numpy as np
import pytest

import nlopt_b200 as nl
import oracle_bindings as ob
import outer_model as om
import synth
from gpu_dual import DualHandle
from outer_model import model_sigma_update, port_sigma_init, port_sigma_update

pytestmark = pytest.mark.gpu

VARIANTS = (om.MMA, om.CCSAQ)
SIZES = (1, 2, 3, 255, 256, 257, 511, 512, 513, 1023, 1025, 4095, 4097, 100003, 299999, 300000, 1250000, 2500001)


def geometry_edges(limit=3_000_000):
    """the n on both sides of every change of groups_total (and with it groups_per_vshard): the geometry depends on n
    through its number of chunks, so a change lies between n = 512 c and 512 c + 1"""
    out, last = [], None
    for c in range(1, limit // om.CHUNK + 1):
        g = om.geometry(c * om.CHUNK)
        assert g.nchunks == c
        key = (g.groups_total, g.groups_per_vshard)
        if last is not None and key != last:
            out += [(c - 1) * om.CHUNK, (c - 1) * om.CHUNK + 1]
        last = key
    return out


def zero_inst(n, o):
    """what DualHandle.upload wants; only lb, ub and sigma matter to the kernels under test"""
    return dict(n=n, m=0, x=o["xprev"], lb=o["lb"], ub=o["ub"], sigma=o["sigma"], grad_f=np.zeros(n), grad_c=None,
                f0=0.0, rho=1.0, c0=[], rhoc=[])


def no_nan(o):
    return dict(o, xcur=np.where(np.isnan(o["xcur"]), 0.25, o["xcur"]))


def end_outer(h, n, o, k, smin, w=None, tol=None):
    """upload the operands, run one end-of-iteration pass, return (dn, xn, below), sigma, xprev, xprevprev"""
    h.upload(zero_inst(n, o))
    h.set_prev(o["xcur"], o["xprev"], o["xprevprev"])
    got = h.end_outer(k, smin, w, tol)
    return got, h.download("sigma"), h.download("xprev"), h.download("xprevprev")


def check_pass(h, n, variant, o, k, smin, w, tol, what):
    g = om.geometry(n)
    got, sigma, xprev, xprevprev = end_outer(h, n, o, k, smin, w, tol)
    if k > 1:
        om.check_bits(sigma, model_sigma_update(variant, o, smin), what + ": sigma against the model", o["ids"])
        om.check_bits(sigma, port_sigma_update(variant, o, smin), what + ": sigma against the oracle port", o["ids"])
    else:
        om.check_bits(sigma, o["sigma"], what + ": the first iteration leaves sigma as it is", o["ids"])
    om.check_bits(xprev, o["xcur"], what + ": xprev <- xcur", o["ids"])
    om.check_bits(xprevprev, o["xprev"], what + ": xprevprev <- xprev", o["ids"])
    om.check_stop(got, o["xcur"], o["xprev"], w, tol, om.depth(g), what)
    again = end_outer(h, n, o, k, smin, w, tol)
    om.check_bits(again[0][:2], got[:2], what + ": the same sums from a second pass")
    assert again[0][2] == got[2]
    om.check_bits(again[1], sigma, what + ": the same sigma from a second pass", o["ids"])


def sigma_and_stop_cases(n, variant, smins, inits):
    h = DualHandle(variant, n=n, m=0)
    shifts = range(0, om.NCLASS, n) if n <= 3 else (None,)
    w = om.weights(n)
    for shift in shifts:
        o = om.operands(n, variant, shift)
        with np.errstate(all="ignore"):
            tol = om.xtol_abs_mixed(n, np.abs(o["xcur"] - o["xprev"]))
        for smin in smins:
            what = f"n={n} variant={variant} shift={shift} sigma_min={smin}"
            h.upload(zero_inst(n, o))
            for kind in inits if not shift else inits[-1:]:      # every kind once per size, "mixed" on every shift
                init = om.sigma_init_arg(kind, n)
                h.sigma_init(init, smin)
                got = h.download("sigma")
                om.check_bits(got, om.sigma_init(o["lb"], o["ub"], init, smin), f"{what}: sigma init ({kind}) against the model", o["ids"])
                om.check_bits(got, port_sigma_init(o["lb"], o["ub"], init, smin), f"{what}: sigma init ({kind}) against the oracle port", o["ids"])
            # with the NaN class the sums are NaN and a NaN |dx| counts as below; without it they are numbers
            check_pass(h, n, variant, o, 2, smin, w, tol, what + " k=2 weights xtol_abs")
            check_pass(h, n, variant, no_nan(o), 3, smin, None, None, what + " k=3")
        # numbers everywhere, with weights: xtol_abs mixed (some variables are not below), and just above every |dx|
        # (all are below)
        clean = no_nan(o)
        d = np.abs(clean["xcur"] - clean["xprev"])
        what = f"n={n} variant={variant} shift={shift}"
        check_pass(h, n, variant, clean, 2, 0.25, w, om.xtol_abs_mixed(n, d), what + " k=2 weights, mixed xtol_abs, no NaN")
        check_pass(h, n, variant, clean, 1, 0.25, w, np.nextafter(d, np.inf), what + " k=1 weights, xtol_abs just above |dx|")


# ---- through the kernel-level handle --------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n", SIZES)
def test_sigma_rotation_and_stop_sums(built, variant, n):
    sigma_and_stop_cases(n, variant, om.SIGMA_MINS, om.INITS)


def test_sigma_rotation_and_stop_sums_at_geometry_edges(built):
    edges = geometry_edges()
    assert len(edges) >= 4
    for i, n in enumerate(edges):
        sigma_and_stop_cases(n, VARIANTS[(i // 2) % 2], (0.25,), ("mixed",))


def test_sigma_rotation_and_stop_sums_at_1e7(built):
    sigma_and_stop_cases(10**7, om.CCSAQ, (0.25,), ("mixed",))


def one_hot_positions(n, g, every_group):
    cuts = om.group_cuts(g) * om.CHUNK if every_group else np.arange(0, g.nchunks + 1) * om.CHUNK
    pos = {0, n - 1}
    for c in cuts[1:-1].tolist():
        pos |= {c - 1, c}
    return sorted(p for p in pos if 0 <= p < n)


@pytest.mark.parametrize("n,every_group", [(s, False) for s in SIZES if s <= 4097] + [(100003, True), (1250000, True)])
def test_one_hot_sums_are_exact(built, n, every_group):
    """all terms but one are +0.0: both sums are that term, wherever it sits, and `below` flips at |dx| == xtol_abs"""
    g = om.geometry(n)
    h = DualHandle(om.MMA, n=n, m=0)
    o = om.operands(n, om.MMA)
    h.upload(zero_inst(n, o))
    w = om.weights(n)
    zeros = np.zeros(n)
    positions = one_hot_positions(n, g, every_group)
    for i, j in enumerate(positions):
        v = -(1.0 + synth.u01(64, 1, j0=j)[0])
        xc = zeros.copy()
        xc[j] = v
        ww = None if i % 2 else w
        if ww is not None and ww[j] == 0.0:
            ww = ww.copy()
            ww[j] = 0.75
        term = abs(v) if ww is None else ww[j] * abs(v)
        what = f"n={n} one-hot at {j} ({'weights' if ww is not None else 'no weights'})"
        with_tol = every_group is False or i < 6 or i >= len(positions) - 6
        if not with_tol:
            h.set_prev(xc, zeros, None)
            om.check_one_hot(h.end_outer(1, 0.0, ww, None), term, term, None, what)
            continue
        for name, t, below in (("xtol_abs == |dx|", abs(v), False), ("just above", np.nextafter(abs(v), np.inf), True),
                               ("just below", np.nextafter(abs(v), 0.0), False)):
            tol = np.ones(n)
            tol[j] = t
            h.set_prev(xc, zeros, None)
            om.check_one_hot(h.end_outer(1, 0.0, ww, tol), term, term, below, f"{what}, {name}")


def test_xtol_abs_zero_and_inf(built):
    n = 4097
    h = DualHandle(om.MMA, n=n, m=0)
    o = om.operands(n, om.MMA)
    h.upload(zero_inst(n, o))
    x = o["xprev"]
    for name, xc, tol, below in (("xtol_abs = 0, dx = 0", x, np.zeros(n), False),
                                 ("xtol_abs = 0 where dx is NaN, inf elsewhere", np.where(np.arange(n) == 4096, om.QNAN, x),
                                  np.where(np.arange(n) == 4096, 0.0, np.inf), True),
                                 ("xtol_abs = inf", o["xcur"], np.full(n, np.inf), True)):
        h.set_prev(xc, x, None)
        assert h.end_outer(1, 0.0, None, tol)[2] == below, name


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n", (1, 3, 257, 511, 513, 4097, 100003))
def test_dual_evaluation_follows_the_floored_sigma(built, variant, n):
    """After sigma_init and end_outer with sigma_min = 0.25, at sizes that are not whole chunks, the next dual
    evaluation agrees with the oracle port on the downloaded sigma.  This does not by itself show that the padding
    lanes kept sigma = 0: there x, the bounds and the gradients are zero, so a padding lane adds exactly 0 to every sum
    whatever its sigma.  That the kernels write no entry beyond n_local is read directly from the guarded buffers of
    test_sigma_init_with_a_sigma_index and test_emulated_ranks_give_the_bits_of_one_rank (sigma_min = 0.25, tail
    slices)."""
    inst = synth.kernel_instance(n, 2)
    h = DualHandle(variant, inst)
    o = om.operands(n, variant)

    def dual_matches(what):
        # the comparison of the dual kernels' parity tests: x* bit for bit, sums to 1e-12 (|value| + n)
        cur = dict(inst, sigma=h.download("sigma"))
        got, want = h.eval(inst["y"], want_xcur=True), ob.port_dual(variant, cur)
        assert np.array_equal(got["xcur"], want["xcur"], equal_nan=True), what
        for key in ("ret", "g0", "w"):
            assert abs(got[key] - want[key]) <= 1e-12 * (abs(want[key]) + n), (what, key, got[key], want[key])
        for i in range(inst["m"]):
            assert abs(got["gc"][i] - want["gc"][i]) <= 1e-12 * (abs(want["gc"][i]) + n), (what, i)

    h.sigma_init(None, 0.25)
    assert np.all(h.download("sigma") >= 0.25)
    dual_matches(f"n={n} variant={variant} after sigma_init(sigma_min=0.25)")
    x = inst["x"]
    h.set_prev(x + 0.01 * (o["xcur"] - o["xprev"] > 0), x, x - 0.01)
    h.end_outer(2, 0.25)
    assert np.all(h.download("sigma") >= 0.25)
    dual_matches(f"n={n} variant={variant} after end_outer(k=2, sigma_min=0.25)")


# ---- through the probe ----------------------------------------------------------------------------------------------------
class Probe:
    def __init__(self, so):
        L = self.L = C.CDLL(so, mode=C.RTLD_LOCAL)
        dp, z, i = ob.dp, C.c_size_t, C.c_int
        L.okp_error.restype = C.c_char_p
        L.okp_sm_count.argtypes = [C.POINTER(C.c_int)]
        L.okp_penalty.argtypes = [dp, z, z, dp, z, z, z, dp, C.POINTER(C.c_int), i, i]
        L.okp_negate.argtypes = [dp, z, z, z, i, i]
        L.okp_fill.argtypes = [dp, z, z, C.c_double, z, i]
        L.okp_sigma_init.argtypes = [dp, C.POINTER(C.c_ushort), z, z, dp, dp, dp, C.c_double, z, i]
        L.okp_end_outer.argtypes = [C.POINTER(C.c_ulonglong), dp, dp, dp, dp, z, z, dp, dp, dp, dp, i, C.c_double,
                                    C.c_double, i, dp, dp]
        L.okp_publish.argtypes = [dp, dp]
        sms = C.c_int(0)
        self.check(L.okp_sm_count(C.byref(sms)))
        self.sms = sms.value

    def check(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.okp_error().decode())

    def grids(self, work):
        """one CTA; the library's rule for element-wise kernels (grid_for in device_backend.cu): one thread per
        element, at most 16 CTAs per SM; more CTAs than there is work"""
        blocks = -(-work // om.THREADS)
        return (1, max(1, min(blocks, 16 * self.sms)), blocks + 3)

    def end_outer(self, g, o, bufs, off, w, tol, update_sigma, variant, smin, publish, out_dev):
        """one rank's launch on its slice; bufs = guarded xprev, xprevprev (or None), sigma"""
        sl = slice(g.j0, g.j0 + g.n_local)
        geo = (C.c_ulonglong * 8)(g.n_local, g.nchunks, g.chunk0, g.groups_total, g.group0, g.groups_per_vshard,
                                  g.local_vshards, g.groups_local)
        cut = [np.ascontiguousarray(a[sl]) if a is not None else None for a in (o["xcur"], o["lb"], o["ub"], w, tol)]
        out4 = np.zeros(4)
        self.check(self.L.okp_end_outer(geo, ob._p(cut[0]), ob._p(bufs[0]), ob._p(bufs[1]), ob._p(bufs[2]), bufs[0].size,
                                        off, ob._p(cut[1]), ob._p(cut[2]), ob._p(cut[3]), ob._p(cut[4]), int(update_sigma),
                                        om.KAPPA[variant], smin, int(publish), ob._p(out_dev), ob._p(out4)))
        return out4


@pytest.fixture(scope="module")
def probe(built):
    return Probe(om.build_probe(built)[0])


def guarded(values, rows_before=1):
    """a buffer of GUARD with `values` in it at a 4 KB aligned offset, the row padded beyond n_local, a guard row after"""
    n = values.size
    ld = (n // om.CHUNK + 1) * om.CHUNK
    off = rows_before * om.CHUNK
    buf = np.full(off + ld + om.CHUNK, om.GUARD)
    buf[off:off + n] = values
    return buf, off


def target(buf, off, n, what):
    om.check_guard(buf, off, n, what)
    return buf[off:off + n]


@pytest.mark.parametrize("n", SIZES)
def test_penalty_gradient_bits(probe, n):
    """Every (count, kind) of om.PENALTY_CASES on one CTA, the library's grid and an oversized grid; tests/
    test_outer_kernels.py shows on the same operands which wrong gradients the assertion rejects.  Above n = 100003
    the 400 MB row block is sent once per launch, so only om.PENALTY_CASES_LARGE run, on the library's grid, and the
    16 ordinary rows also on the other two grids."""
    large = n > 100003
    g, rows = om.penalty_arrays(n)
    ld = (n // om.CHUNK + 1) * om.CHUNK
    block = np.full((rows.shape[0], ld), om.GUARD)
    block[:, :n] = rows
    for count, kind in om.PENALTY_CASES_LARGE if large else om.PENALTY_CASES:
        coefs, row_idx = om.penalty_coefs(count, kind)
        want = om.penalty_axpy(g, rows, coefs, row_idx)
        if count and kind in ("ordinary", "zeros"):
            assert np.signbit(g[0]) and not np.signbit(want[0]), "-0.0 in g with zero products comes out as +0.0"
            assert np.isfinite(want).all()
        c = np.array(coefs + [0.0], dtype=np.float64)
        r = np.array(row_idx + [0], dtype=np.int32)
        grids = probe.grids(n)
        for grid in grids[1:2] if large and (count, kind) != (16, "ordinary") else grids:
            buf, off = guarded(g)
            probe.check(probe.L.okp_penalty(ob._p(buf), buf.size, off, ob._p(block), block.size, ld, n, ob._p(c),
                                            r.ctypes.data_as(C.POINTER(C.c_int)), count, grid))
            what = f"penalty_axpy_kernel n={n} rows={count} ({kind} coefficients) grid={grid}"
            om.check_bits_or_nan(target(buf, off, n, what), want, what)


@pytest.mark.parametrize("n", (1, 2, 3, 511, 512, 513, 100003, 2500001))
def test_negation_bits(probe, n):
    v = om.negate_values(n)
    for grid in probe.grids((n + 1) // 2):
        for times, want in ((1, om.negate_bits(v)), (2, v)):
            buf, off = guarded(v)
            probe.check(probe.L.okp_negate(ob._p(buf), buf.size, off, n, grid, times))
            what = f"negate_kernel n={n} grid={grid} applied {times}x"
            om.check_bits(target(buf, off, n, what), want, what)


@pytest.mark.parametrize("n", SIZES)
def test_fill_writes_n_local_entries(probe, n):
    for value in (2.0, -0.0, om.QNAN):
        for grid in probe.grids(n):
            buf, off = guarded(np.full(n, om.GUARD))
            probe.check(probe.L.okp_fill(ob._p(buf), buf.size, off, value, n, grid))
            what = f"fill_kernel n={n} value={value!r} grid={grid}"
            om.check_bits(target(buf, off, n, what), np.full(n, value), what)


@pytest.mark.parametrize("n", SIZES)
def test_sigma_init_with_a_sigma_index(probe, n):
    o = om.operands(n, om.MMA)
    init = om.sigma_init_arg("mixed", n)
    for grid in probe.grids(n):
        buf, off = guarded(np.full(n, om.GUARD))
        sidx = np.full(buf.size, 0xBEEF, dtype=np.uint16)
        probe.check(probe.L.okp_sigma_init(ob._p(buf), sidx.ctypes.data_as(C.POINTER(C.c_ushort)), buf.size, off,
                                           ob._p(o["lb"]), ob._p(o["ub"]), ob._p(init), 0.25, n, grid))
        what = f"sigma_init_kernel n={n} grid={grid}"
        om.check_bits(target(buf, off, n, what), port_sigma_init(o["lb"], o["ub"], init, 0.25), what, o["ids"])
        assert np.all(sidx[off:off + n] == 1), what + ": the sigma index of every variable is entry 1"
        assert np.all(sidx[:off] == 0xBEEF) and np.all(sidx[off + n:] == 0xBEEF), what + ": index written outside the row"


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n", (4097, 300001, 2500001))
def test_emulated_ranks_give_the_bits_of_one_rank(built, probe, variant, n):
    """end_outer_kernel once per rank of 2, 4 and 8 on the rank's slice, then publish_kernel on the gathered
    virtual-shard sums: the four published values, sigma and the rotated points are those of the one-rank pass"""
    o = no_nan(om.operands(n, variant))
    w = om.weights(n)
    tol = om.xtol_abs_mixed(n, np.abs(o["xcur"] - o["xprev"]))
    count = om.stop_terms(o["xcur"], o["xprev"], w, tol)[2]
    h = DualHandle(variant, n=n, m=0)
    (dn, xn, below), sigma1, xprev1, xprevprev1 = end_outer(h, n, o, 2, 0.25, w, tol)
    assert below == (count == 0)
    for world in (2, 4, 8):
        out_dev = np.zeros(32)
        sigma, xprev, xprevprev = np.zeros(n), np.zeros(n), np.zeros(n)
        for rank in range(world):
            g = om.geometry(n, rank, world)
            assert g.n_local > 0
            sl = slice(g.j0, g.j0 + g.n_local)
            bufs = [guarded(o[k][sl])[0] for k in ("xprev", "xprevprev", "sigma")]
            off = om.CHUNK
            probe.end_outer(g, o, bufs, off, w, tol, True, variant, 0.25, False, out_dev)
            what = f"n={n} variant={variant} rank {rank} of {world}"
            xprev[sl] = target(bufs[0], off, g.n_local, what + " xprev")
            xprevprev[sl] = target(bufs[1], off, g.n_local, what + " xprevprev")
            sigma[sl] = target(bufs[2], off, g.n_local, what + " sigma")
        out4 = np.zeros(4)
        probe.check(probe.L.okp_publish(ob._p(out_dev), ob._p(out4)))
        what = f"n={n} variant={variant} world={world}"
        om.check_bits(out4, [dn, xn, float(count), 0.0], what + ": published sums against one rank")
        om.check_bits(sigma, sigma1, what + ": sigma", o["ids"])
        om.check_bits(xprev, xprev1, what + ": xprev", o["ids"])
        om.check_bits(xprevprev, xprevprev1, what + ": xprevprev", o["ids"])


@pytest.mark.parametrize("n", (1, 3, 513, 4097, 100003, 2500001))
def test_keep_the_point_form(built, probe, n):
    """update_sigma = 0 and a null xprevprev (the AUGLAG outer loop's stop test): the sums, xprev <- xcur, and sigma
    is not touched"""
    o = no_nan(om.operands(n, om.MMA))
    w = om.weights(n)
    tol = om.xtol_abs_mixed(n, np.abs(o["xcur"] - o["xprev"]))
    g = om.geometry(n)
    for ww, tt in ((None, None), (w, tol)):
        xprev, off = guarded(o["xprev"])
        sigma, _ = guarded(o["sigma"])
        out4 = probe.end_outer(g, o, [xprev, None, sigma], off, ww, tt, False, om.MMA, 0.25, True, np.zeros(32))
        what = f"keep-the-point pass n={n} {'weights xtol_abs' if ww is not None else 'plain'}"
        om.check_stop((out4[0], out4[1], out4[2] == 0.0), o["xcur"], o["xprev"], ww, tt, om.depth(g), what)
        if tt is not None:
            assert out4[2] == om.stop_terms(o["xcur"], o["xprev"], ww, tt)[2], what
        assert out4[3] == 0.0
        om.check_bits(target(xprev, off, n, what), o["xcur"], what + ": xprev <- xcur", o["ids"])
        om.check_bits(target(sigma, off, n, what), o["sigma"], what + ": sigma untouched", o["ids"])
        # the same sums as the full pass of the handle on the same points
        h = DualHandle(om.MMA, n=n, m=0)
        full = end_outer(h, n, o, 1, 0.25, ww, tt)[0]
        om.check_bits(out4[:2], full[:2], what + ": the sums of the full pass")


# ---- more penalty rows than one penalty_axpy_kernel launch takes ------------------------------------------------------------
def test_auglag_with_37_penalty_rows_matches_the_cpu_backend(built, hosttest_lib):
    """5 equalities + 32 inequalities: eval_penalty_objective splits the active rows into launches of 16.  At x0 the
    inequalities are active, inactive and (every fourth) exactly on the boundary fc == 0, which is inactive."""
    n = 4097
    j = np.arange(n)
    wobj = 1.0 + 0.5 * np.sin(0.37 * j)
    x0 = 0.1 + 0.05 * np.cos(0.11 * j)

    def f(x, grad):
        if grad.size:
            grad[:] = wobj + x
        return float(np.dot(wobj, x) + 0.5 * np.dot(x, x))

    def linear(a, b):
        def c(x, grad):
            if grad.size:
                grad[:] = a
            return float(np.dot(a, x) - b)
        return c

    def pin(k, b):                        # x_k - b <= 0: exactly 0 at x0 when b = x0[k]
        def c(x, grad):
            if grad.size:
                grad[:] = 0.0
                grad[k] = 1.0
            return float(x[k] - b)
        return c

    eqs = [linear(np.cos(0.01 * (k + 1) * j) / n, 0.02 * k) for k in range(5)]
    ineqs = []
    for k in range(32):
        if k % 4 == 0:
            ineqs.append(pin(100 * k + 7, x0[100 * k + 7]))
        else:
            a = np.sin(0.003 * (k + 1) * j + k) / n
            ineqs.append(linear(a, float(np.dot(a, x0)) + (0.01 if k % 4 == 1 else -0.01)))
    none = np.empty(0)
    values = np.array([c(x0, none) for c in ineqs])
    assert np.count_nonzero(values > 0) + 5 > 16 and np.count_nonzero(values == 0) == 8 and np.any(values < 0)

    def run(lib):
        o = nl.opt(nl.LD_AUGLAG, n, library=lib)
        o.set_lower_bounds(np.full(n, -2.0)); o.set_upper_bounds(np.full(n, 2.0))
        o.set_min_objective(f)
        for c in ineqs:
            o.add_inequality_constraint(c, 1e-8)
        for c in eqs:
            o.add_equality_constraint(c, 1e-8)
        o.set_xtol_rel(1e-12)
        o.set_maxeval(40)
        x = o.optimize(x0.copy())
        return o.last_optimize_result(), o.get_numevals(), o.last_optimum_value(), x

    a, b = run(None), run(hosttest_lib)
    assert a[0] == b[0] and a[1] == b[1], (a[:3], b[:3])
    assert abs(a[2] - b[2]) <= 1e-7 * max(1.0, abs(b[2])), (a[2], b[2])
    assert np.max(np.abs(a[3] - b[3])) <= 1e-5
