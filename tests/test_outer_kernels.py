"""The references of tests/outer_model.py, without a GPU: the sigma models equal the oracle port bit for bit, the stop
model decides like the port's nlopt_stop_x, every assertion used on the kernels' output rejects a deliberately wrong
model, and the probe that launches the kernels compiles for sm_90a without spills."""
import re

import numpy as np
import pytest

import oracle_bindings as ob
import outer_model as om
from outer_model import model_sigma_update, port_sigma_init, port_sigma_update

PROBE_KERNELS = ("penalty_axpy_kernel", "negate_kernel", "fill_kernel", "sigma_init_kernel", "end_outer_kernel",
                 "publish_kernel")
SIZES = (1, 2, 3, 255, 513, 4097, 100003)
VARIANTS = (om.MMA, om.CCSAQ)


def rejects(check, *args):
    with pytest.raises(AssertionError):
        check(*args)


# ---- the models against the oracle port ---------------------------------------------------------------------------------
def test_operands_hold_every_class():
    o = om.operands(om.NCLASS, om.MMA, shift=0)
    osc, bnd, sig = o["ids"]
    assert len(set(zip(osc.tolist(), bnd.tolist(), sig.tolist()))) == om.NCLASS
    with np.errstate(all="ignore"):
        prod = (o["xcur"] - o["xprev"]) * (o["xprev"] - o["xprevprev"])
    assert np.all(prod[osc == 0] < 0) and np.all(prod[osc == 1] > 0)
    for k in (2, 3, 4, 5):
        assert np.all(prod[osc == k] == 0), om.OSC[k]
    assert not np.signbit(prod[osc == 4]).any() and np.signbit(prod[osc == 5]).all()
    assert np.isnan(prod[osc == 6]).all()
    hashed = om.class_ids(100003)
    assert len(set(zip(*[i.tolist() for i in hashed]))) == om.NCLASS


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("n", SIZES)
def test_sigma_models_equal_the_oracle_port(built, variant, n):
    shifts = range(0, om.NCLASS, n) if n <= 3 else (None,)
    for shift in shifts:
        o = om.operands(n, variant, shift)
        for smin in om.SIGMA_MINS:
            what = f"n={n} variant={variant} shift={shift} sigma_min={smin}"
            om.check_bits(model_sigma_update(variant, o, smin), port_sigma_update(variant, o, smin),
                          "sigma update, " + what, o["ids"])
            for kind in om.INITS:
                init = om.sigma_init_arg(kind, n)
                om.check_bits(om.sigma_init(o["lb"], o["ub"], init, smin), port_sigma_init(o["lb"], o["ub"], init, smin),
                              f"sigma init ({kind}), " + what, o["ids"])


@pytest.mark.parametrize("n", SIZES)
def test_stop_model_decides_like_the_port(built, n):
    o = om.operands(n, om.MMA)
    xc, xp = o["xcur"], o["xprev"]
    w = om.weights(n)
    with np.errstate(all="ignore"):
        d = np.abs(xc - xp)
    cases = {"mixed": om.xtol_abs_mixed(n, d), "zero": np.zeros(n), "inf": np.full(n, np.inf),
             "just above": np.nextafter(np.where(np.isnan(d), 1.0, d), np.inf), "none": None}
    for name, tol in cases.items():
        for ww in (None, w):
            td, tx, count = om.stop_terms(xc, xp, ww, tol)
            # xtol_rel = 0: the sums decide nothing (x < 0 and NaN < 0 are false), only the count does
            want = ob.port().port_stop_x(n, ob._p(xc), ob._p(xp), ob._p(ww), 0.0, ob._p(tol))
            assert om.stop_decision(np.sum(td), np.sum(tx), count, 0.0) == bool(want), (name, n)
    # the relative test, on operands without NaN so that the sums are numbers
    xc = np.where(np.isnan(xc), 0.25, xc)
    td, tx, count = om.stop_terms(xc, xp, w, cases["zero"])
    for rel in (0.0, 1e-9, 10.0):
        want = ob.port().port_stop_x(n, ob._p(xc), ob._p(xp), ob._p(w), rel, ob._p(cases["zero"]))
        assert om.stop_decision(om.exact_sum(td), om.exact_sum(tx), count, rel) == bool(want), rel


def test_nan_difference_counts_as_below(built):
    xc, xp = np.array([om.QNAN, 1.0]), np.array([0.0, 1.0])
    tol = np.array([0.0, 1e-3])
    assert om.stop_terms(xc, xp, None, tol)[2] == 0
    assert ob.port().port_stop_x(2, ob._p(xc), ob._p(xp), None, 0.0, ob._p(tol)) == 1


# ---- mutation checks: the assertions of the GPU tests reject wrong results ------------------------------------------------
@pytest.mark.parametrize("n", (3, 513, 4097, 100003))
def test_sum_assertions_reject_a_dropped_and_a_doubled_variable(built, n):
    g = om.geometry(n)
    dep = om.depth(g)
    o = om.operands(n, om.MMA)
    xc, xp = np.where(np.isnan(o["xcur"]), 0.25, o["xcur"]), o["xprev"]
    xc[-1], xp[-1] = 0.75, 0.5                     # the last variable carries ordinary terms
    for w in (None, 0.5 + om.synth.u01(63, n)):
        td, tx, _ = om.stop_terms(xc, xp, w)
        good = (float(np.sum(td)), float(np.sum(tx)), False)         # pairwise summation: a plain float64 sum
        om.check_stop(good, xc, xp, w, None, dep, "numpy sum")
        dropped = (om.exact_sum(td[:-1]), om.exact_sum(tx[:-1]), False)
        doubled = (om.exact_sum(td) + float(td[-1]), om.exact_sum(tx) + float(tx[-1]), False)
        rejects(om.check_stop, dropped, xc, xp, w, None, dep, "last variable dropped")
        rejects(om.check_stop, doubled, xc, xp, w, None, dep, "variable n-1 read twice")
    # one-hot: the only non-zero term sits on the last variable
    rejects(om.check_one_hot, (0.0, 0.0, True), 0.25, 0.75, None, "last variable dropped")
    rejects(om.check_one_hot, (0.5, 1.5, True), 0.25, 0.75, None, "variable n-1 read twice")
    om.check_one_hot((0.25, 0.75, True), 0.25, 0.75, True, "exact")


def test_count_assertion_rejects_a_strict_comparison(built):
    n = 513
    o = om.operands(n, om.MMA)
    xc, xp = np.where(np.isnan(o["xcur"]), 0.25, o["xcur"]), o["xprev"]
    d = np.abs(xc - xp)
    tol = np.full(n, np.inf)
    tol[77] = d[77]                                # |dx| == xtol_abs on one variable: not below
    td, tx, count = om.stop_terms(xc, xp, None, tol)
    strict = om.stop_terms(xc, xp, None, tol, strict=True)[2]
    assert (count, strict) == (1, 0)
    dep = om.depth(om.geometry(n))
    om.check_stop((om.exact_sum(td), om.exact_sum(tx), count == 0), xc, xp, None, tol, dep, "model")
    rejects(om.check_stop, (om.exact_sum(td), om.exact_sum(tx), strict == 0), xc, xp, None, tol, dep, "> for >=")
    rejects(om.check_one_hot, (d[77], 0.0, True), d[77], 0.0, False, "> for >=")


@pytest.mark.parametrize("variant", VARIANTS)
def test_sigma_assertion_rejects_wrong_updates(built, variant):
    o = om.operands(4 * om.NCLASS, variant, shift=0)
    for smin in om.SIGMA_MINS:
        om.check_bits(model_sigma_update(variant, o, smin), port_sigma_update(variant, o, smin), "model", o["ids"])
    # each wrong model at the sigma_min that lets it show: 0.25 lies above kappa * range and hides the floor's kappa
    for name, smin, mutation in (("cap / floor with a one-sided infinite bound", 0.25, dict(one_sided_clamp=True)),
                                 ("kappa of the other variant", 0.0, dict(kappa=om.KAPPA[1 - variant])),
                                 ("sigma_min floor skipped", 0.25, dict(floor=False))):
        with pytest.raises(AssertionError) as e:
            om.check_bits(model_sigma_update(variant, o, smin, **mutation), port_sigma_update(variant, o, smin), name,
                          o["ids"])
        assert " | " in str(e.value), "a failure names the operand class"
    want = port_sigma_update(variant, o, 0.25)
    rejects(om.check_bits, o["sigma"], want, "sigma left as it was")
    init = om.sigma_init_arg("mixed", o["lb"].size)
    rejects(om.check_bits, om.sigma_init(o["lb"], o["ub"], init, 0.0), port_sigma_init(o["lb"], o["ub"], init, 0.25),
            "sigma_min floor skipped in sigma init")


@pytest.mark.parametrize("n", (513, 4097))
@pytest.mark.parametrize("count,kind", om.PENALTY_CASES)
def test_penalty_assertion_rejects_wrong_gradients(built, n, count, kind):
    """on exactly the operands the GPU test gives the kernel: rows dropped, selected by identity or by one wrong index,
    fused multiply-add, reverse order.  The cases whose last coefficient is 1e300, infinite or NaN, and those with only
    zeros and a subnormal, pin special values and carry no such mutation: that row absorbs what came before it."""
    g, rows = om.penalty_arrays(n)
    coefs, row_idx = om.penalty_coefs(count, kind)
    assert row_idx != list(range(count)) or count == 0
    want = om.penalty_axpy(g, rows, coefs, row_idx)
    om.check_bits_or_nan(want.copy(), want, "model")
    wrong = om.penalty_mutations(g, rows, coefs, row_idx)
    expect = {"last ordinary row dropped", "identity row selection", "one wrong row index", "fused multiply-add"}
    if kind == "ordinary" or (kind == "zeros" and count >= 15):
        assert expect <= set(wrong) and (count < 2 or "rows in reverse order" in wrong), sorted(wrong)
    else:
        assert not wrong
    for name, got in wrong.items():
        rejects(om.check_bits_or_nan, got, want, name)
    if count:
        assert np.signbit(g[0]) and not np.signbit(want[0]) or np.isnan(want[0]), "-0.0 + (+0.0) is +0.0"
        rejects(om.check_bits_or_nan, g, want, "g left as it was")


def test_penalty_assertion_wants_a_nan_where_the_model_has_one():
    rejects(om.check_bits_or_nan, np.array([1.0]), np.array([np.nan]), "a number where the model is NaN")
    rejects(om.check_bits_or_nan, np.array([-0.0]), np.array([0.0]), "the sign of zero")
    om.check_bits_or_nan(np.array([om.QNAN, np.inf]), np.array([np.nan, np.inf]), "any NaN")


def test_negate_assertion_rejects_a_subtraction_from_zero(built):
    v = om.negate_values(513)
    want = om.negate_bits(v)
    om.check_bits(om.negate_bits(want), v, "twice")
    assert np.array_equal(om.bits(want) >> np.uint64(63), 1 - (om.bits(v) >> np.uint64(63)))
    with np.errstate(all="ignore"):
        wrong = 0.0 - v
    assert not np.signbit(wrong[om.bits(v) == 0]).any(), "0.0 - (+0.0) is +0.0, the negation is -0.0"
    rejects(om.check_bits, wrong, want, "0.0 - g")


def test_guard_assertion_rejects_a_write_outside_the_row(built):
    buf = np.full(3 * 512, om.GUARD)
    buf[512:512 + 100] = 1.0
    om.check_guard(buf, 512, 100, "clean")
    for j in (511, 612, 3 * 512 - 1):
        bad = buf.copy()
        bad[j] = 0.0
        rejects(om.check_guard, bad, 512, 100, f"write at {j}")


# ---- the probe ---------------------------------------------------------------------------------------------------------
def test_probe_compiles_for_sm_90a_without_spills(built):
    _, log = om.build_probe(built)
    seen = {}
    for name, stores, loads in re.findall(r"Function properties for (\S+)\s+\d+ bytes stack frame, (\d+) bytes spill stores, "
                                          r"(\d+) bytes spill loads", log):
        seen[name] = (int(stores), int(loads))
    assert "sm_90a" in log
    for k in PROBE_KERNELS:
        hits = {name: v for name, v in seen.items() if k in name}
        assert hits, f"{k} is not in the probe"
        assert all(v == (0, 0) for v in hits.values()), (k, hits)
