"""The exact-sum check of tests/dual_sums_model.py on the CPU, on every instance tests/test_dual_sums_gpu.py runs.

(a) The oracle port's sequential sums (mma.c:119-129, ccsa_quadratic.c:133-140 restated) pass the check with the
    depth of a sequential sum, n, the constant leading the chain: the terms of closed_form_model and the constants, in
    the host's order, are those of the reference.  x* of the port is the model's bit for bit.
(b) Wrong sums fail it: one variable's terms dropped, one group record dropped or counted twice, one virtual shard
    dropped, one group summed at the previous multipliers (a stale generation), and the sums of two rows swapped.  Each
    is built from the exact sums of the pieces, so it is what a kernel with that fault would return, up to rounding;
    the depth is that of the GPU form that runs the instance.  With -s the file prints which sums rejected each one,
    and how many of them the older parity tolerance 1e-12 (|value| + n) would have let through.
"""
import numpy as np
import pytest

import closed_form_model as cf
import dual_sums_model as dm
import oracle_bindings as ob
import outer_model as om

VARIANT_NAMES = {dm.MMA: "MMA", dm.CCSAQ: "CCSAQ"}


def case_id(c):
    v, m, fam, n = c
    return f"{VARIANT_NAMES[v]}-m{m}-{fam.replace(' ', '_')}-{n}"


CASES = dm.all_cases()
WIDE_CASES = [(v, m, n, i % 2 == 1) for v in (dm.MMA, dm.CCSAQ) for i, (m, n) in enumerate(dm.WIDE)]


@pytest.mark.parametrize("variant,m,family,n", CASES, ids=[case_id(c) for c in CASES])
def test_the_port_sums_within_a_sequential_depth(built, variant, m, family, n):
    inst = dm.instance(family, n, m, variant)
    xc, terms, consts = dm.expected(variant, inst, inst["y"])
    with np.errstate(all="ignore"):
        p = ob.port_dual(variant, inst)
    assert cf.same_bits(p["xcur"], xc).all(), "x* of the port differs from the model"
    got = dm.raw_values(np.concatenate([[p["ret"], p["g0"], p["w"]], p["gc"]]))
    dm.check_dual_sums(got, dm.leading_constants(terms, consts), dm.depth("port", om.geometry(n), m), None,
                       f"oracle port {case_id((variant, m, family, n))}")


def old_tolerance_accepts(got, want, n):
    """the parity tolerance of test_gpu_parity.check_dual on the constant-plus-sum values"""
    with np.errstate(all="ignore"):
        return bool(np.all((np.abs(got - want) <= 1e-12 * (np.abs(want) + n)) | (np.isnan(got) & np.isnan(want))))


def check_mutants(variant, inst, form, what):
    n, m = inst["n"], inst["m"]
    g = om.geometry(n)
    y = np.asarray(inst["y"], dtype=np.float64)
    _, terms, consts = dm.expected(variant, inst, y)
    ref = dm.Sums(terms, dm.depth(form, g, m), consts)
    right = dm.apply_constants([ref.want[k][1] if ref.want[k][0] == "num" else np.nan for k in range(ref.k)], consts)
    lines, lenient = [], 0
    for name, wrong in dm.mutants(variant, inst, g, y, dm.previous_y(y)).items():
        if wrong is None:
            lines.append(f"  {name}: not applicable (m = {m}, {int(np.count_nonzero(np.isnan(inst['c0'])))} rows off)")
            continue
        bad = ref.rejected(wrong)
        assert bad, f"{what}: the check accepts the mutant '{name}'"
        lenient += old_tolerance_accepts(np.asarray(wrong), right, n)
        lines.append(f"  {name}: rejected by {', '.join(dm.sum_name(k) for k in bad)}")
    print(f"{what} (depth {ref.dep}): {lenient} mutants within the old tolerance\n" + "\n".join(lines))


@pytest.mark.parametrize("variant,m,family,n", CASES, ids=[case_id(c) for c in CASES])
def test_the_check_rejects_wrong_sums(built, variant, m, family, n):
    check_mutants(variant, dm.instance(family, n, m, variant), "eval", case_id((variant, m, family, n)))


@pytest.mark.parametrize("variant,m,n,nan_rows", WIDE_CASES,
                         ids=[f"{VARIANT_NAMES[v]}-m{m}-{n}{'-NaN_rows' if r else ''}" for v, m, n, r in WIDE_CASES])
def test_the_check_rejects_wrong_sums_of_the_wide_kernel(built, variant, m, n, nan_rows):
    check_mutants(variant, dm.wide_instance(m, n, variant, nan_rows), "wide", f"wide {VARIANT_NAMES[variant]} m={m} n={n}")


def test_the_depths_follow_the_geometry(built):
    """2 c + 31 + ceil(P / 256) for the register, TMA and solve forms; the wide kernel's rows need no more"""
    for n in (1, 4097, 100003, 10 ** 7):
        g = om.geometry(n)
        c = int(np.diff(om.group_cuts(g)).max())
        p = -(-int(g.groups_per_vshard) // 256)
        for form in ("eval", "tma", "solve"):
            assert dm.depth(form, g, 4) == 2 * c + 31 + p
        assert dm.depth("wide", g, 2048) == 2 * c + 31 + p
        assert dm.depth("port", g, 4) == n
