"""Uniform box bounds (nlopt_set_lower_bounds1 / nlopt_set_upper_bounds1) reach the default dual kernels as two scalars
instead of two arrays streamed from HBM.  The closed forms see the same values either way, so a run must give the same
bits as the same bounds passed as arrays (which take the array path), and nlopt_b200_stats::dual_operand_bytes must
show which path ran."""
import numpy as np
import pytest

import nlopt_b200 as nl
import problems as P
from test_gpu_parity import _run

pytestmark = pytest.mark.gpu

# the register-form persistent solve kernel (3 CTAs/SM), its 2-CTAs/SM form, and one dual_eval_kernel launch per evaluation
PATHS = {"solve": dict(b200_solve_tma=0), "solve_2cta": dict(b200_solve_tma=0, b200_solve_minb=2),
         "host_driven": dict(b200_fused_solve=0)}


def _ld(n):
    return -(-n // 512) * 512          # one rank's padded shard length: whole 512-variable chunks


@pytest.mark.parametrize("alg", [nl.LD_MMA, nl.LD_CCSAQ])
@pytest.mark.parametrize("n,m", [(3, 1), (3, 16), (100001, 2), (100001, 16), (300000, 3), (300000, 4), (300000, 8),
                                 (1500000, 1)])
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("lb", [-0.3, -0.0])
def test_scalar_bounds_equal_array_bounds(built, alg, n, m, path, lb):
    """A separable quadratic whose minimiser lies outside the box for most coordinates, so that x*(y) is clamped onto
    both bounds (onto -0.0 itself in the second box), with m dense linear constraints; m = 3 runs the kernels whose row
    loops are predicated."""
    ub = 0.3
    f, _ = P.quad_problem(n)
    cons = [P.lin_constraint(k, n) for k in range(m)]
    x0 = np.full(n, 0.1)
    runs = [_run(alg, n, f, cons, [1e-8] * m, lo, hi, x0, maxeval=12, **PATHS[path])
            for lo, hi in ((lb, ub), (np.full(n, lb), np.full(n, ub)))]
    a, b = runs
    sa, sb = a["opt"].get_stats(), b["opt"].get_stats()
    assert a["ret"] == b["ret"] and a["numevals"] == b["numevals"] and a["minf"] == b["minf"]
    assert sa["dual_evals"] == sb["dual_evals"] and sa["dual_solves"] == sb["dual_solves"]
    assert np.array_equal(a["x"].view(np.uint64), b["x"].view(np.uint64))
    # operand bytes: (3 + m) arrays per evaluation with scalar bounds, (5 + m) with arrays, plus one x* store per solve.
    # MMA with more than 8 rows runs the TMA-staged evaluation kernel, which keeps reading the arrays.
    per = 8 * _ld(n)
    scalar = not (alg == nl.LD_MMA and m > 8)
    for st, k in ((sa, 3 if scalar else 5), (sb, 5)):
        assert st["dual_operand_bytes"] == per * ((k + m) * st["dual_evals"] + st["dual_solves"])
    # the clamp ran: many coordinates sit exactly on a bound (on the bit pattern of lb: -0.0, not +0.0)
    at_lb = int(np.sum(a["x"].view(np.uint64) == np.float64(lb).view(np.uint64)))
    at_ub = int(np.sum(a["x"] == ub))
    want = 1000 if n > 3 else 1
    assert at_lb + at_ub >= want and (lb != 0.0 or at_lb >= want), (at_lb, at_ub)
