"""Uniform box bounds in the TMA-staged persistent solve kernel (dual_solve_tma_kernel<..., SB = true>): its stages hold
3 + m arrays and lb / ub arrive as two scalars.  Same check as test_scalar_bounds_gpu.py: the same bits as the same
bounds passed as arrays (the 5 + m array stages), and nlopt_b200_stats::dual_operand_bytes shows which path ran."""
import numpy as np
import pytest

import nlopt_b200 as nl
import problems as P
from test_gpu_parity import _run
from test_scalar_bounds_gpu import _ld

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("alg", [nl.LD_MMA, nl.LD_CCSAQ])
@pytest.mark.parametrize("n,m", [(3, 1), (100001, 2), (300000, 3), (300000, 4), (300000, 8), (1500000, 1), (1500000, 4)])
@pytest.mark.parametrize("lb", [-0.3, -0.0])
def test_tma_solve_scalar_bounds_equal_array_bounds(built, alg, n, m, lb):
    """m = 1, 2, 4 run the TMA-staged form (every row active); m = 3 and 8 fall back to the register form."""
    ub = 0.3
    f, _ = P.quad_problem(n)
    cons = [P.lin_constraint(k, n) for k in range(m)]
    x0 = np.full(n, 0.1)
    runs = [_run(alg, n, f, cons, [1e-8] * m, lo, hi, x0, maxeval=12, b200_solve_tma=1)
            for lo, hi in ((lb, ub), (np.full(n, lb), np.full(n, ub)))]
    a, b = runs
    sa, sb = a["opt"].get_stats(), b["opt"].get_stats()
    assert a["ret"] == b["ret"] and a["numevals"] == b["numevals"] and a["minf"] == b["minf"]
    assert sa["dual_evals"] == sb["dual_evals"] and sa["dual_solves"] == sb["dual_solves"]
    assert sa["dual_solves"] > 0
    assert np.array_equal(a["x"].view(np.uint64), b["x"].view(np.uint64))
    per = 8 * _ld(n)
    for st, k in ((sa, 3), (sb, 5)):
        assert st["dual_operand_bytes"] == per * ((k + m) * st["dual_evals"] + st["dual_solves"])
    at_lb = int(np.sum(a["x"].view(np.uint64) == np.float64(lb).view(np.uint64)))
    at_ub = int(np.sum(a["x"] == ub))
    want = 1000 if n > 3 else 1
    assert at_lb + at_ub >= want and (lb != 0.0 or at_lb >= want), (at_lb, at_ub)
