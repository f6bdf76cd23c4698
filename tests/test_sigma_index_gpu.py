"""The sigma index: with uniform bounds, a uniform initial step and 4 rows, the TMA-staged solve kernel of a large shard
reads sigma as a 16-bit index into the palette of values it can reach (sigma_palette.hpp) instead of the fp64 array.
Every other configuration neither keeps nor reads the index.

Every sigma update of end_outer_kernel moves the index through the transition table and compares the palette value with
the fp64 sigma it stores, for every variable, bit for bit; mismatches are counted into nlopt_b200_stats and switch the
run back to the fp64 path; the index before each update is checked the same way, so sigma_0 is checked at the first.
So a run whose stats show a live palette and no mismatches had pal[sidx] == sigma before and after each of its updates.  Each run is compared with the same problem given its bounds as arrays, which never uses the index, and
dual_operand_bytes shows which path ran."""
import numpy as np
import pytest
import torch

import nlopt_b200 as nl
from nlopt_b200 import problems as NP
from test_scalar_bounds_gpu import _ld

pytestmark = pytest.mark.gpu

LB, UB = -2.0, 2.0
N = 3_500_000        # 196 MB of fp64 operands at m = 4: above NB200_SIGMA_INDEX_MIN_MB


def _run(alg, n, m, tma, maxeval, lo, hi, initial_step):
    o = nl.opt(alg, n)
    o.set_lower_bounds(lo); o.set_upper_bounds(hi)
    p = NP.Problem()
    p.rosenbrock_device(o, m)           # the benchmark's c3 problem, device-resident
    o.set_maxeval(maxeval)
    if tma is not None:
        o.set_param("b200_solve_tma", tma)
    if initial_step is not None:
        o.set_initial_step(initial_step)
    x = torch.from_numpy(NP.rosen_x0(n)).cuda()
    o.optimize_device(x.data_ptr())
    torch.cuda.synchronize()
    return dict(x=x.cpu().numpy(), minf=o.last_optimum_value(), ret=o.last_optimize_result(), numevals=o.get_numevals(),
                st=o.get_stats())


def _pair(alg, n, m, tma, maxeval, initial_step=None):
    a, b = (_run(alg, n, m, tma, maxeval, lo, hi, initial_step) for lo, hi in ((LB, UB), (np.full(n, LB), np.full(n, UB))))
    sa, sb = a["st"], b["st"]
    assert a["ret"] == b["ret"] and a["numevals"] == b["numevals"] and a["minf"] == b["minf"]
    assert sa["dual_evals"] == sb["dual_evals"] and sa["dual_solves"] == sb["dual_solves"] > 0
    assert sa["outer_iters"] == sb["outer_iters"]
    assert np.array_equal(a["x"].view(np.uint64), b["x"].view(np.uint64))
    assert sb["sigma_palette"] == 0 and sb["dual_operand_bytes"] == 8 * _ld(n) * ((5 + m) * sb["dual_evals"] + sb["dual_solves"])
    return sa


def _bytes(n, m, evals, solves, sigma_bytes):
    per = 8 * _ld(n)
    return (per * (2 + m) + _ld(n) * sigma_bytes) * evals + per * solves


@pytest.mark.parametrize("alg", [nl.LD_MMA, nl.LD_CCSAQ])
@pytest.mark.parametrize("m", [1, 2, 4])
@pytest.mark.parametrize("tma", [None, 1, 0])
def test_sigma_index_over_40_outer_iterations(built, alg, m, tma):
    """4 rows in the TMA-staged form chosen by the default rule read the index (2 B of sigma per variable); the TMA form
    forced with b200_solve_tma = 1, the register form (0) and 1 or 2 rows read the fp64 sigma and keep no index"""
    n = N
    st = _pair(alg, n, m, tma, maxeval=300)
    assert st["outer_iters"] >= 41, st["outer_iters"]
    assert st["sigma_index_mismatches"] == 0
    used = tma is None and m == 4
    lo = _bytes(n, m, st["dual_evals"], st["dual_solves"], 2 if used else 8)
    if not used:
        assert st["sigma_palette"] == 0 and st["dual_operand_bytes"] == lo
    elif st["sigma_palette"] == 0:
        # the palette passed its cap: at the 79th sigma update for CCSAQ, the 103rd for MMA (test_sigma_palette.py)
        assert st["outer_iters"] >= (79 if alg == nl.LD_CCSAQ else 103), st["outer_iters"]
        hi = _bytes(n, m, st["dual_evals"], st["dual_solves"], 8)
        assert lo < st["dual_operand_bytes"] < hi
    else:
        assert st["dual_operand_bytes"] == lo


@pytest.mark.parametrize("step,uniform", [(0.05, True), (None, False)])
def test_initial_step_decides_the_path(built, step, uniform):
    """a uniform initial step keeps the index; a per-variable one takes the fp64 path from the start"""
    n, m = N, 4
    init = np.full(n, step) if uniform else 0.02 + 0.06 * (np.arange(n) % 5) / 4
    st = _pair(nl.LD_CCSAQ, n, m, None, maxeval=40, initial_step=init)
    assert st["sigma_index_mismatches"] == 0
    if uniform:
        assert st["sigma_palette"] > 0
        assert st["dual_operand_bytes"] == _bytes(n, m, st["dual_evals"], st["dual_solves"], 2)
    else:
        assert st["sigma_palette"] == 0
        assert st["dual_operand_bytes"] == _bytes(n, m, st["dual_evals"], st["dual_solves"], 8)


def test_palette_cap_crossed_mid_run(built):
    """CCSAQ on [-2, 2]: the palette passes its 65535 entries at the 79th sigma update (test_sigma_palette.py).  The run
    reads the index until then and the fp64 sigma after, with the same bits as the array-bounds run."""
    n, m = N, 4
    st = _pair(nl.LD_CCSAQ, n, m, None, maxeval=900)
    assert st["outer_iters"] >= 82, st["outer_iters"]
    assert st["sigma_palette"] == 0 and st["sigma_index_mismatches"] == 0
    lo = _bytes(n, m, st["dual_evals"], st["dual_solves"], 2)
    hi = _bytes(n, m, st["dual_evals"], st["dual_solves"], 8)
    assert lo < st["dual_operand_bytes"] < hi
