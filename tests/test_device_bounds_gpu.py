"""Box bounds from device memory on the GPU: nlopt_b200_set_lower_bounds_device / nlopt_b200_set_upper_bounds_device and
the torch / __cuda_array_interface__ forms of opt.set_lower_bounds / set_upper_bounds.

Each device-bounds run is compared with the same problem given the same bounds as host arrays: the device path copies the
arrays device to device, snaps them with the setters' rule and checks the start point on the device, so the result code,
the evaluation counts and the bits of f* and x* must be equal.  Bitwise uniform arrays take the scalar-bounds kernels (and
the sigma index) exactly as nlopt_set_*_bounds1 does."""
import ctypes as C

import numpy as np
import pytest
import torch

import nlopt_b200 as nl
from nlopt_b200 import _capi
from nlopt_b200 import problems as NP
from test_device_bounds import PAIRS, bits, first_violation, pair_arrays, set_model
from test_scalar_bounds_gpu import _ld

pytestmark = pytest.mark.gpu

SEED, EPS = 0x5EED0000, 1e-3

# algorithm, local optimiser, volume constraint as an equality
ALGS = {"LD_MMA": (nl.LD_MMA, None, False), "LD_CCSAQ": (nl.LD_CCSAQ, None, False),
        "LD_AUGLAG": (nl.LD_AUGLAG, None, False), "LD_AUGLAG_EQ": (nl.LD_AUGLAG_EQ, None, True),
        "AUGLAG_CCSAQ": (nl.AUGLAG, nl.LD_CCSAQ, True)}


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def passive_box(n, seed=3):
    """SIMP box [1e-3, 1] with ~3% passive elements (lb == ub, solid 1 or void 1e-3), and a start point inside"""
    rng = np.random.default_rng(seed)
    lb, ub, x0 = np.full(n, 1e-3), np.full(n, 1.0), np.full(n, 0.4)
    k = rng.choice(n, n // 33, replace=False)
    v = np.where(rng.random(k.size) < 0.5, 1.0, 1e-3)
    lb[k] = ub[k] = x0[k] = v
    return lb, ub, x0


def make(alg_key, n, callbacks, p, maxeval=30):
    alg, local, eq = ALGS[alg_key]
    o = nl.opt(alg, n)
    o.set_maxeval(maxeval)
    if local is not None:
        lo = nl.opt(local, n)
        lo.set_ftol_rel(1e-8)
        o.set_local_optimizer(lo)
    if callbacks == "host":
        (p.simp_host_eq if eq else p.simp_host)(o, SEED, EPS, tol=1e-6)
    else:
        (p.simp_device_eq if eq else p.simp_device)(o, SEED, EPS, tol=1e-6)
    return o


def solve(o, x0, entry):
    """(ret, numevals, opt_f, x, stats) without raising on negative results"""
    f = C.c_double(0.0)
    if entry == "host":
        x = np.array(x0, dtype=np.float64)
        ret = o._lib.nlopt_optimize(o._h, x.ctypes.data_as(_capi.c_double_p), C.byref(f))
    else:
        xd = cuda(x0)
        ret = o._lib.nlopt_b200_optimize_device(o._h, C.c_void_p(xd.data_ptr()), C.byref(f))
        torch.cuda.synchronize()
        x = xd.cpu().numpy()
    return ret, o.get_numevals(), f.value, x, o.get_stats()


def assert_same_run(a, b):
    assert a[0] == b[0] and a[1] == b[1], (a[:2], b[:2])
    assert a[4]["dual_evals"] == b[4]["dual_evals"] and a[4]["dual_solves"] == b[4]["dual_solves"]
    assert bits(a[2]) == bits(b[2]), (a[2], b[2])
    assert np.array_equal(bits(a[3]), bits(b[3])), np.flatnonzero(bits(a[3]) != bits(b[3]))[:8]


# ---- 1. the setters ------------------------------------------------------------------------------------------------

# a step: (which bound, how): "dev" = device setter, "host" = array setter, "host1" = scalar setter, "one" = set_*_bound(i)
SEQUENCES = [[("lb", "dev"), ("ub", "dev")], [("ub", "dev"), ("lb", "dev")], [("lb", "host"), ("ub", "dev")],
             [("ub", "host"), ("lb", "dev")], [("lb", "dev"), ("ub", "host")], [("ub", "dev"), ("lb", "host")],
             [("lb", "dev"), ("ub", "host1")], [("lb", "host1"), ("ub", "dev"), ("lb", "dev")],
             [("lb", "dev"), ("ub", "dev"), ("lb", "one")], [("ub", "dev"), ("lb", "dev"), ("ub", "dev")]]


def _apply(o, seq, lb, ub, device):
    for which, how in seq:
        v = lb if which == "lb" else ub
        if how == "one":
            (o.set_lower_bound if which == "lb" else o.set_upper_bound)(2, float(v[2]) * 0.5)
        elif how == "host1":
            (o.set_lower_bounds if which == "lb" else o.set_upper_bounds)(float(v[0]))
        else:
            arg = cuda(v) if device and how == "dev" else v
            (o.set_lower_bounds if which == "lb" else o.set_upper_bounds)(arg)


@pytest.mark.parametrize("n", [len(PAIRS), 100003])
@pytest.mark.parametrize("seq", range(len(SEQUENCES)))
def test_device_setters_equal_host_setters(built, n, seq):
    lb, ub = pair_arrays(7, None if n == len(PAIRS) else n)
    got, want = nl.opt(nl.LD_MMA, lb.size), nl.opt(nl.LD_MMA, lb.size)
    _apply(got, SEQUENCES[seq], lb, ub, True)
    _apply(want, SEQUENCES[seq], lb, ub, False)
    for a, b in ((got.get_lower_bounds(), want.get_lower_bounds()), (got.get_upper_bounds(), want.get_upper_bounds())):
        assert isinstance(a, np.ndarray)
        assert np.array_equal(bits(a), bits(b)), np.flatnonzero(bits(a) != bits(b))[:8]
    if all(how in ("dev", "host") for _, how in SEQUENCES[seq]):      # and the numpy model of the snap
        cur = (np.full(lb.size, -np.inf), np.full(lb.size, np.inf))
        for which, _ in SEQUENCES[seq]:
            cur = set_model(*cur, lb if which == "lb" else ub, which == "lb")
        assert np.array_equal(bits(got.get_lower_bounds()), bits(cur[0]))
        assert np.array_equal(bits(got.get_upper_bounds()), bits(cur[1]))


def test_host_readers_see_the_device_values(built):
    n = 1000
    lb, ub, x0 = passive_box(n)
    o = nl.opt(nl.LD_MMA, n)
    o.set_lower_bounds(cuda(lb))
    o.set_upper_bounds(cuda(ub))
    h = nl.opt(nl.LD_MMA, n)
    h.set_lower_bounds(lb)
    h.set_upper_bounds(ub)
    assert np.array_equal(bits(o.get_initial_step(x0)), bits(h.get_initial_step(x0)))
    assert np.array_equal(bits(o.get_lower_bounds()), bits(lb)) and np.array_equal(bits(o.get_upper_bounds()), bits(ub))
    o.set_local_optimizer(nl.opt(nl.LD_MMA, n))        # reads the device values through the same download


def test_copy_runs_after_the_original_is_destroyed(built):
    n = 20011
    lb, ub, x0 = passive_box(n)
    p = NP.Problem()
    o = make("LD_MMA", n, "device", p)
    o.set_lower_bounds(cuda(lb))
    o.set_upper_bounds(cuda(ub))
    lib = o._lib
    h2 = lib.nlopt_copy(o._h)
    assert h2
    want = solve(o, x0, "device")
    assert want[0] > 0
    del o
    x = cuda(x0)
    f = C.c_double(0.0)
    assert lib.nlopt_b200_optimize_device(h2, C.c_void_p(x.data_ptr()), C.byref(f)) == want[0]
    torch.cuda.synchronize()
    assert bits(f.value) == bits(want[2]) and np.array_equal(bits(x.cpu().numpy()), bits(want[3]))
    got = np.empty(n)
    assert lib.nlopt_get_upper_bounds(h2, got.ctypes.data_as(_capi.c_double_p)) == nl.SUCCESS
    assert np.array_equal(bits(got), bits(ub))
    lib.nlopt_destroy(h2)


# ---- 3. runs with passive elements -----------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [20011, 250000])
@pytest.mark.parametrize("callbacks", ["host", "device"])
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("alg", list(ALGS))
def test_passive_elements_equal_host_arrays(built, alg, entry, callbacks, n):
    lb, ub, x0 = passive_box(n)
    runs = []
    for device in (True, False):
        p = NP.Problem()
        o = make(alg, n, callbacks, p)
        o.set_lower_bounds(cuda(lb) if device else lb)
        o.set_upper_bounds(cuda(ub) if device else ub)
        runs.append(solve(o, x0, entry))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(*runs)


# ---- 4. / 5. uniform arrays and the bit contract --------------------------------------------------------------------

def test_uniform_device_arrays_take_the_scalar_bounds_and_sigma_index(built):
    """BASELINE config 3 (CCSAQ, m = 4, n = 1e7): uniform arrays through the device setters run as *_bounds1"""
    n, m = 10_000_000, 4
    runs = []
    for device in (True, False):
        o = nl.opt(nl.LD_CCSAQ, n)
        if device:
            o.set_lower_bounds(torch.full((n,), -2.0, dtype=torch.float64, device="cuda"))
            o.set_upper_bounds(torch.full((n,), 2.0, dtype=torch.float64, device="cuda"))
        else:
            o.set_lower_bounds(-2.0)
            o.set_upper_bounds(2.0)
        p = NP.Problem()
        p.rosenbrock_device(o, m)
        o.set_maxeval(8)
        runs.append(solve(o, NP.rosen_x0(n), "device"))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(*runs)
    a, b = runs[0][4], runs[1][4]
    assert a["sigma_palette"] > 0 and a["sigma_palette"] == b["sigma_palette"]
    assert a["dual_operand_bytes"] == b["dual_operand_bytes"]


@pytest.mark.parametrize("entry", ["host", "device"])
def test_one_negative_zero_lane_keeps_the_arrays(built, entry):
    n = 20011
    lb, ub = np.full(n, 0.0), np.full(n, 1.0)
    lb[4321] = -0.0
    x0 = np.full(n, 0.4)
    runs = []
    for how in ("device", "host", "uniform"):
        p = NP.Problem()
        o = make("LD_MMA", n, "device", p)
        lo = lb if how != "uniform" else np.full(n, 0.0)
        o.set_lower_bounds(cuda(lo) if how != "host" else lo)
        o.set_upper_bounds(cuda(ub) if how != "host" else ub)
        runs.append(solve(o, x0, entry))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(runs[0], runs[1])
    per = 8 * _ld(n)
    for r, k in ((runs[0], 5), (runs[1], 5), (runs[2], 3)):     # arrays: 5 + m operand arrays, scalar bounds: 3 + m
        st = r[4]
        assert st["dual_operand_bytes"] == per * ((k + 1) * st["dual_evals"] + st["dual_solves"]), (k, st)


# ---- 6. a bad start --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", ["outside", "crossed", "subnormal"])
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("alg", ["LD_MMA", "LD_AUGLAG"])
def test_bad_start_gives_the_host_message(built, alg, entry, case):
    n = 250000
    lb, ub, x0 = passive_box(n)
    if case == "outside":
        x0[[90001, 1234, 200000]] = [2.0, 1e-4, -1.0]
    elif case == "crossed":
        lb[[777, 150000]], ub[[777, 150000]] = 0.9, 0.8
    else:
        lb[:] = 0.0
        x0[60000] = -5e-324
    want = first_violation(lb, ub, x0)
    msgs = []
    for device in (True, False):
        p = NP.Problem()
        o = make(alg, n, "device", p)
        o.set_lower_bounds(cuda(lb) if device else lb)
        o.set_upper_bounds(cuda(ub) if device else ub)
        r = solve(o, x0, entry if device else "host")
        assert r[0] == nl.INVALID_ARGS and r[1] == 0
        msgs.append(o.get_errmsg())
    assert msgs[0] == msgs[1] == want[1]


# ---- 7. bytes copied -------------------------------------------------------------------------------------------------

def test_device_bounds_save_the_host_copies(built):
    n = 250000
    lb, ub, x0 = passive_box(n)
    runs = []
    for device in (True, False):
        p = NP.Problem()
        o = make("LD_MMA", n, "device", p)
        o.set_lower_bounds(cuda(lb) if device else lb)
        o.set_upper_bounds(cuda(ub) if device else ub)
        runs.append(solve(o, x0, "device"))
    assert_same_run(*runs)
    assert runs[1][4]["h2d_bytes"] - runs[0][4]["h2d_bytes"] == 2 * 8 * n


# ---- 8. Python ---------------------------------------------------------------------------------------------------------

def test_bad_tensors_raise_value_error(built):
    n = 1000
    o = nl.opt(nl.LD_MMA, n)
    for t in (torch.zeros(n, dtype=torch.float32, device="cuda"), torch.zeros(n + 1, dtype=torch.float64, device="cuda"),
              torch.zeros(2 * n, dtype=torch.float64, device="cuda")[::2], torch.zeros(n, 2, dtype=torch.float64, device="cuda").t()):
        with pytest.raises(ValueError):
            o.set_lower_bounds(t)
        with pytest.raises(ValueError):
            o.set_upper_bounds(t)
    assert np.array_equal(o.get_lower_bounds(), np.full(n, -np.inf))


def test_preconditioned_ccsaq_refuses_device_bounds(built):
    def f(x, g):
        if g.size:
            g[:] = 2.0 * x
        return float(x @ x)

    def pre(x, v, vpre):
        vpre[:] = 2.0 * v

    n = 100
    o = nl.opt(nl.LD_CCSAQ, n)
    o.set_precond_min_objective(f, pre)
    o.set_lower_bounds(cuda(np.full(n, -1.0)))
    o.set_upper_bounds(cuda(np.full(n, 1.0)))
    with pytest.raises(ValueError, match="host bounds"):
        o.optimize(np.full(n, 0.5))
    o.set_lower_bounds(-1.0)                  # back to host bounds: the run goes through
    o.set_maxeval(5)
    o.optimize(np.full(n, 0.5))
    assert o.last_optimize_result() > 0
