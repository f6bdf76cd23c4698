"""Box bounds from device memory (nlopt_b200_set_lower_bounds_device / nlopt_b200_set_upper_bounds_device): the argument
checks that need no GPU, the Python layer's validation of __cuda_array_interface__ objects, and a numpy model of the two
rules the device kernels restate -- the setters' snap (options.c:375-377 / :429-431) and the start-point test
(optimize.c:547-551) -- pinned against the host setters and the host check.  tests/test_device_bounds_gpu.py compares the
device kernels with the host paths."""
import ctypes as C

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi

TINY = np.finfo(np.float64).tiny      # DBL_MIN: a nonzero gap below it is subnormal (nlopt_istiny)
SUB = 5e-324

# (lb, ub) pairs: subnormal gaps (snapped), a gap of DBL_MIN (kept), +-0, +-inf, NaN, crossed bounds
PAIRS = [(0.0, SUB), (-SUB, 0.0), (-1e-310, 1e-310), (-1e-308, 1e-308), (0.0, TINY), (1.0, 1.0 + 2.0 ** -52),
         (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0), (-np.inf, np.inf), (np.inf, np.inf), (-np.inf, -np.inf), (np.nan, 1.0),
         (1.0, np.nan), (np.nan, np.nan), (2.0, 1.0), (-np.inf, SUB), (TINY, TINY + SUB), (-TINY, -TINY + SUB),
         (3.0, 3.0)]


def snap_model(v, other, lower):
    """the setter's snap of new values v against the opposite bound: lower -> lb <- ub, else ub <- lb, where
    lb < ub and ub - lb is zero or subnormal"""
    v = np.array(v, dtype=np.float64)
    other = np.asarray(other, dtype=np.float64)
    lo, hi = (v, other) if lower else (other, v)
    with np.errstate(invalid="ignore", over="ignore"):
        shut = (lo < hi) & (np.abs(hi - lo) < TINY)
    v[shut] = other[shut]
    return v


def set_model(lb, ub, new, lower):
    """(lb, ub) after a host or device setter of the lower (or upper) bounds"""
    return (snap_model(new, ub, True), ub) if lower else (lb, snap_model(new, lb, False))


def first_violation(lb, ub, x):
    """(index, message) of the start-point test, or None: the smallest i with lb > ub or x outside [lb, ub]"""
    with np.errstate(invalid="ignore"):
        bad = np.flatnonzero((lb > ub) | (x < lb) | (x > ub))
    if bad.size == 0:
        return None
    i = int(bad[0])
    return i, "bounds %d fail %g <= %g <= %g" % (i, lb[i], x[i], ub[i])


def pair_arrays(seed=0, n=None):
    lb = np.array([p[0] for p in PAIRS])
    ub = np.array([p[1] for p in PAIRS])
    if n is None:
        return lb, ub
    rng = np.random.default_rng(seed)
    k = rng.integers(0, len(PAIRS), n)
    return lb[k], ub[k]


def bits(a):
    return np.asarray(a, dtype=np.float64).view(np.uint64)


def test_entry_points_declared_and_bound(built):
    src = open(_capi.os.path.join(_capi.REPO_DIR, "include", "nlopt_b200.h")).read()
    for name in ("nlopt_b200_set_lower_bounds_device", "nlopt_b200_set_upper_bounds_device"):
        assert name + "(" in src
        assert name in _capi.EXT_SYMBOLS


def test_null_pointer_is_invalid_args(built):
    o = nl.opt(nl.LD_MMA, 4)
    lib = o._lib
    assert lib.nlopt_b200_set_lower_bounds_device(o._h, None) == nl.INVALID_ARGS
    assert lib.nlopt_b200_set_upper_bounds_device(o._h, None) == nl.INVALID_ARGS
    assert lib.nlopt_b200_set_lower_bounds_device(None, None) == nl.INVALID_ARGS


def test_zero_variables_is_a_no_op(built):
    o = nl.opt(nl.LD_MMA, 0)
    buf = (C.c_double * 1)()
    assert o._lib.nlopt_b200_set_lower_bounds_device(o._h, C.addressof(buf)) == nl.SUCCESS
    assert o._lib.nlopt_b200_set_upper_bounds_device(o._h, C.addressof(buf)) == nl.SUCCESS


@pytest.mark.skipif(nl.device_count() > 0, reason="checks the behaviour without a CUDA device")
def test_no_device_fails_and_keeps_the_bounds(built):
    o = nl.opt(nl.LD_MMA, 3)
    o.set_lower_bounds([-1.0, 0.0, 2.0])
    o.set_upper_bounds(5.0)
    buf = (C.c_double * 3)(7.0, 8.0, 9.0)
    for fn in (o._lib.nlopt_b200_set_lower_bounds_device, o._lib.nlopt_b200_set_upper_bounds_device):
        assert fn(o._h, C.addressof(buf)) == nl.FAILURE
        assert "CUDA" in o.get_errmsg()
        assert np.array_equal(o.get_lower_bounds(), [-1.0, 0.0, 2.0]) and np.array_equal(o.get_upper_bounds(), [5.0] * 3)


class _FakeCuda:
    """an object exporting __cuda_array_interface__ only"""

    def __init__(self, ptr, shape, typestr="<f8", strides=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "strides": strides,
                                         "version": 2}


@pytest.mark.parametrize("shape,typestr,strides", [((3,), "<f8", None), ((5,), "<f4", None), ((4,), "<f8", None),
                                                   ((5,), "<f8", (16,)), ((1, 5), "<f8", (8, 8))])
def test_python_rejects_bad_device_arrays(built, shape, typestr, strides):
    o = nl.opt(nl.LD_MMA, 5)
    with pytest.raises(ValueError):
        o.set_lower_bounds(_FakeCuda(0x1000, shape, typestr, strides))
    with pytest.raises(ValueError):
        o.set_upper_bounds(_FakeCuda(0x1000, shape, typestr, strides))


@pytest.mark.skipif(nl.device_count() > 0, reason="checks the behaviour without a CUDA device")
@pytest.mark.parametrize("shape,strides", [((5,), None), ((5,), (8,)), ((1, 5), (40, 8))])
def test_python_passes_good_device_arrays_to_the_library(built, shape, strides):
    o = nl.opt(nl.LD_MMA, 5)
    buf = (C.c_double * 5)()
    with pytest.raises(RuntimeError, match="CUDA"):
        o.set_lower_bounds(_FakeCuda(C.addressof(buf), shape, strides=strides))
    assert np.array_equal(o.get_lower_bounds(), [-np.inf] * 5)


@pytest.mark.parametrize("lower_first", [True, False])
@pytest.mark.parametrize("n", [len(PAIRS), 997])
def test_snap_model_matches_the_host_setters(built, lower_first, n):
    lb, ub = pair_arrays(1, None if n == len(PAIRS) else n)
    o = nl.opt(nl.LD_MMA, lb.size)
    cur = (np.full(lb.size, -np.inf), np.full(lb.size, np.inf))
    for lower in ((True, False) if lower_first else (False, True)):
        (o.set_lower_bounds if lower else o.set_upper_bounds)(lb if lower else ub)
        cur = set_model(*cur, lb if lower else ub, lower)
        assert np.array_equal(bits(o.get_lower_bounds()), bits(cur[0]))
        assert np.array_equal(bits(o.get_upper_bounds()), bits(cur[1]))
    if n == len(PAIRS):                          # the first pair's subnormal gap was shut, in either order
        assert bits(cur[0])[0] == bits(cur[1])[0]


def _host_check(lb, ub, x):
    o = nl.opt(nl.LD_MMA, lb.size)
    o.set_lower_bounds(lb)
    o.set_upper_bounds(ub)
    o.set_min_objective(lambda x, g: 0.0)
    with pytest.raises(ValueError) as e:
        o.optimize(x)
    assert o.last_optimize_result() == nl.INVALID_ARGS and o.get_numevals() == 0
    return o.get_lower_bounds(), o.get_upper_bounds(), str(e.value)


@pytest.mark.parametrize("case", range(6))
def test_first_violation_model_matches_the_host_check(built, case):
    n = 4001
    rng = np.random.default_rng(case)
    lb, ub = np.full(n, -1.0), np.full(n, 1.0)
    x = rng.uniform(-0.5, 0.5, n)
    bad = np.sort(rng.choice(n, 3, replace=False))
    if case == 0:
        x[bad] = [2.0, -3.0, 1.5]               # outside, several indices
    elif case == 1:
        lb[bad], ub[bad] = 0.5, 0.25            # crossed bounds
    elif case == 2:
        x[bad] = np.nan                         # NaN passes ...
        x[bad[2]] = np.inf                      # ... inf does not
    elif case == 3:
        lb[bad] = np.nan                        # NaN bounds pass as in the reference
        ub[bad[1]] = -np.inf
    elif case == 4:
        lb[bad], ub[bad], x[bad] = -0.0, 0.0, 0.0
        x[bad[2]] = -SUB
    else:
        lb[bad], ub[bad] = -SUB, SUB
        x[bad] = 2 * SUB
    lbs, ubs, msg = _host_check(lb, ub, x)
    want = first_violation(lbs, ubs, x)
    assert want is not None and msg == want[1]
