"""Per-variable options from device memory (nlopt_b200_set_xtol_abs_device, nlopt_b200_set_x_weights_device,
nlopt_b200_set_initial_step_device): the argument checks that need no GPU, the Python layer's validation of
__cuda_array_interface__ objects, and a numpy model of what option_check_kernel restates -- the host setters' rules
(a negative weight, a zero step) and bitwise uniformity -- pinned against the host setters.
tests/test_device_options_gpu.py compares the device kernel and runs with the host paths."""
import ctypes as C

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi
from test_device_bounds import _FakeCuda

SUB = 5e-324
TINY = np.finfo(np.float64).tiny

# option name -> (device entry point, host array setter, host scalar setter, getter)
OPTIONS = {
    "xtol_abs": ("nlopt_b200_set_xtol_abs_device", "nlopt_set_xtol_abs", "nlopt_set_xtol_abs1", "get_xtol_abs"),
    "x_weights": ("nlopt_b200_set_x_weights_device", "nlopt_set_x_weights", "nlopt_set_x_weights1", "get_x_weights"),
    "initial_step": ("nlopt_b200_set_initial_step_device", "nlopt_set_initial_step", "nlopt_set_initial_step1",
                     "get_initial_step"),
}
MESSAGES = {"x_weights": "invalid negative weight", "initial_step": "zero step size"}

# the values the rules and the bit test must tell apart
SPECIAL = [0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, SUB, -SUB, TINY, -TINY, 1.0, -1.0, 1e308, -1e-300]


def bits(a):
    return np.asarray(a, dtype=np.float64).view(np.uint64)


def rejects(name, v):
    """the host setter's rule (options.c): a negative weight, or a zero step (+0.0 or -0.0); NaN passes both"""
    v = np.asarray(v, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        if name == "x_weights":
            return bool(np.any(v < 0))
        if name == "initial_step":
            return bool(np.any(v == 0))
    return False


def uniform(v):
    """every lane has the bits of lane 0 (the sigma index's condition: -0.0 next to +0.0 is not uniform)"""
    b = bits(v)
    return bool(np.all(b == b[0]))


def get(o, name):
    if name == "initial_step":
        return o.get_initial_step(np.zeros(o._n))
    return getattr(o, OPTIONS[name][3])()


def host_set(o, name, v):
    """the host array setter's return code and message"""
    a = np.ascontiguousarray(v, dtype=np.float64)
    r = getattr(o._lib, OPTIONS[name][1])(o._h, a.ctypes.data_as(_capi.c_double_p))
    return r, o.get_errmsg()


def test_entry_points_declared_and_bound(built):
    src = open(_capi.os.path.join(_capi.REPO_DIR, "include", "nlopt_b200.h")).read()
    for dev, _, _, _ in OPTIONS.values():
        assert dev + "(" in src
        assert dev in _capi.EXT_SYMBOLS


@pytest.mark.parametrize("name", list(OPTIONS))
def test_null_pointer_is_invalid_args(built, name):
    o = nl.opt(nl.LD_MMA, 4)
    fn = getattr(o._lib, OPTIONS[name][0])
    assert fn(o._h, None) == nl.INVALID_ARGS
    assert fn(None, None) == nl.INVALID_ARGS


@pytest.mark.parametrize("name", list(OPTIONS))
def test_zero_variables_is_a_no_op(built, name):
    o = nl.opt(nl.LD_MMA, 0)
    buf = (C.c_double * 1)(0.0)                # a zero step or a negative weight would be refused if it were read
    assert getattr(o._lib, OPTIONS[name][0])(o._h, C.addressof(buf)) == nl.SUCCESS


@pytest.mark.skipif(nl.device_count() > 0, reason="checks the behaviour without a CUDA device")
@pytest.mark.parametrize("name", list(OPTIONS))
def test_no_device_fails_and_keeps_the_option(built, name):
    o = nl.opt(nl.LD_MMA, 3)
    prev = np.array([0.5, 2.0, 3.0])
    getattr(o, "set_" + name)(prev)
    buf = (C.c_double * 3)(7.0, 8.0, 9.0)
    assert getattr(o._lib, OPTIONS[name][0])(o._h, C.addressof(buf)) == nl.FAILURE
    assert "no usable CUDA device" in o.get_errmsg()
    assert np.array_equal(bits(get(o, name)), bits(prev))


@pytest.mark.parametrize("name", list(OPTIONS))
@pytest.mark.parametrize("shape,typestr,strides", [((3,), "<f8", None), ((5,), "<f4", None), ((4,), "<f8", None),
                                                   ((5,), "<f8", (16,)), ((1, 5), "<f8", (8, 8))])
def test_python_rejects_bad_device_arrays(built, name, shape, typestr, strides):
    o = nl.opt(nl.LD_MMA, 5)
    with pytest.raises(ValueError, match="contiguous float64"):
        getattr(o, "set_" + name)(_FakeCuda(0x1000, shape, typestr, strides))


@pytest.mark.skipif(nl.device_count() > 0, reason="checks the behaviour without a CUDA device")
@pytest.mark.parametrize("name", list(OPTIONS))
@pytest.mark.parametrize("shape,strides", [((5,), None), ((5,), (8,)), ((1, 5), (40, 8))])
def test_python_passes_good_device_arrays_to_the_library(built, name, shape, strides):
    o = nl.opt(nl.LD_MMA, 5)
    prev = np.full(5, 0.25)
    getattr(o, "set_" + name)(prev)
    buf = (C.c_double * 5)()
    with pytest.raises(RuntimeError, match="CUDA"):
        getattr(o, "set_" + name)(_FakeCuda(C.addressof(buf), shape, strides=strides))
    assert np.array_equal(get(o, name), prev)


def special_arrays(n):
    """(label, array): each special value alone, and as the one odd lane at the first, a middle and the last position of
    an array of ones"""
    out = [(f"all {tag(v)}", np.full(n, v)) for v in SPECIAL]
    for v in SPECIAL:
        for i in (0, n // 2, n - 1):
            a = np.ones(n)
            a[i] = v
            out.append((f"{tag(v)} at {i}", a))
    return out


def tag(v):
    return f"{v!r}/{int(bits(v)):#x}"


@pytest.mark.parametrize("name", ["x_weights", "initial_step", "xtol_abs"])
def test_rule_model_matches_the_host_setters(built, name):
    n = 1031
    for label, a in special_arrays(n):
        o = nl.opt(nl.LD_MMA, n)
        r, msg = host_set(o, name, a)
        if rejects(name, a):
            assert r == nl.INVALID_ARGS and msg == MESSAGES[name], label
        else:
            assert r == nl.SUCCESS, (label, msg)
            assert np.array_equal(bits(get(o, name)), bits(a)), label


@pytest.mark.parametrize("name", ["x_weights", "initial_step"])
def test_a_rejected_host_array_keeps_the_previous_one(built, name):
    n = 64
    o = nl.opt(nl.LD_MMA, n)
    prev = np.linspace(0.5, 1.5, n)
    getattr(o, "set_" + name)(prev)
    bad = np.ones(n)
    bad[n - 1] = -1.0 if name == "x_weights" else -0.0
    assert host_set(o, name, bad)[0] == nl.INVALID_ARGS
    assert np.array_equal(bits(get(o, name)), bits(prev))


def test_uniformity_model():
    n = 1031
    verdicts = {label: uniform(a) for label, a in special_arrays(n)}
    for v in SPECIAL:
        assert verdicts[f"all {tag(v)}"]                           # one value, one bit pattern (NaN included)
        assert verdicts[f"{tag(v)} at 0"] == (v == 1.0)
    assert not uniform(np.array([0.0, -0.0])) and not uniform(np.array([-0.0, 0.0]))
    assert uniform(np.array([np.nan, np.nan])) and not uniform(np.array([np.nan, -np.nan]))
    one_ulp = np.full(n, 0.2)
    one_ulp[n // 2] = np.nextafter(0.2, 1.0)
    assert not uniform(one_ulp) and one_ulp[n // 2] == pytest.approx(0.2)
