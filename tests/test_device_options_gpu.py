"""Per-variable options from device memory on the GPU: nlopt_b200_set_{xtol_abs,x_weights,initial_step}_device and the
torch / __cuda_array_interface__ forms of opt.set_xtol_abs / set_x_weights / set_initial_step.

The setters check the arrays on the device with the host setters' rule, and a run reads them in place; every result is
compared with the same problem given the same options as host arrays: result code, evaluation counts and the bits of f*
and x* must be equal.  Each comparison also shows that the options change the run, so a device path that ignored one
would fail."""
import ctypes as C

import numpy as np
import pytest
import torch

import nlopt_b200 as nl
from nlopt_b200 import _capi
from nlopt_b200 import problems as NP
from test_device_bounds_gpu import ALGS, assert_same_run, cuda, make, passive_box, solve
from test_device_options import MESSAGES, OPTIONS, bits, get, rejects

pytestmark = pytest.mark.gpu


def options(n, seed=11):
    """a non-uniform step with ~5% negative lanes (those take the default sigma), weights in [0, 2] with ~5% zeros, and
    xtol_abs above any first move (so XTOL_REACHED ends an MMA / CCSAQ run after its first outer iteration)"""
    rng = np.random.default_rng(seed)
    dx = rng.uniform(0.02, 0.3, n)
    dx[rng.random(n) < 0.05] *= -1.0
    w = rng.uniform(0.0, 2.0, n)
    w[rng.random(n) < 0.05] = 0.0
    xtol = rng.uniform(0.5, 1.0, n)
    return {"initial_step": dx, "x_weights": w, "xtol_abs": xtol}


def apply(o, opts, device):
    for name, v in opts.items():
        getattr(o, "set_" + name)(cuda(v) if device else v)


def differs(a, b):
    """the runs differ in result code, evaluation counts, or the bits of f* or x*"""
    return (a[0] != b[0] or a[1] != b[1] or bits(a[2]) != bits(b[2]) or not np.array_equal(bits(a[3]), bits(b[3]))
            or a[4]["dual_evals"] != b[4]["dual_evals"] or a[4]["dual_solves"] != b[4]["dual_solves"])


# ---- 1. the setters ------------------------------------------------------------------------------------------------

VALUES = {"x_weights": [np.nan, np.inf, -0.0, 0.0, 5e-324, 2.0],
          "initial_step": [np.nan, np.inf, -np.inf, -0.25, -5e-324, 0.5],
          "xtol_abs": [np.nan, np.inf, -np.inf, -0.0, -1.0, 0.0]}


@pytest.mark.parametrize("name", list(OPTIONS))
def test_device_values_read_back_with_the_host_bits(built, name):
    n = 20011
    rng = np.random.default_rng(5)
    v = np.asarray(VALUES[name])[rng.integers(0, len(VALUES[name]), n)]
    got, want = nl.opt(nl.LD_MMA, n), nl.opt(nl.LD_MMA, n)
    getattr(got, "set_" + name)(cuda(v))
    getattr(want, "set_" + name)(v)
    assert isinstance(get(got, name), np.ndarray)
    assert np.array_equal(bits(get(got, name)), bits(get(want, name)))
    assert np.array_equal(bits(get(got, name)), bits(v))


# a step: "dev" = device setter, "host" = array setter, "host1" = scalar setter, "none" = the array setter with NULL
SEQUENCES = [["dev"], ["host", "dev"], ["dev", "host"], ["dev", "host1"], ["host1", "dev", "dev"], ["dev", "none"],
             ["dev", "none", "dev"], ["dev", "dev", "host"]]


def _apply_seq(o, name, seq, vals, device):
    lib = o._lib
    for k, how in enumerate(seq):
        v = vals[k]
        if how == "host1":
            getattr(o, "set_" + name)(float(v[0]))
        elif how == "none":
            fn = getattr(lib, OPTIONS[name][1])
            assert fn(o._h, None) == nl.SUCCESS
        else:
            getattr(o, "set_" + name)(cuda(v) if device and how == "dev" else v)


@pytest.mark.parametrize("name", list(OPTIONS))
@pytest.mark.parametrize("seq", range(len(SEQUENCES)))
def test_setter_sequences_end_in_the_expected_mode_and_values(built, name, seq):
    """values through the getters, and the mode through the host-to-device bytes of a run (a device-mode option adds
    none, a host array 8 n)"""
    n = 20011
    lb, ub, x0 = passive_box(n)
    vals = [options(n, seed)[name] for seed in range(len(SEQUENCES[seq]))]
    runs, objs = [], []
    for device in (True, False):
        p = NP.Problem()
        o = make("LD_MMA", n, "device", p, maxeval=4)
        o.set_lower_bounds(cuda(lb))
        o.set_upper_bounds(cuda(ub))
        _apply_seq(o, name, SEQUENCES[seq], vals, device)
        runs.append(solve(o, x0, "device"))
        objs.append((o, p))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(*runs)
    assert np.array_equal(bits(get(objs[0][0], name)), bits(get(objs[1][0], name)))
    last = SEQUENCES[seq][-1]
    want_gap = 8 * n if last == "dev" else 0              # the host twin's array goes up; the device one does not
    assert runs[1][4]["h2d_bytes"] - runs[0][4]["h2d_bytes"] == want_gap


def test_a_host_setter_frees_the_device_copy(built):
    n = 25_000_000                                         # 200 MB: well above anything else that moves meanwhile
    o = nl.opt(nl.LD_MMA, n)
    warm = nl.opt(nl.LD_MMA, 4)                            # loads the check kernel's module before the window
    warm.set_initial_step(torch.ones(4, dtype=torch.float64, device="cuda"))
    t = torch.full((n,), 0.5, dtype=torch.float64, device="cuda")
    # torch allocates and releases nothing inside the window: its cache (from earlier tests too) is emptied first, and
    # the source tensor lives through it
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    o.set_initial_step(t)
    free1 = torch.cuda.mem_get_info()[0]
    o.set_initial_step(0.25)
    free2 = torch.cuda.mem_get_info()[0]
    del t
    held, freed = free0 - free1, free2 - free1
    assert held >= 0.75 * 8 * n, (held, freed)
    assert freed >= 0.75 * 8 * n, (held, freed)
    assert np.array_equal(get(o, "initial_step"), np.full(n, 0.25))


# ---- 2. rejections ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [20011, 10_000_000])
@pytest.mark.parametrize("case", ["negative weight", "+0.0 step", "-0.0 step"])
def test_rejected_arrays_keep_the_previous_values(built, n, case):
    name = "x_weights" if case == "negative weight" else "initial_step"
    bad_value = {"negative weight": -1e-300, "+0.0 step": 0.0, "-0.0 step": -0.0}[case]
    o = nl.opt(nl.LD_MMA, n)
    prev = torch.linspace(0.5, 1.5, n, dtype=torch.float64, device="cuda")
    getattr(o, "set_" + name)(prev)
    prev_host = prev.cpu().numpy()
    fn = getattr(o._lib, OPTIONS[name][0])
    for i in (0, 511, 512, 513, n - 1):
        bad = torch.ones(n, dtype=torch.float64, device="cuda")
        bad[i] = bad_value
        torch.cuda.synchronize()
        assert rejects(name, bad.cpu().numpy())
        assert fn(o._h, C.c_void_p(bad.data_ptr())) == nl.INVALID_ARGS, i
        assert o.get_errmsg() == MESSAGES[name]
        assert np.array_equal(bits(get(o, name)), bits(prev_host)), i
        good = torch.full((n,), 0.75, dtype=torch.float64, device="cuda")   # the check rearms: a good call goes through
        torch.cuda.synchronize()
        assert fn(o._h, C.c_void_p(good.data_ptr())) == nl.SUCCESS, i
        getattr(o, "set_" + name)(prev)
    # a rejected device array also keeps a host array
    getattr(o, "set_" + name)(prev_host)
    bad = torch.ones(n, dtype=torch.float64, device="cuda")
    bad[n // 2] = bad_value
    with pytest.raises(ValueError, match=MESSAGES[name]):
        getattr(o, "set_" + name)(bad)
    assert np.array_equal(bits(get(o, name)), bits(prev_host))


# ---- 3. runs, bit for bit against host arrays --------------------------------------------------------------------------

@pytest.mark.parametrize("n", [20011, 250000])
@pytest.mark.parametrize("callbacks", ["host", "device"])
@pytest.mark.parametrize("entry", ["host", "device"])
@pytest.mark.parametrize("alg", list(ALGS))
def test_runs_equal_host_arrays(built, alg, entry, callbacks, n):
    lb, ub, x0 = passive_box(n)
    opts = options(n)
    runs = []
    for how in ("device", "host", "none"):
        p = NP.Problem()
        o = make(alg, n, callbacks, p)
        o.set_lower_bounds(lb)
        o.set_upper_bounds(ub)
        if how != "none":
            apply(o, opts, how == "device")
        runs.append(solve(o, x0, entry))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(runs[0], runs[1])
    assert differs(runs[0], runs[2])
    if alg in ("LD_MMA", "LD_CCSAQ"):
        assert runs[0][0] == nl.XTOL_REACHED


@pytest.mark.parametrize("alg", list(ALGS))
def test_runs_with_device_bounds_equal_host_arrays(built, alg):
    n = 250000
    lb, ub, x0 = passive_box(n)
    opts = options(n, seed=12)
    runs = []
    for device in (True, False):
        p = NP.Problem()
        o = make(alg, n, "device", p)
        o.set_lower_bounds(cuda(lb) if device else lb)
        o.set_upper_bounds(cuda(ub) if device else ub)
        apply(o, opts, device)
        runs.append(solve(o, x0, "device"))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(*runs)


# each stop-test array alone decides the run: xtol_abs above any move stops after the first outer iteration; weights only
# on passive lanes (which never move) make the weighted change zero, so xtol_rel stops it as early
@pytest.mark.parametrize("which", ["xtol_abs", "x_weights"])
@pytest.mark.parametrize("callbacks", ["host", "device"])
@pytest.mark.parametrize("alg", list(ALGS))
def test_each_stop_array_decides_the_run(built, alg, callbacks, which):
    n = 20011
    lb, ub, x0 = passive_box(n)
    if which == "xtol_abs":
        v = np.random.default_rng(2).uniform(1.0, 2.0, n)
    else:
        v = np.where(lb == ub, 1.0, 0.0)
    runs = []
    for how in ("device", "host", "none"):
        p = NP.Problem()
        o = make(alg, n, callbacks, p)
        o.set_lower_bounds(lb)
        o.set_upper_bounds(ub)
        if which == "x_weights":
            o.set_xtol_rel(1e-6)              # below the first move (~1e-4 relative)
        if how != "none":
            getattr(o, "set_" + which)(cuda(v) if how == "device" else v)
        runs.append(solve(o, x0, "device"))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(runs[0], runs[1])
    if alg in ("LD_MMA", "LD_CCSAQ"):
        assert runs[0][0] == nl.XTOL_REACHED and differs(runs[0], runs[2])


# ---- 4. the sigma index ------------------------------------------------------------------------------------------------

def _rosen_run(step):
    n, m = 10_000_000, 4
    o = nl.opt(nl.LD_CCSAQ, n)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_initial_step(step)
    p = NP.Problem()
    p.rosenbrock_device(o, m)
    o.set_maxeval(8)
    r = solve(o, NP.rosen_x0(n), "device")
    assert r[0] > 0, o.get_errmsg()
    return r


def test_uniform_device_step_takes_the_sigma_index(built):
    n = 10_000_000
    dev = _rosen_run(torch.full((n,), 0.3, dtype=torch.float64, device="cuda"))
    one = _rosen_run(0.3)
    assert_same_run(dev, one)
    assert dev[4]["sigma_palette"] > 0 and dev[4]["sigma_palette"] == one[4]["sigma_palette"]
    odd = np.full(n, 0.3)
    odd[n // 2] = np.nextafter(0.3, 1.0)
    dev_odd = _rosen_run(cuda(odd))
    host_odd = _rosen_run(odd)
    assert_same_run(dev_odd, host_odd)
    assert dev_odd[4]["sigma_palette"] == 0 and host_odd[4]["sigma_palette"] == 0


# ---- 5. bytes copied ---------------------------------------------------------------------------------------------------

def test_device_options_save_the_host_copies(built):
    n = 250000
    lb, ub, x0 = passive_box(n)
    opts = options(n)
    runs = []
    for how in ("device", "host", "none"):
        p = NP.Problem()
        o = make("LD_MMA", n, "device", p)
        o.set_lower_bounds(cuda(lb))
        o.set_upper_bounds(cuda(ub))
        if how != "none":
            apply(o, opts, how == "device")
        runs.append(solve(o, x0, "device"))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(runs[0], runs[1])
    assert runs[0][4]["h2d_bytes"] == runs[2][4]["h2d_bytes"]
    assert runs[1][4]["h2d_bytes"] - runs[0][4]["h2d_bytes"] == 3 * 8 * n


# ---- 6. objects and placement ------------------------------------------------------------------------------------------

def test_copy_runs_after_the_original_is_destroyed(built):
    n = 20011
    lb, ub, x0 = passive_box(n)
    opts = options(n)
    p = NP.Problem()
    o = make("LD_CCSAQ", n, "device", p)
    o.set_lower_bounds(lb)
    o.set_upper_bounds(ub)
    apply(o, opts, True)
    lib = o._lib
    h2 = lib.nlopt_copy(o._h)
    assert h2
    want = solve(o, x0, "device")
    assert want[0] > 0
    # changing the copy's arrays leaves the original alone
    other = cuda(np.full(n, 0.125))
    h3 = lib.nlopt_copy(o._h)
    assert lib.nlopt_b200_set_initial_step_device(h3, C.c_void_p(other.data_ptr())) == nl.SUCCESS
    assert lib.nlopt_b200_set_x_weights_device(h3, C.c_void_p(other.data_ptr())) == nl.SUCCESS
    assert np.array_equal(bits(get(o, "initial_step")), bits(opts["initial_step"]))
    assert np.array_equal(bits(get(o, "x_weights")), bits(opts["x_weights"]))
    lib.nlopt_destroy(h3)
    del o
    x = cuda(x0)
    f = C.c_double(0.0)
    assert lib.nlopt_b200_optimize_device(h2, C.c_void_p(x.data_ptr()), C.byref(f)) == want[0]
    torch.cuda.synchronize()
    assert bits(f.value) == bits(want[2]) and np.array_equal(bits(x.cpu().numpy()), bits(want[3]))
    got = np.empty(n)
    assert lib.nlopt_get_xtol_abs(h2, got.ctypes.data_as(_capi.c_double_p)) == nl.SUCCESS
    assert np.array_equal(bits(got), bits(opts["xtol_abs"]))
    lib.nlopt_destroy(h2)


@pytest.mark.parametrize("local", [nl.LD_MMA, nl.LD_CCSAQ])
def test_local_optimizer_with_device_arrays(built, local):
    n = 20011
    lb, ub, x0 = passive_box(n)
    opts = options(n)
    runs = []
    for device in (True, False):
        p = NP.Problem()
        o = nl.opt(nl.AUGLAG, n)
        o.set_maxeval(30)
        lo = nl.opt(local, n)
        lo.set_ftol_rel(1e-8)
        apply(lo, {"initial_step": opts["initial_step"], "xtol_abs": opts["xtol_abs"]}, device)
        o.set_local_optimizer(lo)
        del lo                                             # the outer object holds a copy
        p.simp_device_eq(o, 0x5EED0000, 1e-3, tol=1e-6)
        o.set_lower_bounds(lb)
        o.set_upper_bounds(ub)
        runs.append(solve(o, x0, "device"))
        assert runs[-1][0] > 0, o.get_errmsg()
    assert_same_run(*runs)


def test_preconditioned_ccsaq_reads_device_arrays_through_the_mirror(built):
    def f(x, g):
        if g.size:
            g[:] = 2.0 * (x - 0.3)
        return float((x - 0.3) @ (x - 0.3))

    def pre(x, v, vpre):
        vpre[:] = 2.0 * v

    n = 200
    opts = options(n, seed=4)
    opts["xtol_abs"] = np.full(n, 1e-6)
    opts["xtol_abs"][7] = 1e-5
    runs = []
    for how in ("device", "host", "none"):
        o = nl.opt(nl.LD_CCSAQ, n)
        o.set_precond_min_objective(f, pre)
        o.set_lower_bounds(-1.0)
        o.set_upper_bounds(1.0)
        o.set_maxeval(40)
        if how != "none":
            apply(o, opts, how == "device")
        x = o.optimize(np.full(n, 0.9))
        runs.append((o.last_optimize_result(), o.get_numevals(), o.last_optimum_value(), x, o.get_stats()))
    assert_same_run(runs[0], runs[1])
    assert differs(runs[0], runs[2])


def test_other_device_is_refused(built):
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device visible: a run on a device other than the arrays' is not checked here")
    n = 20011
    lb, ub, x0 = passive_box(n)
    p = NP.Problem()
    o = make("LD_MMA", n, "host", p)
    o.set_lower_bounds(lb)
    o.set_upper_bounds(ub)
    with torch.cuda.device(0):
        o.set_x_weights(cuda(options(n)["x_weights"]))
    with torch.cuda.device(1):
        x = np.array(x0)
        f = C.c_double(0.0)
        assert o._lib.nlopt_optimize(o._h, x.ctypes.data_as(_capi.c_double_p), C.byref(f)) == nl.INVALID_ARGS
        assert "live on CUDA device 0" in o.get_errmsg()
