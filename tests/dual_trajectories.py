"""The catalogue of dual-optimiser trajectories: the m-dimensional problems that the nested MMA of the CCSA solvers
(mma.c:248-288 with optimize.c:818-826) is run on, for tests/golden/make_dual_trajectories.py, tests/test_dual_machine.py
and tests/test_dual_machine_gpu.py.

The dual optimiser sees F only through its values and gradients.  So the reference's trajectory -- every point y_k it
evaluates, with F(y_k) and grad F(y_k) -- can be recorded once and then fed to the library's machines, which must ask
for exactly the same points and end with the same result.  tests/golden/reference_dual_trajectories.json stores the
reference's result and a fingerprint of its trajectory; the tests regenerate the trajectory with the oracle port
(oracle/ccsa_port.c) and check it against that fingerprint.

Every F gives the same bits on every machine: either the port's own dual function on a seeded synthetic instance, or a
rational function written with + - * / sqrt abs and comparisons, evaluated in a fixed order on Python floats (one IEEE
operation each).  Some are stateful (they depend on how often they were called): the optimiser cannot tell.
"""
import ctypes as C
import hashlib

import numpy as np

import oracle_bindings as ob
import synth

INF = float("inf")
NAN = float("nan")
# the reference's defaults for the dual optimiser (optimize.c:822-826)
DEFAULT_STOP = dict(ftol_rel=1e-14, ftol_abs=0.0, xtol_rel=0.0, xtol_abs=0.0, maxeval=100000)
RET_INVALID = -2


def _case(name, m, kind, stop=None, **kw):
    c = dict(name=name, m=m, kind=kind, stop=dict(DEFAULT_STOP, **(stop or {})))
    c.update(kw)
    return c


def catalogue():
    """the cases, in a fixed order; every field is a plain JSON value"""
    cases = []
    # ---- real duals: the MMA and CCSAQ dual functions of seeded instances --------------------------------------------
    for variant in ("mma", "ccsaq"):
        for m in (1, 2, 3, 4, 5, 7, 8, 12, 16, 17, 40):
            for c0 in ("feasible", "infeasible"):
                cases.append(_case(f"{variant}-m{m}-{c0}", m, variant, n=48 + m, seed=2000 + m, c0=c0, rho=1.0,
                                   warm="zero"))
        for m in (3, 8, 16):
            cases.append(_case(f"{variant}-m{m}-rho-floor", m, variant, n=64, seed=2100 + m, c0="feasible", rho=1e-5,
                               warm="zero"))
            cases.append(_case(f"{variant}-m{m}-rho-large", m, variant, n=64, seed=2200 + m, c0="infeasible", rho=1e3,
                               warm="zero"))
            for c0 in ("feasible", "infeasible"):
                cases.append(_case(f"{variant}-m{m}-{c0}-warm", m, variant, n=64, seed=2300 + m, c0=c0, rho=1.0,
                                   warm="prev"))
        for m in (2, 5, 13):
            rules = [("ftol_rel", dict(ftol_rel=1e-6)), ("ftol_abs", dict(ftol_rel=0.0, ftol_abs=1e-9)),
                     ("xtol_rel", dict(ftol_rel=0.0, xtol_rel=1e-5)), ("xtol_abs", dict(ftol_rel=0.0, xtol_abs=1e-7)),
                     ("maxeval1", dict(maxeval=1)), ("maxeval2", dict(maxeval=2)), ("maxeval7", dict(maxeval=7))]
            for rule, stop in rules:
                for c0 in ("feasible", "infeasible"):
                    cases.append(_case(f"{variant}-m{m}-{c0}-{rule}", m, variant, stop=stop, n=40, seed=2400 + m, c0=c0,
                                       rho=1.0, warm="zero"))
    # an MMA row switched off by a NaN constraint value (mma.c:75-78)
    for m in (2, 4, 9):
        for c0 in ("nanrow", "nanrow-infeasible"):
            cases.append(_case(f"mma-m{m}-{c0}", m, "mma", n=56, seed=2500 + m, c0=c0, rho=1.0, warm="zero"))
    # ---- edges: closed-form functions --------------------------------------------------------------------------------
    box = dict(lo=0.0, hi=1.0)
    for m in (1, 3):
        cases.append(_case(f"flat-m{m}", m, "flat", stop=dict(maxeval=50), lo=0.0, hi=INF, y0=0.5))
        cases.append(_case(f"flat-m{m}-noftol", m, "flat", stop=dict(ftol_rel=0.0, maxeval=30), lo=0.0, hi=INF, y0=0.5))
        cases.append(_case(f"flat-m{m}-xtol_abs", m, "flat", stop=dict(xtol_abs=1e-7, maxeval=30), lo=0.0, hi=INF,
                           y0=0.5))
    for m in (1, 2, 6):
        cases.append(_case(f"linear-m{m}", m, "linear", stop=dict(maxeval=400), lo=0.0, hi=1e40, y0=0.0))
    for m in (1, 3, 5):
        cases.append(_case(f"box-approach-m{m}", m, "approach", stop=dict(ftol_rel=0.0, maxeval=200), y0=0.0, **box))
        cases.append(_case(f"box-far-m{m}", m, "quadratic", stop=dict(maxeval=200), y0=0.5, target=3.0, **box))
        cases.append(_case(f"box-below-m{m}", m, "quadratic", stop=dict(maxeval=200), y0=0.5, target=-2.0, **box))
        cases.append(_case(f"box-oscillate-m{m}", m, "oscillate", stop=dict(ftol_rel=0.0, maxeval=200), y0=0.1,
                           **box))
        cases.append(_case(f"oscillate-m{m}", m, "oscillate", stop=dict(ftol_rel=0.0, maxeval=150), lo=0.0, hi=INF,
                           y0=0.1))
        cases.append(_case(f"quadratic-m{m}", m, "quadratic", stop=dict(maxeval=300), lo=0.0, hi=INF, y0=0.0,
                           target=2.5))
        cases.append(_case(f"box-switch-m{m}", m, "switch", stop=dict(ftol_rel=0.0, maxeval=300), y0=0.9, **box))
        # a warm start above the minimiser: the first moves go down towards 0.3, not away from 0
        cases.append(_case(f"warm-quadratic-m{m}", m, "quadratic", stop=dict(maxeval=300), lo=0.0, hi=INF, y0=2.0,
                           target=0.3))
    for m in (1, 4):
        for k in (0, 1, 5):
            cases.append(_case(f"nan-after{k}-m{m}", m, "nan_after", stop=dict(maxeval=40), lo=0.0, hi=INF, y0=0.0,
                               k=k))
        for sign in ("+", "-"):
            for k in (0, 3):
                cases.append(_case(f"inf{sign}-after{k}-m{m}", m, "inf_after", stop=dict(maxeval=30), lo=0.0, hi=INF,
                                   y0=0.0, k=k, sign=sign))
        cases.append(_case(f"nan-grad-m{m}", m, "nan_grad", stop=dict(maxeval=40), lo=0.0, hi=INF, y0=0.0, k=3))
        cases.append(_case(f"huge-grad-m{m}", m, "scaled", stop=dict(maxeval=60), lo=0.0, hi=1e40, y0=0.0,
                           scale=1e300))
        cases.append(_case(f"tiny-grad-m{m}", m, "scaled", stop=dict(maxeval=60), lo=0.0, hi=INF, y0=0.0,
                           scale=5e-320))
        # wval = 0 at the rho raise: every multiplier pushed against its bound, F rising with every call
        cases.append(_case(f"wval0-m{m}", m, "rising", stop=dict(maxeval=12), lo=0.0, hi=INF, y0=0.0))
        cases.append(_case(f"on-hi-m{m}", m, "quadratic", stop=dict(maxeval=100), lo=0.0, hi=2.0, y0=2.0, target=5.0))
        cases.append(_case(f"on-lo-m{m}", m, "quadratic", stop=dict(maxeval=100), lo=0.0, hi=INF, y0=0.0, target=-1.0))
        cases.append(_case(f"invalid-y0-above-m{m}", m, "quadratic", lo=0.0, hi=1.0, y0=1.5, target=0.5))
        cases.append(_case(f"invalid-lo-above-hi-m{m}", m, "quadratic", lo=0.0, hi=-1.0, y0=0.0, target=0.5))
        cases.append(_case(f"invalid-y0-below-m{m}", m, "quadratic", lo=0.5, hi=1.0, y0=0.25, target=0.5))
        cases.append(_case(f"lo-minus-inf-m{m}", m, "quadratic", stop=dict(maxeval=100), lo=-INF, hi=1.0, y0=0.0,
                           target=-3.0))
        # multiplier 0 held by lo = hi: sigma 0, no step
        cases.append(_case(f"pinned-m{m}", m, "quadratic", stop=dict(maxeval=100), lo=0.0, hi=4.0, y0=0.5, target=2.0,
                           pin=True))
        cases.append(_case(f"no-maxeval-m{m}", m, "quadratic", stop=dict(maxeval=0), lo=0.0, hi=INF, y0=0.0,
                           target=1.25))
    return cases


# ---- the functions ----------------------------------------------------------------------------------------------------
class RealDual:
    """F = the port's dual function (minus the dual value, minus its gradient) of a seeded instance"""

    def __init__(self, variant, inst):
        self.fn = ob.port().port_dual_mma if variant == "mma" else ob.port().port_dual_ccsaq
        self.arrs = {k: np.ascontiguousarray(inst[k], dtype=np.float64) for k in
                     ("x", "lb", "ub", "sigma", "grad_f", "grad_c", "c0", "rhoc")}
        p = {k: ob._p(a) for k, a in self.arrs.items()}
        n, m = inst["n"], inst["m"]
        self.din = ob.DualIn(n, m, p["x"], p["lb"], p["ub"], p["sigma"], p["grad_f"], p["grad_c"], inst["f0"],
                             inst["rho"], p["c0"], p["rhoc"])
        self.xcur, self.gc = np.empty(n), np.empty(m)
        self.dout = ob.DualOut(ob._p(self.xcur), ob._p(self.gc), 0.0, 0.0)

    def __call__(self, y, grad):
        y = np.ascontiguousarray(y, dtype=np.float64)
        return self.fn(C.byref(self.din), ob._p(y), grad.ctypes.data_as(ob.dp), C.byref(self.dout))


def _instance(case):
    m = case["m"]
    inst = synth.kernel_instance(case["n"], m, seed=synth.SEED0 + 7919 * case["seed"])
    inst["rho"] = case["rho"]
    i = np.arange(m, dtype=np.float64)
    if case["c0"] in ("infeasible", "nanrow-infeasible"):
        inst["c0"] = 0.25 + 0.125 * i             # every constraint violated at x: the driver caps y at 1e40
    if case["c0"].startswith("nanrow"):
        inst["c0"][m // 2] = NAN
    return inst


class Closed:
    """the closed-form edge functions; `calls` counts evaluations (some functions change with it)"""

    def __init__(self, case):
        self.case, self.calls = case, 0
        m = case["m"]
        self.a = [1.0 + 0.375 * i for i in range(m)]               # per-coordinate weights
        self.c = [0.3 + 0.1 * i for i in range(m)]                 # per-coordinate kinks of the oscillating F

    def __call__(self, y, grad):
        case, kind, m, a = self.case, self.case["kind"], self.case["m"], self.a
        k = self.calls
        self.calls += 1
        y = [float(v) for v in y]
        g = [0.0] * m
        if kind == "flat":
            v = 7.0
        elif kind == "linear":
            v = 0.0
            for i in range(m):
                v = v - a[i] * y[i]
                g[i] = -a[i]
        elif kind in ("quadratic", "nan_after", "inf_after", "nan_grad", "scaled"):
            t = case.get("target", 1.5)
            scale = case.get("scale", 1.0)
            v = 1.0
            for i in range(m):
                d = y[i] - t
                v = v + a[i] * d * d
                g[i] = 2.0 * a[i] * d
            if kind == "scaled":
                v = v * scale
                g = [gi * scale for gi in g]
            if kind == "nan_after" and k >= case["k"]:
                v = NAN
            if kind == "inf_after" and k == case["k"]:
                v = INF if case["sign"] == "+" else -INF
            if kind == "nan_grad" and k >= case["k"]:
                g[m - 1] = NAN
        elif kind == "approach":
            # strictly convex, minimum at 0.9 inside [0, 1]: approached from one side, sigma grows to its cap
            v = 0.0
            for i in range(m):
                d = 0.9 - y[i]
                v = v + a[i] * d * d * d * d + 0.001 * d * d
                g[i] = -(4.0 * a[i] * d * d * d + 0.002 * d)
        elif kind == "oscillate":
            # |y - c| plus a small quadratic: the sign of the gradient flips across the kink, the steps alternate
            v = 0.0
            for i in range(m):
                d = y[i] - self.c[i]
                v = v + a[i] * abs(d) + 0.01 * d * d
                g[i] = (a[i] if d > 0 else (-a[i] if d < 0 else 0.0)) + 0.02 * d
        elif kind == "switch":
            # the minimiser jumps across 0.5 with the side: every step crosses it, sigma shrinks to its floor
            v = 0.0
            for i in range(m):
                d = y[i] - (0.25 if y[i] > 0.5 else 0.75)
                v = v + a[i] * d * d
                g[i] = 2.0 * a[i] * d
        elif kind == "rising":
            # pushes every multiplier below its lower bound and rises with every call: the step is 0, so wval = 0,
            # and F(y) > gval = fbase at the same point
            v = 1.0 + k
            for i in range(m):
                g[i] = a[i]
        else:
            raise ValueError(kind)
        grad[:m] = g
        return v


def problem(case):
    """(F, y0, lo, hi): F(y, grad) -> value with grad[:m] filled; fresh state on every call"""
    m = case["m"]
    if case["kind"] in ("mma", "ccsaq"):
        inst = _instance(case)
        F = RealDual(case["kind"], inst)
        lo = np.zeros(m)
        hi = np.full(m, 1e40 if case["c0"] in ("infeasible", "nanrow-infeasible") else INF)
        y0 = np.zeros(m)
        if case["warm"] == "prev":
            # warm start where the driver's previous inner iteration ended: the solution (default stop rules, from 0)
            # of the same instance with a ten times smaller rho
            prev = dict(case, rho=case["rho"] * 0.1)
            y0 = port_run(prev, RealDual(case["kind"], _instance(prev)), y0, lo, hi, stop=DEFAULT_STOP)["y"]
        return F, y0, lo, hi
    lo, hi, y0 = np.full(m, float(case["lo"])), np.full(m, float(case["hi"])), np.full(m, float(case["y0"]))
    if case.get("pin"):
        lo[0] = hi[0] = y0[0]
    return Closed(case), y0, lo, hi


class Recorder:
    """wraps F and records every evaluation"""

    def __init__(self, F, m):
        self.F, self.m, self.ys, self.fs, self.gs = F, m, [], [], []

    def __call__(self, y, grad):
        g = np.zeros(self.m)
        v = float(self.F(np.array(y[:self.m], dtype=np.float64), g))
        if grad is not None and len(grad):
            grad[:self.m] = g
        self.ys.append(np.array(y[:self.m], dtype=np.float64))
        self.fs.append(v)
        self.gs.append(g.copy())
        return v

    def arrays(self):
        m, k = self.m, len(self.fs)
        ys = np.array(self.ys, dtype=np.float64).reshape(k, m)
        gs = np.array(self.gs, dtype=np.float64).reshape(k, m)
        return ys, np.array(self.fs, dtype=np.float64), gs


def fingerprint(ys, fs, gs):
    """sha256 of the trajectory's bits: per evaluation y_k, F_k, grad F_k, in order (tests/reference_runs.sha256_bits)"""
    k = len(fs)
    rows = np.concatenate([ys.reshape(k, -1), fs.reshape(k, 1), gs.reshape(k, -1)], axis=1) if k else np.zeros(0)
    return hashlib.sha256(np.ascontiguousarray(rows, dtype=np.float64).tobytes()).hexdigest()


def port_run(case, F, y0, lo, hi, stop=None):
    """the oracle port's nested level: port_ccsa_minimize(PORT_MMA, m, F, ..., 0 constraints) with the dual
    optimiser's stop rules.  Returns ret, y, minf, nevals and the trajectory (ys, fs, gs)."""
    m = case["m"]
    stop = case["stop"] if stop is None else stop
    rec = Recorder(F, m)
    L = ob.port()

    def thunk(nn, x, g, _d):
        xa = np.ctypeslib.as_array(x, shape=(nn,))
        ga = np.ctypeslib.as_array(g, shape=(nn,)) if g else None
        return rec(xa, ga)

    fcb = ob.PORT_FUNC(thunk)
    o = ob.Options()
    L.port_default_options(C.byref(o))
    xtol_abs = np.full(m, float(stop["xtol_abs"]))
    o.ftol_rel, o.ftol_abs, o.xtol_rel = stop["ftol_rel"], stop["ftol_abs"], stop["xtol_rel"]
    o.xtol_abs, o.maxeval = ob._p(xtol_abs), stop["maxeval"]
    lo, hi = np.ascontiguousarray(lo, dtype=np.float64), np.ascontiguousarray(hi, dtype=np.float64)
    y = np.array(y0, dtype=np.float64)
    tol = np.zeros(1)
    carr = (ob.PORT_FUNC * 1)()
    cdata = (C.c_void_p * 1)()
    minf = C.c_double(0.0)
    ret = L.port_ccsa_minimize(ob.MMA, m, fcb, None, 0, carr, cdata, ob._p(tol), ob._p(lo), ob._p(hi), ob._p(y),
                               C.byref(minf), C.byref(o), None)
    ys, fs, gs = rec.arrays()
    return dict(ret=ret, y=y, minf=minf.value, nevals=len(fs), ys=ys, fs=fs, gs=gs)


def trajectory(case):
    """(y0, lo, hi, port result with its trajectory) of one case"""
    F, y0, lo, hi = problem(case)
    if isinstance(F, Closed):
        F.calls = 0
    return y0, lo, hi, port_run(case, F, y0, lo, hi)


def hexs(a):
    return [float(v).hex() for v in np.asarray(a, dtype=np.float64).reshape(-1)]


def unhex(s):
    return np.array([float.fromhex(v) for v in s], dtype=np.float64)
