"""Registration of every user-callback form, checked on the CPU-backed build of the host logic (hosttest_lib).

For each public entry point (objectives, scalar and vector constraints, in every callback form) and each bad-argument
case: the result code, the error message, and which user data reach the munge hooks through a refusal, nlopt_copy,
nlopt_munge_data and nlopt_destroy.  The terms forms' agreement with their _device2 twins is in test_terms_callbacks.py;
this file extends that pattern to every form.  Also: NLOPT_AUGLAG_EQ drops the preconditioners of its sub-problem
(auglag.c:109-135), so a preconditioned run gives the bits of the plain one.
"""
import ctypes as C

import numpy as np
import pytest

import nlopt_b200 as nl
from nlopt_b200 import _capi
from test_terms_callbacks import DFUNC2, DMFUNC2, MUNGE, _errmsg, _tolp

SFUNC = C.CFUNCTYPE(C.c_double, C.c_uint, C.c_ulonglong, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p)
MUNGE2 = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_void_p)
ALGS = (nl.LD_MMA, nl.LD_CCSAQ, nl.LD_AUGLAG)
PRIOR = "invalid bound index"          # an error message set before each registration: shows whether it was cleared

# (group, form): the entry points of each form, "min"/"max" objectives or "inequality"/"equality" constraints
OBJECTIVE_FORMS = ("host", "precond", "device", "device2", "terms", "sharded")
CONSTRAINT_FORMS = ("host", "precond", "device", "device2", "terms", "sharded")
VECTOR_FORMS = ("host", "device2", "terms")
ENTRY_POINTS = ([("objective", what, form) for form in OBJECTIVE_FORMS for what in ("min", "max")]
                + [("constraint", what, form) for form in CONSTRAINT_FORMS for what in ("inequality", "equality")
                   if not (form == "sharded" and what == "equality")]           # no sharded equality entry point
                + [("vector", what, form) for form in VECTOR_FORMS for what in ("inequality", "equality")])


@pytest.fixture(scope="module")
def cbs():
    """callables to register: their addresses only; none of them is called"""
    keep = dict(f=_capi.NLOPT_FUNC(lambda *a: 0.0), mf=_capi.NLOPT_MFUNC(lambda *a: None),
                pre=_capi.NLOPT_PRECOND(lambda *a: None), df=_capi.NLOPT_B200_DFUNC(lambda *a: 0.0),
                f2=DFUNC2(lambda *a: None), mf2=DMFUNC2(lambda *a: None), terms=_capi.NLOPT_B200_DTFUNC(lambda *a: None),
                fin=_capi.NLOPT_B200_DFINISH(lambda t, d: t), mfin=_capi.NLOPT_B200_DMFINISH(lambda *a: None),
                sf=SFUNC(lambda *a: 0.0))
    out = {k: C.cast(v, C.c_void_p) for k, v in keep.items()}
    out["_keep"] = keep
    return out


def _cases(group, form):
    """keyword sets for _register: good input first, then each bad-argument case of this form"""
    if group == "objective":
        return {"device2": [{}, dict(fn=False), dict(fin=False), dict(halo=-1), dict(halo=2), dict(halo=1)],
                "terms": [{}, dict(fn=False), dict(fin=False), dict(halo=-1), dict(halo=2), dict(halo=1)],
                "precond": [{}, dict(fn=False), dict(pre=False)]}.get(form, [{}, dict(fn=False)])
    if group == "constraint":
        return {"device2": [{}, dict(fn=False), dict(fin=False), dict(halo=-1), dict(halo=2), dict(halo=1), dict(tol=-1e-3),
                            dict(fn=False, tol=-1e-3)],
                "terms": [{}, dict(fn=False), dict(fin=False), dict(halo=-1), dict(halo=2), dict(halo=1), dict(tol=-1e-3),
                          dict(fn=False, tol=-1e-3)],
                "precond": [{}, dict(fn=False), dict(pre=False), dict(tol=-1e-3), dict(fn=False, tol=-1e-3)]}.get(
                    form, [{}, dict(fn=False), dict(tol=-1e-3), dict(fn=False, tol=-1e-3)])
    cases = [{}, dict(tol=None), dict(m=1, tol=[0.5]), dict(fn=False), dict(tol=[0.0, -1e-3, 0.0]),
             dict(fn=False, tol=[0.0, -1e-3, 0.0]), dict(m=0, tol=None), dict(m=0, tol=None, fn=False, fin=False, halo=5)]
    if form != "host":
        cases += [dict(fin=False), dict(halo=-1), dict(halo=2), dict(halo=1, tol=[1e-6, 0.0, 2.0])]
    return cases


def _register(L, h, cbs, group, what, form, fn=True, fin=True, pre=True, tol=0.0, halo=0, m=3, data=None):
    """one registration through the public entry point of (group, what, form)"""
    raw = L.raw
    h, d, hl = C.c_void_p(h), C.c_void_p(data), C.c_int(halo)
    vector = group == "vector"
    fnp = (cbs[{"host": "mf" if vector else "f", "precond": "f", "device": "df", "device2": "mf2" if vector else "f2",
                "terms": "terms", "sharded": "sf"}[form]] if fn else None)
    finp = (cbs["mfin" if vector else "fin"] if fin else None)
    prep = cbs["pre"] if pre else None
    if group == "objective":
        name, args = {"host": (f"nlopt_set_{what}_objective", (fnp, d)),
                      "precond": (f"nlopt_set_precond_{what}_objective", (fnp, prep, d)),
                      "device": (f"nlopt_b200_set_{what}_objective_device", (fnp, d)),
                      "device2": (f"nlopt_b200_set_{what}_objective_device2", (fnp, finp, d, hl)),
                      "terms": (f"nlopt_b200_set_{what}_objective_terms", (fnp, finp, d, hl)),
                      "sharded": (f"nlopt_b200_set_{what}_objective_sharded", (fnp, d))}[form]
    elif group == "constraint":
        t = C.c_double(tol)
        name, args = {"host": (f"nlopt_add_{what}_constraint", (fnp, d, t)),
                      "precond": (f"nlopt_add_precond_{what}_constraint", (fnp, prep, d, t)),
                      "device": (f"nlopt_b200_add_{what}_constraint_device", (fnp, d, t)),
                      "device2": (f"nlopt_b200_add_{what}_constraint_device2", (fnp, finp, d, t, hl)),
                      "terms": (f"nlopt_b200_add_{what}_constraint_terms", (fnp, finp, d, t, hl)),
                      "sharded": (f"nlopt_b200_add_{what}_constraint_sharded", (fnp, d, t))}[form]
    else:
        if tol is not None and np.isscalar(tol):
            tol = np.full(max(m, 1), tol)
        tp = _tolp(tol)
        name, args = {"host": (f"nlopt_add_{what}_mconstraint", (C.c_uint(m), fnp, d, tp)),
                      "device2": (f"nlopt_b200_add_{what}_mconstraint_device2", (C.c_uint(m), fnp, finp, d, tp, hl)),
                      "terms": (f"nlopt_b200_add_{what}_mconstraint_terms", (C.c_uint(m), fnp, finp, d, tp, hl))}[form]
    return getattr(raw, name)(h, *args)


def _expected(alg, group, what, form, kw, data):
    """(result, errmsg, destroyed at registration, registered) by the rules of options.c and the extension entry points"""
    fn, fin, halo, m = kw.get("fn", True), kw.get("fin", True), kw.get("halo", 0), kw.get("m", 1 if group != "vector" else 3)
    tol = kw.get("tol", 0.0)
    checked = form in ("device2", "terms") and not (group == "vector" and m == 0)
    if (checked and (not fn or not fin or halo not in (0, 1))) or (form == "sharded" and not fn):
        return nl.INVALID_ARGS, PRIOR, [], False            # refused before clear_err, the data untouched
    if group == "objective":
        return nl.SUCCESS, None, [None], True                # the previous objective's (NULL) data is munged
    if group == "vector" and m == 0:
        return nl.SUCCESS, None, [data], False               # options.c:560-564
    if what == "equality" and alg != nl.LD_AUGLAG:
        return nl.INVALID_ARGS, "invalid algorithm for constraints", [data], False
    if not fn:
        return nl.INVALID_ARGS, None, [data], False
    if tol is not None and np.any(np.asarray(tol) < 0):
        return nl.INVALID_ARGS, "negative constraint tolerance", [data], False
    return nl.SUCCESS, None, [], True


@pytest.fixture(scope="module")
def lib(hosttest_lib):
    hosttest_lib.raw = C.CDLL(hosttest_lib.path, mode=C.RTLD_LOCAL)      # untyped: every argument passed as a ctypes value
    return hosttest_lib


@pytest.mark.parametrize("group,what,form", ENTRY_POINTS)
def test_registration_codes_messages_and_munge(lib, cbs, group, what, form):
    L = lib
    destroyed, copied, munged = [], [], []
    on_destroy = MUNGE(lambda d: destroyed.append(d) or None)
    on_copy = MUNGE(lambda d: copied.append(d) or d)
    mg = MUNGE2(lambda p, d: munged.append(p) or p)
    for alg in ALGS:
        for i, kw in enumerate(_cases(group, form)):
            data = 0x1000 + 16 * i
            destroyed.clear(), copied.clear(), munged.clear()
            o = L.nlopt_create(alg, 5)
            L.nlopt_set_munge(o, C.cast(on_destroy, C.c_void_p), C.cast(on_copy, C.c_void_p))
            assert L.nlopt_set_lower_bound(o, -1, 0.0) == nl.INVALID_ARGS and _errmsg(L, o) == PRIOR
            got = (_register(L, o, cbs, group, what, form, data=data, **kw), _errmsg(L, o), list(destroyed))
            ret, msg, gone, registered = _expected(alg, group, what, form, kw, data)
            assert got == (ret, msg, gone), (alg, kw, got)
            mine = [data] if registered else []
            c = L.nlopt_copy(o)
            assert c and copied == mine, (alg, kw, copied)
            L.nlopt_munge_data(o, C.cast(mg, C.c_void_p), None)
            objective = (mine or [None]) if group == "objective" else [None] + mine      # the objective's data, NULL too
            assert munged == objective, (alg, kw, munged)
            for h in (c, o):
                destroyed.clear()
                L.nlopt_destroy(h)
                assert destroyed == objective, (alg, kw, destroyed)


def test_munge_order_across_lists(lib, cbs):
    """the objective's data first, then the inequality constraints', then the equality constraints', each list in
    registration order, whatever order and form they were registered in"""
    L = lib
    destroyed, copied, munged = [], [], []
    on_destroy = MUNGE(lambda d: destroyed.append(d) or None)
    on_copy = MUNGE(lambda d: copied.append(d) or d)
    mg = MUNGE2(lambda p, d: munged.append(p) or p)
    o = L.nlopt_create(nl.LD_AUGLAG, 5)
    L.nlopt_set_munge(o, C.cast(on_destroy, C.c_void_p), C.cast(on_copy, C.c_void_p))
    steps = [("constraint", "equality", "host", 0x21), ("constraint", "inequality", "device2", 0x11),
             ("vector", "equality", "terms", 0x22), ("constraint", "inequality", "sharded", 0x12),
             ("objective", "max", "precond", 0x01), ("vector", "inequality", "host", 0x13),
             ("constraint", "equality", "device", 0x23)]
    for group, what, form, data in steps:
        assert _register(L, o, cbs, group, what, form, data=data) == nl.SUCCESS
    order = [0x01, 0x11, 0x12, 0x13, 0x21, 0x22, 0x23]
    c = L.nlopt_copy(o)
    assert copied == order
    L.nlopt_munge_data(o, C.cast(mg, C.c_void_p), None)
    assert munged == order
    destroyed.clear()
    L.nlopt_remove_inequality_constraints(c)
    assert destroyed == [0x11, 0x12, 0x13]
    for h in (c, o):
        destroyed.clear()
        L.nlopt_destroy(h)
    assert destroyed == order


def _eq_run(L, alg, local, precond):
    """min sum (x - 1)^2 + x0 x1  s.t.  x0 + x1 - 1 <= 0,  x2 - x3 = 0.5"""
    n = 4
    o = nl.opt(alg, n, library=L)
    o.set_lower_bounds(-3.0)
    o.set_upper_bounds(3.0)
    o.set_xtol_rel(1e-10)
    o.set_maxeval(400)

    def f(x, g):
        if g.size:
            g[:] = 2 * (x - 1)
            g[0] += x[1]
            g[1] += x[0]
        return float((x - 1) @ (x - 1) + x[0] * x[1])

    def c(x, g):
        if g.size:
            g[:] = [1.0, 1.0, 0.0, 0.0]
        return float(x[0] + x[1] - 1)

    def h(x, g):
        if g.size:
            g[:] = [0.0, 0.0, 1.0, -1.0]
        return float(x[2] - x[3] - 0.5)

    def pre(x, v, vpre):
        vpre[:] = 3.0 * v

    if precond:
        o.set_precond_min_objective(f, pre)
        o.add_precond_inequality_constraint(c, pre, 1e-8)
    else:
        o.set_min_objective(f)
        o.add_inequality_constraint(c, 1e-8)
    if local is not None:
        lo = nl.opt(local, n, library=L)
        lo.set_xtol_rel(1e-10)
        lo.set_maxeval(200)
        o.set_local_optimizer(lo)
        o.add_equality_constraint(h, 1e-8)
    x = np.array([0.2, -0.1, 0.4, 0.3])
    ret = L.nlopt_optimize(o._h, x.ctypes.data_as(_capi.c_double_p), C.byref(fv := C.c_double()))
    return ret, o.get_numevals(), fv.value.hex(), x.tobytes()


def test_auglag_eq_drops_preconditioners(lib):
    """NLOPT_AUGLAG_EQ over LD_CCSAQ: the sub-problem takes the objective and the inequality constraint without their
    preconditioners (auglag.c:109-135), so the run is the plain run bit for bit -- while a CCSAQ run of its own does
    use them"""
    L = lib
    plain, pre = _eq_run(L, nl.AUGLAG_EQ, nl.LD_CCSAQ, False), _eq_run(L, nl.AUGLAG_EQ, nl.LD_CCSAQ, True)
    assert plain[0] > 0 and plain[1] > 0, plain
    assert pre == plain
    alone, alone_pre = _eq_run(L, nl.LD_CCSAQ, None, False), _eq_run(L, nl.LD_CCSAQ, None, True)
    assert alone[0] > 0 and alone_pre[0] > 0
    assert alone_pre != alone
