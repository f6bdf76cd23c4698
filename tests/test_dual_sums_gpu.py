"""The 3 + m sums of the library's dual kernels against exact sums of the model's terms (tests/dual_sums_model.py), on
the instances whose mutants tests/test_dual_sums.py shows the check rejects.

(a) Every evaluation form of test_closed_forms_gpu.EVAL_FORMS through DualHandle, with array bounds and, where the
    instance's bounds are uniform, with scalar bounds (the SB instantiations): x* bit for bit against
    closed_form_model, every sum within its depth bound of the exact sum.  m in dual_sums_model.MS, n at the geometry
    edges and ragged, two instances at n = 1e7.
(b) Every solve form of test_closed_forms_gpu.SOLVE_FORMS through DualHandle.solve: the returned sums at the returned
    y, and the x* it leaves, the same way.
(c) The wide kernel at m = 17 .. 2048, with NaN constraint values on some rows; m = 2049 is refused with the library's
    message.
(d) dual_eval_kernel, dual_eval_tma_kernel and dual_eval_wide_kernel as rank r of 2, 4 and 8 on one GPU through
    tests/cpp/dual_ranks_probe.cu (the NCCL path: the folder writes its virtual-shard sums, publish_kernel folds the
    gathered records): the published sums are those of one rank bit for bit, and those of the library's handle.

With -s the file prints the largest |got - exact| / (2^-53 sum|t|) per form against its depth bound (over the sums
whose constant is zero or absent: w, and every sum of the instances without constants), and the dynamic shared
memory and occupancy of the wide kernel at m = 2048.
"""
import ctypes as C
import os
import subprocess
from collections import defaultdict

import numpy as np
import pytest

import closed_form_model as cf
import dual_sums_model as dm
import oracle_bindings as ob
import outer_model as om
from gpu_dual import DualHandle
from test_closed_forms_gpu import EVAL_FORMS, SOLVE_FORMS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = (dm.MMA, dm.CCSAQ)
NAMES = {dm.MMA: "MMA", dm.CCSAQ: "CCSAQ"}
WIDE_FORMS = ((-1, 0), (-1, 1), (-1, 3))
LARGEST = defaultdict(lambda: [0.0, 0, ""])         # form -> [largest ratio, its depth, where]


def note(form, ref, got, what):
    r = ref.largest_ratio(got)
    if r >= LARGEST[form][0]:
        LARGEST[form][:] = [r, ref.dep, what]


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for form, (r, dep, what) in sorted(LARGEST.items()):
        print(f"largest |got - exact| / (2^-53 sum|t|): {form}: {r:.3g} (depth bound {dep}; {what})")


def first_bad(ok, *arrays):
    j = int(np.flatnonzero(~ok)[0])
    return f"{np.count_nonzero(~ok)} lanes, first {j}: " + ", ".join(f"{a[j]!r}" for a in arrays)


def returned(out):
    return dm.raw_values(np.concatenate([[out["ret"], out["g0"], out["w"]], out["gc"]]))


# ---- (a) evaluation forms ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("m", dm.MS)
def test_evaluation_forms_give_the_exact_sums(built, variant, m):
    for family, n in dm.cases(variant, m):
        inst = dm.instance(family, n, m, variant)
        y = inst["y"]
        xc, terms, consts = dm.expected(variant, inst, y)
        ref = dm.Sums(terms, dm.depth("eval", om.geometry(n), m), consts)
        h = DualHandle(variant, inst)
        for sb in ((False, True) if dm.uniform_bounds(inst) else (False,)):
            h.configure("scalar_bounds", int(sb))
            for cfg, cps in (EVAL_FORMS if n < 10 ** 7 else EVAL_FORMS[:1] + EVAL_FORMS[-3:-2]):
                h.configure("kernel_cfg", cfg)
                h.configure("ctas_per_sm", cps)
                what = f"{NAMES[variant]} m={m} {family} n={n} cfg={cfg} cps={cps}{' scalar bounds' if sb else ''}"
                with np.errstate(all="ignore"):
                    got = h.eval(y, want_xcur=True)
                ok = cf.same_bits(got["xcur"], xc)
                assert ok.all(), what + " x*: " + first_bad(ok, got["xcur"], xc)
                ref.check(returned(got), what)
                note("eval" + (" (scalar bounds)" if sb else ""), ref, returned(got), what)


# ---- (b) solve forms ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("m", [m for m in dm.MS if m >= 1])
def test_solve_forms_give_the_exact_sums(built, variant, m):
    for family, n in dm.cases(variant, m)[:2]:
        inst = dm.instance(family, n, m, variant)
        _, terms, consts = dm.expected(variant, inst, inst["y"])
        if not all(np.isfinite(t).all() for t in terms) or not np.isfinite([c for c in consts if c is not None]).all():
            continue          # the solve stops at once on a dual function that is NaN at the start
        for name, value in SOLVE_FORMS:
            for sb in ((False, True) if dm.uniform_bounds(inst) else (False,)):
                h = DualHandle(variant, inst)
                h.configure("scalar_bounds", int(sb))
                h.configure(name, value)
                what = f"{NAMES[variant]} m={m} {family} n={n} {name}={value}{' scalar bounds' if sb else ''}"
                with np.errstate(all="ignore"):
                    r = h.solve(inst["y"], maxeval=4)
                assert r["result"] != -2, what + ": the solve refused its arguments"
                y = r["y"][:m]
                xc, terms, consts = dm.expected(variant, inst, y)
                ok = cf.same_bits(r["xcur"], xc)
                assert ok.all(), what + " x*: " + first_bad(ok, r["xcur"], xc)
                ref = dm.Sums(terms, dm.depth("solve", om.geometry(n), m), consts)
                got = dm.raw_values(r["out"][:3 + m])
                ref.check(got, what + f" at y = {y}")
                note("solve", ref, got, what)


# ---- (c) the wide kernel ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("i", range(len(dm.WIDE)))
def test_the_wide_kernel_gives_the_exact_sums(built, variant, i):
    m, n = dm.WIDE[i]
    inst = dm.wide_instance(m, n, variant, i % 2 == 1)
    xc, terms, consts = dm.expected(variant, inst, inst["y"])
    ref = dm.Sums(terms, dm.depth("wide", om.geometry(n), m), consts)
    h = DualHandle(variant, inst)
    for cfg, cps in WIDE_FORMS:
        h.configure("kernel_cfg", cfg)
        h.configure("ctas_per_sm", cps)
        what = f"wide {NAMES[variant]} m={m} n={n} cps={cps}{' NaN rows' if i % 2 else ''}"
        with np.errstate(all="ignore"):
            got = h.eval(inst["y"], want_xcur=True)
        ok = cf.same_bits(got["xcur"], xc)
        assert ok.all(), what + " x*: " + first_bad(ok, got["xcur"], xc)
        ref.check(returned(got), what)
        note("wide", ref, returned(got), what)


def test_more_than_2048_rows_are_refused(built, capfd):
    with pytest.raises(RuntimeError):
        DualHandle(dm.MMA, n=1025, m=2049)
    err = capfd.readouterr().err
    assert "more than 2048 inequality constraints" in err and "96 bytes" in err, err
    DualHandle(dm.MMA, n=1025, m=2048)                  # the cap itself is accepted


# ---- (d) emulated ranks --------------------------------------------------------------------------------------------------
KINDS = {"register": 0, "tma": 1, "wide": 2}


class Probe:
    def __init__(self, so):
        L = self.L = C.CDLL(so, mode=C.RTLD_LOCAL)
        dp, i = ob.dp, C.c_int
        L.drp_error.restype = C.c_char_p
        L.drp_occupancy.argtypes = [i, i, i, C.POINTER(C.c_longlong), C.POINTER(i), C.POINTER(i)]
        L.drp_eval.argtypes = [i, i, i, C.POINTER(C.c_ulonglong), C.c_ulonglong, dp, dp, dp, dp, dp, dp, dp, dp,
                               C.POINTER(i), C.c_double, i, i, i, i, dp, dp, dp]
        L.drp_publish.argtypes = [dp, i, i, dp]

    def check(self, rc):
        if rc != 0:
            raise RuntimeError(self.L.drp_error().decode())

    def occupancy(self, kind, variant, m):
        smem, per_sm, sms = C.c_longlong(0), C.c_int(0), C.c_int(0)
        self.check(self.L.drp_occupancy(KINDS[kind], variant, m, C.byref(smem), C.byref(per_sm), C.byref(sms)))
        return smem.value, per_sm.value, sms.value

    def eval(self, kind, variant, inst, g, publish, nvp, out_dev):
        """one rank's launch on its slice: (totals [nvp], x* of the slice)"""
        m = inst["m"]
        nl = int(g.n_local)
        ld = -(-nl // om.CHUNK) * om.CHUNK
        sl = slice(int(g.j0), int(g.j0) + nl)

        def cut(a, fill=0.0):
            out = np.full(ld, fill)
            out[:nl] = a[sl]
            return out
        arr = [cut(inst[k]) for k in ("x", "lb", "ub", "sigma", "grad_f")]
        G = np.zeros((m, ld))
        G[:, :nl] = np.reshape(inst["grad_c"], (m, inst["n"]))[:, sl]
        geo = (C.c_ulonglong * 8)(g.n_local, g.nchunks, g.chunk0, g.groups_total, g.group0, g.groups_per_vshard,
                                  g.local_vshards, g.groups_local)
        y = np.ascontiguousarray(inst["y"], dtype=np.float64)
        rhoc = np.ascontiguousarray(inst["rhoc"], dtype=np.float64)
        active = np.ascontiguousarray(~np.isnan(inst["c0"]) if variant == dm.MMA else np.ones(m, dtype=bool), dtype=np.int32)
        out = np.zeros(nvp)
        xcur = np.zeros(ld)
        self.check(self.L.drp_eval(KINDS[kind], variant, m, geo, ld, *[ob._p(a) for a in arr], ob._p(G), ob._p(y),
                                   ob._p(rhoc), active.ctypes.data_as(C.POINTER(C.c_int)), float(inst["rho"]), g.rank,
                                   g.world, int(publish), nvp, ob._p(out_dev), ob._p(out), ob._p(xcur)))
        return out, xcur[:nl]

    def publish(self, out_dev, nv, nvp):
        out = np.zeros(nvp)
        self.check(self.L.drp_publish(ob._p(out_dev), nv, nvp, ob._p(out)))
        return out


@pytest.fixture(scope="module")
def probe(built):
    """tests/cpp/dual_ranks_probe.cu -> tests/_build/ with the library's compiler flags; the ptxas log is kept beside
    the library.  Rebuilt when the probe, any file of nlopt_b200/csrc or the command line changes."""
    g = built
    csrc = os.path.join(ROOT, "nlopt_b200", "csrc")
    src = os.path.join(ROOT, "tests", "cpp", "dual_ranks_probe.cu")
    so = os.path.join(ROOT, "tests", "_build", "libdual_ranks_probe.so")
    log = so + ".ptxas.log"
    cmd = [g.NVCC, *g.ARCH, *g.NVCC_FLAGS, "-I" + csrc, "-shared", src, "-cudart", "shared", "-o"]
    head = " ".join(cmd) + "\n"
    deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
    fresh = os.path.exists(so) and os.path.exists(log) and all(os.path.getmtime(d) <= os.path.getmtime(so) for d in deps)
    if fresh:
        with open(log) as f:
            fresh = f.readline() == head
    if not fresh:
        os.makedirs(os.path.dirname(so), exist_ok=True)
        tmp = so + f".{os.getpid()}.tmp"
        r = subprocess.run(cmd + [tmp], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        with open(log, "w") as f:
            f.write(head + r.stdout)
        os.replace(tmp, so)
    return Probe(so)


def test_wide_kernel_occupancy_at_2048_rows(probe):
    for variant in VARIANTS:
        smem, per_sm, sms = probe.occupancy("wide", variant, 2048)
        assert smem == 12 * 2048 * 8 and per_sm >= 1
        print(f"dual_eval_wide_kernel {NAMES[variant]} m = 2048: {smem} bytes ({smem / 1024:.0f} KiB) of dynamic shared "
              f"memory, {per_sm} CTA(s) of 256 threads per SM, {sms} SMs")


RANK_CASES = [(k, v, n) for k in ("register", "tma", "wide") for v in VARIANTS for n in (4097, 300001, 1250001)]


@pytest.mark.parametrize("kind,variant,n", RANK_CASES, ids=[f"{k}-{NAMES[v]}-{n}" for k, v, n in RANK_CASES])
def test_emulated_ranks_give_the_bits_of_one_rank(probe, kind, variant, n):
    m = 20 if kind == "wide" else 4
    inst = dm.instance("2^+-30 jumps", n, m, variant, seed=2)
    inst["f0"], inst["c0"] = 0.0, np.zeros(m)
    if kind == "wide" and variant == dm.MMA:
        inst["c0"][5] = np.nan                           # a row switched off
    nvp = (3 + m + 3) // 4 * 4
    xc, terms, _ = dm.expected(variant, inst, inst["y"])
    one, x1 = probe.eval(kind, variant, inst, om.geometry(n), True, nvp, np.zeros(8 * nvp))
    what = f"{kind} {NAMES[variant]} n={n}"
    ok = cf.same_bits(x1, xc)
    assert ok.all(), what + " one rank x*: " + first_bad(ok, x1, xc)
    ref = dm.Sums(terms, dm.depth("wide" if kind == "wide" else "eval", om.geometry(n), m))
    ref.check(one[:3 + m], what + " one rank")
    note(f"{kind} kernel (probe, no constants)", ref, one[:3 + m], what)
    # the library's handle on the same instance: the same sums (f0 = c0 = 0: its constants add nothing)
    h = DualHandle(variant, inst)
    if kind == "tma":
        h.configure("kernel_cfg", 11)
    lib = h.eval(inst["y"])
    assert cf.same_term(returned(lib)[:3 + m], np.concatenate([[one[0]], one[1:3 + m]])).all(), \
        f"{what}: the probe's one-rank sums {one[:3 + m]} differ from the library's {returned(lib)}"
    for world in (2, 4, 8):
        out_dev = np.full(8 * nvp, om.GUARD)
        x = np.zeros(n)
        for rank in range(world):
            g = om.geometry(n, rank, world)
            assert g.n_local > 0
            _, xs = probe.eval(kind, variant, inst, g, False, nvp, out_dev)
            x[int(g.j0):int(g.j0) + int(g.n_local)] = xs
        assert not np.any(om.bits(out_dev.reshape(8, nvp)[:, :3 + m]) == om.bits(np.array([om.GUARD]))[0]), \
            f"{what} world={world}: a virtual-shard record was not written"
        got = probe.publish(out_dev, 3 + m, nvp)
        om.check_bits(got[:3 + m], one[:3 + m], f"{what} world={world}: published sums against one rank")
        ok = cf.same_bits(x, xc)
        assert ok.all(), f"{what} world={world} x*: " + first_bad(ok, x, xc)
