"""The device dual optimiser (WarpDualMachine<MAXM> in nlopt_b200/csrc/ccsa_kernels.cuh) against the reference's nested
MMA, bit for bit, on the H100; and the persistent dual-solve kernel around it against the host-driven solve.

tests/cpp/warp_dual_machine_probe.cu runs the machine on one warp with the calls solve_folder makes.  Every trajectory of
tests/dual_trajectories.py with m <= 16 is replayed in the instantiation the library picks for m and, for m < 16, in
MAXM = 16 as well, so the predicated lanes of the wider instantiations run too.  The time limit cannot be replayed from
the reference; there the device machine is compared with the host machine (tests/test_dual_machine.py's probe).
"""
import ctypes as C
import functools
import os
import subprocess
import time

import numpy as np
import pytest

import nlopt_b200 as nl
import oracle_bindings as ob
import problems as P
import synth
import test_dual_machine as H
from gpu_dual import DualHandle
from test_gpu_parity import _run

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nlopt_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "cpp", "warp_dual_machine_probe.cu")
SO = os.path.join(ROOT, "tests", "_build", "libwarp_dual_machine_probe.so")
MAXMS = (1, 2, 4, 8, 16)


def build_probe(g):
    """warp_dual_machine_probe.cu -> tests/_build/ with the library's nvcc flags (g = __graft_entry__); rebuilt when the
    probe, any file of nlopt_b200/csrc or the command line changes.  Returns the library and the ptxas log."""
    log = SO + ".ptxas.log"
    cmd = [g.NVCC, *g.ARCH, *g.NVCC_FLAGS, "-I" + CSRC, "-shared", SRC, "-cudart", "shared", "-o"]
    head = " ".join(cmd) + "\n"
    deps = [SRC] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    fresh = os.path.exists(SO) and os.path.exists(log) and all(os.path.getmtime(d) <= os.path.getmtime(SO) for d in deps)
    if fresh:
        with open(log) as f:
            fresh = f.readline() == head
    if not fresh:
        os.makedirs(os.path.dirname(SO), exist_ok=True)
        tmp = SO + f".{os.getpid()}.tmp"
        r = subprocess.run(cmd + [tmp], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 0, r.stdout
        with open(log, "w") as f:
            f.write(head + r.stdout)
        os.replace(tmp, SO)
    L = C.CDLL(SO)
    dp = C.POINTER(C.c_double)
    L.wdm_replay.restype = C.c_int
    L.wdm_replay.argtypes = [C.c_int, C.c_int, dp, dp, dp, dp, C.c_long, C.c_long, dp, dp, dp, dp,
                             C.POINTER(C.c_longlong)]
    L.wdm_error.restype = C.c_char_p
    with open(log) as f:
        return L, f.read()


@pytest.fixture(scope="module")
def probe(built):
    L, log = build_probe(built)
    spills = [ln.strip() for ln in log.splitlines() if "spill" in ln and "0 bytes spill stores, 0 bytes spill loads" not in ln]
    print("warp machine probe, ptxas lines with spills (information only):", spills or "none")
    return L


def device_replay(L, maxm, case, t, k_time=-1):
    m = case["m"]
    y0, lo, hi, run = t
    K = len(run["fs"])
    ys, fs, gs = (np.ascontiguousarray(a, dtype=np.float64).reshape(-1) for a in (run["ys"], run["fs"], run["gs"]))
    dummy = np.zeros(1)
    yf = np.zeros(33)
    counts = (C.c_longlong * 5)()
    rc = L.wdm_replay(maxm, m, H._p(np.ascontiguousarray(y0, dtype=np.float64)), H._p(lo), H._p(hi),
                      H._p(H.stop5(case["stop"])), k_time, K, H._p(ys if K else dummy), H._p(fs if K else dummy),
                      H._p(gs if K else dummy), H._p(yf), counts)
    assert rc == 0, L.wdm_error().decode()
    return dict(ret=counts[0], nevals=counts[1], feeds=counts[2], status=counts[3], where=counts[4], y=yf[:m].copy(),
                fmin=yf[32])


@functools.lru_cache(maxsize=None)
def maxm_of(m):
    """the instantiation the library runs for m rows (DeviceBackend's pick_maxm)"""
    return int(DualHandle(ob.MMA, n=1024, m=m, synthetic_seed=1).query("maxm"))


@pytest.fixture(scope="module")
def cases(built):
    return H.load_cases()


def test_warp_machine_replays_every_trajectory(cases, probe):
    """every trajectory with m <= 16: the device machine asks for the reference's points bit for bit and ends with the
    reference's code, y, fmin and count, in pick_maxm(m) and in MAXM = 16"""
    t0 = time.perf_counter()
    bad, per_maxm = [], {k: 0 for k in MAXMS}
    picks = {}
    for case, t, want in cases:
        m = case["m"]
        if m > 16:
            continue
        if m not in picks:
            picks[m] = maxm_of(m)
            assert picks[m] in MAXMS and picks[m] >= m
        for maxm in sorted({picks[m], 16}):
            why = H.agrees(case, t, device_replay(probe, maxm, case, t), want)
            per_maxm[maxm] += 1
            if why:
                bad.append((case["name"], maxm, why))
    print(f"device replays per MAXM: {per_maxm} in {time.perf_counter() - t0:.1f} s")
    assert not bad, bad
    assert all(per_maxm[k] > 0 for k in MAXMS)


def test_warp_machine_time_limit_equals_host_machine(built, cases, probe):
    """time_up from evaluation k on (device) and elapsed >= maxtime from k on (host): the same MAXTIME exit"""
    host = H.build_probe(built)
    picked = [c for c in cases if c[0]["kind"] in ("mma", "ccsaq") and c[0]["m"] in (1, 3, 5, 8, 12, 16)
              and c[0]["warm"] == "zero" and len(c[1][3]["fs"]) >= 8][::3]
    assert len(picked) >= 6
    for case, t, _ in picked:
        K = len(t[3]["fs"])
        for k in sorted({0, 1, K // 2, K - 1}):
            h = H.replay(host, case, t, k_time=k)
            assert h["ret"] in (5, 6) and h["feeds"] == k + 1, (case["name"], k, h)
            for maxm in sorted({maxm_of(case["m"]), 16}):
                d = device_replay(probe, maxm, case, t, k_time=k)
                assert (d["status"], d["ret"], d["nevals"], d["feeds"]) == (h["status"], h["ret"], h["nevals"], h["feeds"])
                assert H.bits(d["y"]) == H.bits(h["y"]) and H.bits([d["fmin"]]) == H.bits([h["fmin"]]), (case["name"], k)


# ---- the library glue: the persistent kernel against the host-driven loop ---------------------------------------------
def _solve(h, fused, y0, lo, hi, ftol_rel, maxeval):
    h.configure("fused_solve", fused)
    return h.solve(y0, lo, hi, ftol_rel=ftol_rel, maxeval=maxeval)


def _same(a, b):
    return (a["result"] == b["result"] and a["nevals"] == b["nevals"] and H.bits(a["y"]) == H.bits(b["y"])
            and H.bits(a["out"]) == H.bits(b["out"]) and H.bits(a["xcur"]) == H.bits(b["xcur"]))


@pytest.mark.parametrize("variant", [ob.MMA, ob.CCSAQ])
def test_fused_handle_solve_equals_host_driven(built, variant):
    """nlopt_b200_dual_solve with the persistent kernel (fused_solve 1) and with one launch per evaluation (0), at every
    m = 1 .. 16: the same y, sums, result, count and x*(y) bits.  Then a start outside the box on the same handle: result
    -2, y untouched, and the same count on both paths (no evaluation inside the solve)"""
    n = 20011
    for m in range(1, 17):
        inst = synth.kernel_instance(n, m, seed=synth.SEED0 + 31 * m)
        h = DualHandle(variant, inst)
        infeasible = 0.25 + 0.125 * np.arange(m)
        warm = 0.5 + 0.25 * np.arange(m)
        warm[::2] = 0.0                                   # on the lower bound
        for ftol_rel, maxeval, hi, c0, y0 in ((1e-14, 2000, np.inf, inst["c0"], np.zeros(m)),
                                              (1e-6, 2000, 1e40, infeasible, np.zeros(m)),
                                              (1e-14, 7, np.inf, inst["c0"], np.zeros(m)),
                                              (1e-14, 2000, 1e40, infeasible, warm)):
            h.set_scalars(inst["f0"], inst["rho"], c0, inst["rhoc"])
            lo, hiv = np.zeros(m), np.full(m, hi)
            a, b = (_solve(h, f, y0, lo, hiv, ftol_rel, maxeval) for f in (1, 0))
            assert _same(a, b), (m, ftol_rel, maxeval, hi, a["result"], b["result"], a["nevals"], b["nevals"])
            assert a["result"] in (3, 4, 5) and a["nevals"] >= 2
        bad = np.zeros(m)
        bad[m - 1] = -1.0                                 # below lo = 0
        for f in (1, 0):
            r = _solve(h, f, bad, np.zeros(m), np.full(m, np.inf), 1e-14, 2000)
            assert r["result"] == -2 and H.bits(r["y"]) == H.bits(bad)
            assert r["nevals"] == 1, (m, f, r["nevals"])  # the final evaluation at y0 only
        assert h.query("maxm") >= m


# ---- whole runs: the persistent kernel against the host-driven loop at the m the stop-rule test of test_gpu_parity.py
# leaves out (it runs m = 4) -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", [ob.MMA, ob.CCSAQ])
@pytest.mark.parametrize("opts", [dict(dual_ftol_rel=1e-6), dict(dual_xtol_rel=1e-5), dict(dual_xtol_abs=1e-7, dual_ftol_rel=0.0),
                                  dict(dual_maxeval=7), dict(dual_ftol_abs=1e-9), dict(dual_maxeval=1)])
@pytest.mark.parametrize("m", [3, 5, 8, 13, 16])
def test_fused_run_stop_rules_equal_host_driven_at_every_maxm(built, m, variant, opts):
    """test_gpu_parity.py::test_fused_solve_stop_rules_equal_host_driven at m < MAXM (3, 5, 13) and m = MAXM (8, 16):
    whole runs with the persistent kernel (TMA-staged and register form) and with one launch per evaluation are
    bit-identical, and follow the oracle to the end-to-end tolerance.  (MMA with m > 8 always takes the host loop.)"""
    alg = nl.LD_MMA if variant == ob.MMA else nl.LD_CCSAQ
    n = 30000
    cons = [P.lin_constraint(k, n) for k in range(m)]
    lb, ub = np.full(n, -2.0), np.full(n, 2.0)
    trio = [_run(alg, n, P.rosen_f, cons, [1e-8] * m, lb, ub, P.rosen_x0(n), maxeval=12, b200_fused_solve=f,
                 b200_solve_tma=t, **opts) for f, t in ((1, 1), (1, 0), (0, 0))]
    a = trio[0]
    for r in trio[1:]:
        assert a["ret"] == r["ret"] and a["numevals"] == r["numevals"] and a["minf"] == r["minf"]
        assert np.array_equal(a["x"], r["x"])
        assert a["opt"].get_stats()["dual_evals"] == r["opt"].get_stats()["dual_evals"]
    ref = ob.port_minimize(variant, P.rosen_f, cons, [1e-8] * m, lb, ub, P.rosen_x0(n), maxeval=12, **opts)
    assert a["ret"] == ref["ret"] and a["numevals"] == ref["numevals"]
    assert abs(a["minf"] - ref["minf"]) <= 1e-6 * abs(ref["minf"])
