"""Config 4 (synthetic SIMP compliance + volume inequality mean(x) <= 0.4, box [1e-3, 1]^n, x on the device), LD_MMA, in
four arms:

  functor  problems.cu's SimpDev + MeanDev as __device__ functors (nlopt_b200_device.cuh)
  cterms   the same functors called once per variable by C terms callbacks (nlopt_b200_dtfunc,
           tests/cpp/terms_callback_probe.cu, compiled here into a temporary directory)
  torch    PyTorch terms callbacks with the functors' operation order (set_min_objective_torch /
           add_inequality_constraint_torch)
  numpy    numpy host callbacks (what a PyTorch user without the terms path writes)

Timed runs: a fixed maxeval, the arms alternated, `--repeats` runs each; wall time of the optimisation up to a device
synchronisation.  Profiled runs (separate, after the timed ones): torch.profiler with CUDA activities, device time of
every kernel the callbacks of a point cause, per evaluation, and terms_group_kernel's HBM rate against its byte model
(8 n m bytes of terms read + 16 groups m of group sums, per launch; m = 1 here).  The first three arms must end in the
same counts and f* bits; the card's name and power limit are read in the same process.

    python tools/terms_callback_compare.py --sizes 1000000 10000000 --repeats 3
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import nlopt_b200 as nl  # noqa: E402
import synth  # noqa: E402
from nlopt_b200 import _capi  # noqa: E402
from nlopt_b200.problems import Problem  # noqa: E402

ARMS = ("functor", "cterms", "torch", "numpy")
SEED, EPS, VOL = 0x5EED0000, 1e-3, 0.4
# the kernels of the library's dual solve and outer loop; everything else in a trace is caused by the callbacks
LIBRARY_KERNELS = ("dual_", "sigma_", "end_outer", "fill_kernel", "publish", "penalty_axpy", "negate_kernel")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"unknown ({e})"


def build_probe(tmp):
    import __graft_entry__ as g
    so = os.path.join(tmp, "libterms_callback_probe.so")
    flags = [f for f in g.NVCC_FLAGS if f not in ("--fmad=false", "-Xptxas", "-v")] + ["--fmad=false"]
    subprocess.run([g.NVCC, *g.ARCH, *flags, "-shared", os.path.join(ROOT, "tests", "cpp", "terms_callback_probe.cu"), "-o", so,
                    "-cudart", "shared", "-L" + os.path.dirname(g.LIB), "-lnlopt_b200", "-Xlinker", "-rpath=" + os.path.dirname(g.LIB)],
                   check=True, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    _capi.default_library()
    L = C.CDLL(so, mode=C.RTLD_LOCAL)
    L.probe_terms_register.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


class Arms:
    def __init__(self, probe, n):
        import torch
        self.probe, self.n = probe, n
        self.p = Problem()
        a = 0.5 + synth.u01(0, n, SEED)
        self.a_np = a
        self.a_t = torch.from_numpy(a).cuda()
        self.keep = []

    def register(self, o, arm):
        import torch
        n, ome, inv_n = self.n, 1.0 - EPS, 1.0 / self.n
        if arm == "functor":
            self.p.set_simp_device(o, SEED, EPS)
            self.p.add_mean_device(o, -VOL, 0.0)
        elif arm == "cterms":
            pe, pm = np.array([EPS]), np.array([-VOL])
            self.keep += [pe, pm]
            o._check(self.probe.probe_terms_register(o._h, 0, 0, 1, SEED, pe.ctypes.data, None, None))
            o._check(self.probe.probe_terms_register(o._h, 1, 2, 1, SEED, pm.ctypes.data, None, None))
        elif arm == "torch":
            a = self.a_t

            def simp(x, g):
                x2 = x * x
                x3 = x2 * x
                d = EPS + ome * x3
                if g.numel():
                    g.copy_(-(((a * (ome * 3.0)) * x2) / (d * d)))
                return a / d

            def mean(x, g):
                if g.numel():
                    g.fill_(inv_n)
                return x

            o.set_min_objective_torch(simp)
            o.add_inequality_constraint_torch(mean, 0.0, finish=lambda s: s * inv_n - VOL)
        else:
            a = self.a_np

            def simp(x, g):
                x2 = x * x
                x3 = x2 * x
                d = EPS + ome * x3
                if g.size:
                    g[:] = -(((a * (ome * 3.0)) * x2) / (d * d))
                return float(np.sum(a / d))

            def mean(x, g):
                if g.size:
                    g[:] = inv_n
                return float(np.sum(x)) * inv_n - VOL

            o.set_min_objective(simp)
            o.add_inequality_constraint(mean, 0.0)
        torch.cuda.synchronize()

    def make(self, arm, maxeval):
        import torch
        o = nl.opt(nl.LD_MMA, self.n)
        o.set_lower_bounds(1e-3)
        o.set_upper_bounds(1.0)
        o.set_maxeval(maxeval)
        self.register(o, arm)
        x = torch.full((self.n,), VOL, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        return o, x


def timed(arms, arm, maxeval):
    import torch
    o, x = arms.make(arm, maxeval)
    t0 = time.perf_counter()
    o.optimize_torch(x)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    st = o.get_stats()
    return {"arm": arm, "n": arms.n, "ret": o.last_optimize_result(), "wall_s": round(wall, 4), "evals": o.get_numevals(),
            "dual_evals": st["dual_evals"], "f_star_bits": np.float64(o.last_optimum_value()).view(np.uint64).item()}


def profiled(arms, arm, maxeval):
    """device time per evaluation of the kernels the callbacks cause, and terms_group_kernel's rate"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    o, x = arms.make(arm, maxeval)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        o.optimize_torch(x)
        torch.cuda.synchronize()
    evals = o.get_numevals()
    cb_us, terms_us, terms_launches, kernels = 0.0, 0.0, 0, {}
    for e in prof.key_averages():
        if e.device_time_total <= 0 or any(k in e.key for k in LIBRARY_KERNELS) or "Memcpy" in e.key or "Memset" in e.key:
            continue
        cb_us += e.device_time_total
        kernels[e.key[:80]] = round(e.device_time_total / 1e3 / evals, 4)
        if "terms_group_kernel" in e.key:
            terms_us += e.device_time_total
            terms_launches += e.count
    out = {"arm": arm, "n": arms.n, "evals": evals, "callback_kernels_ms_per_eval": round(cb_us / 1e3 / evals, 4),
           "kernels_ms_per_eval": kernels}
    if terms_launches:
        from test_device_callbacks_gpu import geometry
        model_bytes = 8.0 * arms.n + 16.0 * geometry(arms.n).groups_total
        per = terms_us / terms_launches * 1e-6
        out.update({"terms_kernel_ms_per_launch": round(per * 1e3, 4), "terms_model_bytes": model_bytes,
                    "terms_GB_per_s": round(model_bytes / per / 1e9, 1)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10**6, 10**7])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--maxeval", type=int, default=30)
    ap.add_argument("--arms", nargs="+", default=list(ARMS))
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        probe = build_probe(tmp)
        for n in a.sizes:
            arms = Arms(probe, n)
            for arm in a.arms:
                timed(arms, arm, 3)                 # warm-up: module load, allocations of this size
            walls, res = {k: [] for k in a.arms}, {k: set() for k in a.arms}
            for _ in range(a.repeats):
                for arm in a.arms:
                    r = timed(arms, arm, a.maxeval)
                    walls[arm].append(r["wall_s"])
                    res[arm].add((r["ret"], r["evals"], r["dual_evals"], r["f_star_bits"]))
                    print(json.dumps(r), flush=True)
            profs = {arm: profiled(arms, arm, a.maxeval) for arm in a.arms if arm != "numpy"}
            for p in profs.values():
                print(json.dumps(p), flush=True)
            device_arms = [k for k in ("functor", "cterms", "torch") if k in a.arms]
            med = {k: float(np.median(v)) for k, v in walls.items()}
            print(json.dumps({"n": n, "median_wall_s": med,
                              "over_functor": {k: round(v / med["functor"], 3) for k, v in med.items()} if "functor" in med else None,
                              "callback_kernels_ms_per_eval": {k: p["callback_kernels_ms_per_eval"] for k, p in profs.items()},
                              "same_counts_and_f_star_bits": len(set().union(*(res[k] for k in device_arms))) == 1}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
