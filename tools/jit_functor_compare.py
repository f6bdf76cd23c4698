"""Config 4 (synthetic SIMP compliance + volume inequality mean(x) <= 0.4, box [1e-3, 1]^n, x on the device), LD_MMA, in
three arms:

  functor  problems.cu's SimpDev + MeanDev, __device__ functors built by nvcc (nlopt_b200_device.cuh)
  jit      the same functors as source (tests/jit_twins.py), compiled at run time by nlopt_b200.CudaFunctor
  torch    PyTorch terms callbacks with the functors' operation order (set_min_objective_torch /
           add_inequality_constraint_torch)

First the compile times of the jit arm: the first CudaFunctor of each functor (NVRTC) and a second one of the same
source (the per-process cache).  Timed runs: a fixed maxeval, the arms alternated, `--repeats` runs each; wall time of
the optimisation up to a device synchronisation.  Profiled runs (separate, after the timed ones): torch.profiler with
CUDA activities, device time per evaluation of the map_group* / fold_groups* kernels and of every kernel the callbacks
of a point cause.  The three arms must end in the same counts and f* bits; the card's name and power limit are read in
the same process.

    python tools/jit_functor_compare.py --sizes 1000000 10000000 --repeats 3
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import jit_twins  # noqa: E402
import nlopt_b200 as nl  # noqa: E402
import synth  # noqa: E402
from nlopt_b200.problems import Problem  # noqa: E402
from terms_callback_compare import LIBRARY_KERNELS, card  # noqa: E402

ARMS = ("functor", "jit", "torch")
SEED, EPS, VOL = 0x5EED0000, 1e-3, 0.4


def compile_times():
    out = {}
    for name in ("SimpDev", "MeanDev"):
        t0 = time.perf_counter()
        nl.CudaFunctor(jit_twins.SOURCE, "twin::" + name)
        t1 = time.perf_counter()
        nl.CudaFunctor(jit_twins.SOURCE, "twin::" + name)
        t2 = time.perf_counter()
        out[name] = {"first_compile_s": round(t1 - t0, 4), "cached_s": round(t2 - t1, 6)}
    return out


class Arms:
    def __init__(self, n):
        import torch
        self.n = n
        self.p = Problem()
        self.a_t = torch.from_numpy(0.5 + synth.u01(0, n, SEED)).cuda()
        self.simp, self.mean = jit_twins.functor("SimpDev"), jit_twins.functor("MeanDev")

    def register(self, o, arm):
        import torch
        ome, inv_n = 1.0 - EPS, 1.0 / self.n
        if arm == "functor":
            self.p.set_simp_device(o, SEED, EPS)
            self.p.add_mean_device(o, -VOL, 0.0)
        elif arm == "jit":
            o.set_min_objective_cuda(self.simp, jit_twins.simp(SEED, EPS))
            o.add_inequality_constraint_cuda(self.mean, jit_twins.two_doubles(inv_n, -VOL), 0.0,
                                             finish=lambda s: s * inv_n + -VOL)
        else:
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
    return {"arm": arm, "n": arms.n, "ret": o.last_optimize_result(), "wall_s": round(wall, 4), "evals": o.get_numevals(),
            "dual_evals": o.get_stats()["dual_evals"], "f_star_bits": np.float64(o.last_optimum_value()).view(np.uint64).item()}


def profiled(arms, arm, maxeval):
    """device time per evaluation: the map / fold kernels, and every kernel the callbacks of a point cause"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    o, x = arms.make(arm, maxeval)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        o.optimize_torch(x)
        torch.cuda.synchronize()
    evals = o.get_numevals()
    cb_us, map_fold_us, kernels = 0.0, 0.0, {}
    for e in prof.key_averages():
        if e.device_time_total <= 0 or any(k in e.key for k in LIBRARY_KERNELS) or "Memcpy" in e.key or "Memset" in e.key:
            continue
        cb_us += e.device_time_total
        kernels[e.key[:80]] = round(e.device_time_total / 1e3 / evals, 4)
        if "map_group" in e.key or "fold_groups" in e.key:
            map_fold_us += e.device_time_total
    return {"arm": arm, "n": arms.n, "evals": evals, "map_fold_ms_per_eval": round(map_fold_us / 1e3 / evals, 4),
            "callback_kernels_ms_per_eval": round(cb_us / 1e3 / evals, 4), "kernels_ms_per_eval": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10**6, 10**7])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--maxeval", type=int, default=30)
    ap.add_argument("--arms", nargs="+", default=list(ARMS))
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    print(json.dumps({"compile": compile_times()}), flush=True)
    for n in a.sizes:
        arms = Arms(n)
        for arm in a.arms:
            timed(arms, arm, 3)                 # warm-up: module load, allocations of this size
        walls, res = {k: [] for k in a.arms}, {k: set() for k in a.arms}
        for _ in range(a.repeats):
            for arm in a.arms:
                r = timed(arms, arm, a.maxeval)
                walls[arm].append(r["wall_s"])
                res[arm].add((r["ret"], r["evals"], r["dual_evals"], r["f_star_bits"]))
                print(json.dumps(r), flush=True)
        profs = {arm: profiled(arms, arm, a.maxeval) for arm in a.arms}
        for p in profs.values():
            print(json.dumps(p), flush=True)
        med = {k: float(np.median(v)) for k, v in walls.items()}
        print(json.dumps({"n": n, "median_wall_s": med, "min_max_wall_s": {k: [min(v), max(v)] for k, v in walls.items()},
                          "over_functor": {k: round(v / med["functor"], 3) for k, v in med.items()} if "functor" in med else None,
                          "map_fold_ms_per_eval": {k: p["map_fold_ms_per_eval"] for k, p in profs.items()},
                          "callback_kernels_ms_per_eval": {k: p["callback_kernels_ms_per_eval"] for k, p in profs.items()},
                          "same_counts_and_f_star_bits": len(set().union(*res.values())) == 1}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
