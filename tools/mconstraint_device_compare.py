"""Config 3 (chained Rosenbrock + m dense linear inequality rows, box [-2, 2]^n, x on the device): m scalar LinearDev
functors against one vector LinearRowsDev<m>, which computes the same rows in one pass over x.

Timed runs: a fixed maxeval, the two arms alternated, `--repeats` runs each; wall time of nlopt_b200_optimize_device
up to a device synchronisation.  Profiled runs (separate, after the timed ones): torch.profiler with CUDA activities,
device time of the callback kernels (names containing map_group / fold_groups) per evaluation.  Both arms must end in
the same bits of opt_f; the card's name and power limit are read in the same process.

    python tools/mconstraint_device_compare.py --sizes 1000000 10000000 --ms 4 16 --repeats 3
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import nlopt_b200 as nl  # noqa: E402
from nlopt_b200.problems import Problem, rosen_x0  # noqa: E402

ARMS = ("scalar", "vector")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"unknown ({e})"


def setup(n, m, arm, maxeval, alg):
    import torch
    p = Problem()
    o = nl.opt(alg, n)
    o.set_lower_bounds(-2.0)
    o.set_upper_bounds(2.0)
    o.set_maxeval(maxeval)
    (p.rosenbrock_device if arm == "scalar" else p.rosenbrock_device_rows)(o, m)
    x = torch.from_numpy(rosen_x0(n)).cuda()
    torch.cuda.synchronize()
    return p, o, x


def timed(n, m, arm, maxeval, alg):
    import torch
    p, o, x = setup(n, m, arm, maxeval, alg)
    t0 = time.perf_counter()
    o.optimize_device(x.data_ptr())
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    f = o.last_optimum_value()
    return {"arm": arm, "n": n, "m": m, "ret": o.last_optimize_result(), "wall_s": round(wall, 4), "evals": o.get_numevals(),
            "dual_evals": o.get_stats()["dual_evals"], "opt_f": f, "opt_f_bits": np.float64(f).view(np.uint64).item()}


def profiled(n, m, arm, maxeval, alg):
    """device seconds of the callback kernels per evaluation, and their launch count per evaluation"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    p, o, x = setup(n, m, arm, maxeval, alg)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        o.optimize_device(x.data_ptr())
        torch.cuda.synchronize()
    evals = o.get_numevals()
    us, launches = 0.0, 0
    for e in prof.key_averages():
        if "map_group" in e.key or "fold_groups" in e.key:
            us += e.device_time_total
            launches += e.count
    return {"arm": arm, "n": n, "m": m, "evals": evals, "callback_kernel_ms_per_eval": round(us / 1e3 / evals, 4),
            "callback_launches_per_eval": launches / evals}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10**6, 10**7])
    ap.add_argument("--ms", type=int, nargs="+", default=[4, 16])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--maxeval", type=int, default=20)
    ap.add_argument("--alg", choices=["mma", "ccsaq"], default="ccsaq")
    a = ap.parse_args()
    alg = nl.LD_CCSAQ if a.alg == "ccsaq" else nl.LD_MMA
    print(json.dumps({"card": card()}), flush=True)
    for n in a.sizes:
        for m in a.ms:
            for arm in ARMS:
                timed(n, m, arm, 3, alg)            # warm-up: module load, allocations of this size
            walls, bits = {k: [] for k in ARMS}, {k: set() for k in ARMS}
            for _ in range(a.repeats):
                for arm in ARMS:
                    r = timed(n, m, arm, a.maxeval, alg)
                    walls[arm].append(r["wall_s"])
                    bits[arm].add(r["opt_f_bits"])
                    print(json.dumps(r), flush=True)
            prof = {arm: profiled(n, m, arm, a.maxeval, alg) for arm in ARMS}
            for r in prof.values():
                print(json.dumps(r), flush=True)
            print(json.dumps({"n": n, "m": m, "median_wall_s": {k: float(np.median(v)) for k, v in walls.items()},
                              "vector_speedup_wall": float(np.median(walls["scalar"]) / np.median(walls["vector"])),
                              "callback_kernel_ms_per_eval": {k: prof[k]["callback_kernel_ms_per_eval"] for k in ARMS},
                              "opt_f_bits_equal": len(bits["scalar"] | bits["vector"]) == 1}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
