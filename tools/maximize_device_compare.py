"""Config 4 (synthetic SIMP compliance + volume inequality mean(x) <= 0.4, box [1e-3, 1]^n, x on the device), LD_MMA:
a maximisation of Negated<SimpDev> (problems.cu) against the minimisation of SimpDev.  Both runs take the same points;
the max run adds one negate_kernel launch per gradient evaluation (16 bytes per variable) and a scalar negation.

Timed runs: a fixed maxeval, the two arms alternated, `--repeats` runs each; wall time of nlopt_b200_optimize_device
up to a device synchronisation.  Profiled run (separate, after the timed ones): torch.profiler with CUDA activities,
device time of negate_kernel per evaluation in the max arm.  Both arms must end in opt_f bits that are each other's
negation and in the same counts; the card's name and power limit are read in the same process.

    python tools/maximize_device_compare.py --sizes 1000000 10000000 --repeats 3
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
from nlopt_b200.problems import Problem  # noqa: E402

ARMS = ("min", "max")
SEED, EPS, VOL = 0x5EED0000, 1e-3, 0.4


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"unknown ({e})"


def setup(n, arm, maxeval):
    import torch
    p = Problem()
    o = nl.opt(nl.LD_MMA, n)
    o.set_lower_bounds(1e-3)
    o.set_upper_bounds(1.0)
    o.set_maxeval(maxeval)
    (p.set_simp_device_max if arm == "max" else p.set_simp_device)(o, SEED, EPS)
    p.add_mean_device(o, -VOL, 0.0)
    x = torch.full((n,), VOL, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    return p, o, x


def timed(n, arm, maxeval):
    import torch
    p, o, x = setup(n, arm, maxeval)
    t0 = time.perf_counter()
    o.optimize_device(x.data_ptr())
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    f = o.last_optimum_value()
    if arm == "max":
        f = -f                  # compared with the min arm's f*
    st = o.get_stats()
    return {"arm": arm, "n": n, "ret": o.last_optimize_result(), "wall_s": round(wall, 4), "evals": o.get_numevals(),
            "dual_evals": st["dual_evals"], "kernel_launches": st["kernel_launches"],
            "f_star_bits": np.float64(f).view(np.uint64).item()}


def profiled(n, maxeval):
    """device time of negate_kernel per evaluation in the max arm, and its launches per evaluation"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    p, o, x = setup(n, "max", maxeval)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        o.optimize_device(x.data_ptr())
        torch.cuda.synchronize()
    evals = o.get_numevals()
    us, launches = 0.0, 0
    for e in prof.key_averages():
        if "negate_kernel" in e.key:
            us += e.device_time_total
            launches += e.count
    per_launch = us / launches if launches else float("nan")
    return {"n": n, "evals": evals, "negate_ms_per_eval": round(us / 1e3 / evals, 4), "negate_launches_per_eval": launches / evals,
            "negate_GB_per_s": round(16.0 * n / (per_launch * 1e-6) / 1e9, 1) if launches else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10**6, 10**7])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--maxeval", type=int, default=30)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for n in a.sizes:
        for arm in ARMS:
            timed(n, arm, 3)                    # warm-up: module load, allocations of this size
        walls, res = {k: [] for k in ARMS}, {k: set() for k in ARMS}
        for _ in range(a.repeats):
            for arm in ARMS:
                r = timed(n, arm, a.maxeval)
                walls[arm].append(r["wall_s"])
                res[arm].add((r["ret"], r["evals"], r["dual_evals"], r["f_star_bits"]))
                print(json.dumps(r), flush=True)
        prof = profiled(n, a.maxeval)
        print(json.dumps(prof), flush=True)
        print(json.dumps({"n": n, "median_wall_s": {k: float(np.median(v)) for k, v in walls.items()},
                          "max_over_min_wall": float(np.median(walls["max"]) / np.median(walls["min"])),
                          "negate_ms_per_eval": prof["negate_ms_per_eval"],
                          "same_counts_and_f_star_bits": len(res["min"] | res["max"]) == 1}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
