"""SIMP compliance with a volume EQUALITY under NLOPT_LD_AUGLAG over MMA: __device__ functors with x on the device
against problems.cu's C host callbacks (nb200p_simp_host, nb200p_mean_host registered as an equality) with host x.

The two arms run alternately, `--repeats` times per size.  Each run prints one JSON line: wall seconds, evaluations,
seconds in callbacks, f, h(x*) and the statistics of the last sub-run (nlopt_b200_get_stats after an AUGLAG run: its
dual solves, outer iterations and PCIe bytes).  The card's name and power limit are read in the same process.

    python tools/auglag_device_compare.py --sizes 1000000 10000000 --repeats 3
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

SEED, EPS, VOL, LB, UB, X0 = 0x5EED0000, 1e-3, 0.4, 1e-3, 1.0, 0.4


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError) as e:
        return f"unknown ({e})"


def run(n, arm, maxeval, tol):
    import torch
    p = Problem()
    o = nl.opt(nl.LD_AUGLAG, n)
    o.set_lower_bounds(LB)
    o.set_upper_bounds(UB)
    o.set_ftol_rel(1e-8)
    o.set_maxeval(maxeval)
    subs = [0]
    if arm == "device":
        p.simp_device_eq(o, SEED, EPS, VOL, tol)
        x = torch.full((n,), X0, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        p.reset_callback_seconds()
        t0 = time.perf_counter()
        o.optimize_device(x.data_ptr())
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        h = float(x.mean().item()) - VOL
    else:
        p.simp_host_eq(o, SEED, EPS, VOL, tol)
        x = np.full(n, X0)
        p.reset_callback_seconds()
        t0 = time.perf_counter()
        o.optimize_inplace(x)
        wall = time.perf_counter() - t0
        h = float(np.mean(x)) - VOL
    st = o.get_stats()
    return {"arm": arm, "n": n, "ret": o.last_optimize_result(), "wall_s": round(wall, 4), "evals": o.get_numevals(),
            "f": o.last_optimum_value(), "h": h,
            # host arm: time inside the C callbacks; device arm: time inside the callback launchers (enqueue + finish)
            "callback_s": round(p.callback_seconds() if arm == "host" else st["seconds_callbacks"], 4),
            "last_sub": {k: st[k] for k in ("dual_solves", "outer_iters", "h2d_bytes", "d2h_bytes", "seconds_total")}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[10**6, 10**7])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--maxeval", type=int, default=200)
    ap.add_argument("--tol", type=float, default=1e-6)
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for n in a.sizes:
        run(n, "device", 3, a.tol)              # warm-up: module load, allocations of this size
        run(n, "host", 3, a.tol)
        walls = {"device": [], "host": []}
        for _ in range(a.repeats):
            for arm in ("device", "host"):
                r = run(n, arm, a.maxeval, a.tol)
                walls[arm].append(r["wall_s"])
                print(json.dumps(r), flush=True)
        print(json.dumps({"n": n, "median_wall_s": {k: float(np.median(v)) for k, v in walls.items()},
                          "speedup": float(np.median(walls["host"]) / np.median(walls["device"]))}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
