"""Bounds that a PyTorch program holds on the GPU: handed over through the host (arm "host": `.cpu().numpy()` and the
host setters, what a user had to do before the device setters existed) against the device setters (arm "device":
opt.set_lower_bounds(tensor), nlopt_b200_set_*_bounds_device).

Workload: SIMP compliance with a volume inequality under LD_MMA, __device__ functors, x on the device (optimize_torch),
maxeval 30, and ~3% passive elements (lb == ub: solid 1 or void 1e-3) in a [1e-3, 1] box built by torch on the device.
The arms alternate, `--repeats` times per size.  The timed window is the two setters plus optimize_torch and ends in a
device synchronise.  Each run prints one JSON line with that time, nlopt_b200_stats::seconds_setup and h2d_bytes and f*;
both arms must end with the same bits of f*.  The card's name and power limit are read in the same process.

    python tools/device_bounds_compare.py --sizes 1000000 10000000 --repeats 3 --out device_bounds.jsonl
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


def passive_box(n):
    """lb, ub, x0 on the device: 1 in 33 elements passive (lb == ub == x0)"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(3)
    lb = torch.full((n,), LB, dtype=torch.float64, device="cuda")
    ub = torch.full((n,), UB, dtype=torch.float64, device="cuda")
    x0 = torch.full((n,), X0, dtype=torch.float64, device="cuda")
    k = torch.randperm(n, generator=g, device="cuda")[: n // 33]
    v = torch.where(torch.rand(k.numel(), generator=g, device="cuda") < 0.5, UB, LB).to(torch.float64)
    lb[k] = v
    ub[k] = v
    x0[k] = v
    return lb, ub, x0


def run(n, arm, maxeval, box):
    import torch
    lb, ub, x0 = box
    p = Problem()
    o = nl.opt(nl.LD_MMA, n)
    p.simp_device(o, SEED, EPS, VOL)
    o.set_maxeval(maxeval)
    x = x0.clone()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if arm == "host":
        o.set_lower_bounds(lb.cpu().numpy())
        o.set_upper_bounds(ub.cpu().numpy())
    else:
        o.set_lower_bounds(lb)
        o.set_upper_bounds(ub)
    o.optimize_torch(x)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    st = o.get_stats()
    return dict(n=n, arm=arm, seconds=wall, seconds_setup=st["seconds_setup"], h2d_bytes=st["h2d_bytes"],
                ret=o.last_optimize_result(), numevals=o.get_numevals(), f=o.last_optimum_value(),
                f_bits=int(np.float64(o.last_optimum_value()).view(np.uint64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--maxeval", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if nl.device_count() <= 0:
        sys.exit("device_bounds_compare.py needs a CUDA device")
    out = open(a.out, "w") if a.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out:
            out.write(line + "\n")
            out.flush()

    emit(dict(card=card()))
    for n in a.sizes:
        box = passive_box(n)
        run(n, "device", 2, box)             # warm-up: module load, block cache, both arms' shapes
        run(n, "host", 2, box)
        fbits = set()
        for _ in range(a.repeats):
            for arm in ("host", "device"):
                r = run(n, arm, a.maxeval, box)
                fbits.add(r["f_bits"])
                emit(r)
        if len(fbits) != 1:
            sys.exit(f"n={n}: the arms ended with different f* bits: {sorted(fbits)}")
    emit(dict(card=card()))


if __name__ == "__main__":
    main()
