"""Preconditioned CCSAQ, host path against device path, on the tridiagonal problem of tests/test_device_precond_gpu.py.

    host   : numpy callbacks and nlopt_precond, host x and host bounds (run_ccsa_precond)
    device : torch terms callbacks and a torch device preconditioner, x and bounds on the device (model_solve)

Both arms run with the same fixed maxeval and dual_maxeval, alternated, `--reps` times each; per run the line reports wall
time, seconds_callbacks, the bytes moved between host and device, and the final f.  The card's name and power limit are
read in the same run.  The host arm runs with maxtime = --host-budget seconds: a run that reaches it is reported as not
measured, and so are the host arm's later runs at that n.

    python tools/precond_device_compare.py --n 1000000 10000000 --maxeval 10 --dual-maxeval 50
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nlopt_b200 as nl  # noqa: E402


def problem(n, seed=3):
    rng = np.random.default_rng(seed)
    d = 2.5 + rng.random(n)
    b = rng.standard_normal(n)
    w = (1.0 + 0.5 * np.sin(0.37 * np.arange(n))) / n
    return d, b, w


def A(d, v):
    out = d * v
    out[:-1] -= v[1:]
    out[1:] -= v[:-1]
    return out


def configure(o, args):
    o.set_maxeval(args.maxeval)
    o.set_param("dual_maxeval", args.dual_maxeval)
    o.set_param("dual_ftol_rel", 1e-12)


def run_host(n, args):
    d, b, w = problem(n)

    def f(x, g):
        Ax = A(d, x)
        if g.size:
            g[:] = Ax - b
        return float(0.5 * x @ Ax - b @ x)

    def c(x, g):
        if g.size:
            g[:] = w
        return float(w @ x) + 0.05

    o = nl.opt(nl.LD_CCSAQ, n)
    o.set_lower_bounds(np.full(n, -2.0))
    o.set_upper_bounds(np.full(n, 2.0))
    configure(o, args)
    o.set_precond_min_objective(f, lambda x, v, vpre: vpre.__setitem__(slice(None), A(d, v)))
    o.add_inequality_constraint(c, 1e-8)
    o.set_maxtime(args.host_budget)
    t0 = time.perf_counter()
    o.optimize(np.zeros(n))
    return o, time.perf_counter() - t0


def run_device(n, args):
    import torch
    d, b, w = (torch.tensor(a, dtype=torch.float64, device="cuda") for a in problem(n))

    def f(x, g):
        Ax = A(d, x)
        if g.numel():
            g.copy_(Ax - b)
        return 0.5 * x * Ax - b * x

    def c(x, g):
        if g.numel():
            g.copy_(w)
        return w * x

    o = nl.opt(nl.LD_CCSAQ, n)
    o.set_lower_bounds(torch.full((n,), -2.0, dtype=torch.float64, device="cuda"))
    o.set_upper_bounds(torch.full((n,), 2.0, dtype=torch.float64, device="cuda"))
    configure(o, args)
    o.set_min_objective_torch(f)
    o.add_inequality_constraint_torch(c, 1e-8, finish=lambda t: t + 0.05)
    o.set_objective_precond_torch(lambda x, v, vpre: vpre.copy_(A(d, v)))
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    o.optimize_torch(x)
    torch.cuda.synchronize()
    return o, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--maxeval", type=int, default=10)
    ap.add_argument("--dual-maxeval", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-budget", type=float, default=120.0)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card, "maxeval": args.maxeval, "dual_maxeval": args.dual_maxeval}))
    for n in args.n:
        host_ok = True
        for rep in range(args.reps):
            for arm, fn in (("device", run_device), ("host", run_host)):
                if arm == "host" and not host_ok:
                    print(json.dumps({"n": n, "arm": arm, "rep": rep, "result": "not measured (over the time budget)"}))
                    continue
                o, wall = fn(n, args)
                if arm == "host" and o.last_optimize_result() == nl.MAXTIME_REACHED:
                    host_ok = False
                    print(json.dumps({"n": n, "arm": arm, "rep": rep, "result": "not measured (over the time budget)"}))
                    continue
                st = o.get_stats()
                print(json.dumps({"n": n, "arm": arm, "rep": rep, "ret": o.last_optimize_result(), "wall_s": round(wall, 4),
                                  "seconds_callbacks": round(st["seconds_callbacks"], 4),
                                  "h2d_bytes": st["h2d_bytes"], "d2h_bytes": st["d2h_bytes"],
                                  "f": o.last_optimum_value(), "numevals": o.get_numevals()}), flush=True)


if __name__ == "__main__":
    main()
