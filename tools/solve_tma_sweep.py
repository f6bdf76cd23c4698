"""The persistent dual-solve kernel on one GPU: register form (b200_solve_tma=0) against the TMA-staged form
(b200_solve_tma=1), on bench.py's c3 problem (chained Rosenbrock + m dense linear constraints, __device__ callbacks,
box [-2, 2]^n) for n x m x algorithm, with the box given as two scalars (the kernels read 3 + m arrays) and as two
arrays (5 + m).  One point = `--steps` inner iterations after a `--warmup` run, both forms alternated `--reps` times on
fresh objects; reported per form: microseconds of kernel time per dual evaluation (best rep), the HBM rate of the
operand bytes the kernels were asked for (nlopt_b200_stats.dual_operand_bytes over seconds_dual_kernel) and f after the
steps (the forms must agree bit for bit), and whether the TMA form read the sigma index (`tma_index`).  To set the
sigma-index form against the fp64-sigma TMA form, run the sweep again in the same session under
NLOPT_B200_LIBDIR=build/ab/NAME, a build from tools/ab_build.py with -DNB200_SIGMA_INDEX_MIN_MB=1048576 (the register
column then shows the drift between the two runs).  Writes build/solve_tma_sweep.json (--out to change).
    python tools/solve_tma_sweep.py [--n 1.25e6,2.5e6,...] [--m 1,4] [--alg mma,ccsaq] [--bounds scalar,array]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="1.25e6,2.5e6,5e6,1e7,2e7,5e7")
    ap.add_argument("--m", default="1,4")
    ap.add_argument("--alg", default="mma,ccsaq")
    ap.add_argument("--bounds", default="scalar,array")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "build", "solve_tma_sweep.json"))
    a = ap.parse_args()
    import torch
    import nlopt_b200 as nl
    from nlopt_b200.problems import Problem, rosen_x0

    def run(alg, n, m, bounds, tma, x0dev):
        o = nl.opt(nl.LD_CCSAQ if alg == "ccsaq" else nl.LD_MMA, n)
        if bounds == "scalar":
            o.set_lower_bounds(-2.0); o.set_upper_bounds(2.0)
        else:
            o.set_lower_bounds(np.full(n, -2.0)); o.set_upper_bounds(np.full(n, 2.0))
        p = Problem()
        p.rosenbrock_device(o, m)
        o.set_param("b200_time_kernels", 1)
        if not (tma and m == 4 and bounds == "scalar"):   # there the default rule takes the TMA form, with the sigma index
            o.set_param("b200_solve_tma", tma)            # above NB200_SIGMA_INDEX_MIN_MB; the knob would force fp64 sigma
        xdev = x0dev.clone()
        o.set_maxeval(a.warmup + 1)
        o.optimize_device(xdev.data_ptr())
        xdev.copy_(x0dev)
        o.set_maxeval(a.steps + 1)
        o.optimize_device(xdev.data_ptr())
        s = o.get_stats()      # of the last call
        kern = s["seconds_dual_kernel"]
        return dict(us_per_eval=1e6 * kern / max(1, s["dual_evals"]), gbs=s["dual_operand_bytes"] / kern * 1e-9 if kern > 0 else None,
                    dual_evals=s["dual_evals"], f_hex=float(o.last_optimum_value()).hex(), sigma_palette=s["sigma_palette"])

    rows = []
    for alg in a.alg.split(","):
        for m in [int(v) for v in a.m.split(",")]:
            for n in [int(float(v)) for v in a.n.split(",")]:
                x0dev = torch.from_numpy(rosen_x0(n)).cuda()
                for bounds in a.bounds.split(","):
                    res = {0: [], 1: []}
                    for _ in range(a.reps):
                        for tma in (0, 1):
                            res[tma].append(run(alg, n, m, bounds, tma, x0dev))
                    best = {t: min(r, key=lambda v: v["us_per_eval"]) for t, r in res.items()}
                    row = dict(alg=alg, n=n, m=m, bounds=bounds,
                               register_us=best[0]["us_per_eval"], tma_us=best[1]["us_per_eval"],
                               register_gbs=best[0]["gbs"], tma_gbs=best[1]["gbs"],
                               tma_speedup=best[0]["us_per_eval"] / best[1]["us_per_eval"],
                               same_f=len({r["f_hex"] for t in res for r in res[t]}) == 1,
                               same_evals=len({r["dual_evals"] for t in res for r in res[t]}) == 1,
                               tma_index=best[1]["sigma_palette"] > 0,
                               all_us={t: [round(r["us_per_eval"], 2) for r in res[t]] for t in res})
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                del x0dev
    out = a.out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    json.dump(dict(gpu=torch.cuda.get_device_name(0), rows=rows), open(out, "w"), indent=1)
    print("wrote", out)


if __name__ == "__main__":
    main()
