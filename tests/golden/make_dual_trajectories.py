"""Generate tests/golden/reference_dual_trajectories.json by running the UNMODIFIED reference (oracle/_ref, built from
the reference sources by oracle/Makefile) on every case of tests/dual_trajectories.py.  Commit the JSON; the tests
compare against it without the reference.

    python tests/golden/make_dual_trajectories.py

For each case the reference's own dual optimiser is set up through the public API exactly as mma.c:248-253 and
optimize.c:818-826 configure `dual_opt`: nlopt_create(NLOPT_LD_MMA, m), the min objective F, the box [lo, hi],
stopval -HUGE_VAL, ftol_rel, ftol_abs, xtol_rel, xtol_abs1 and maxeval.  Stored per case: the case parameters; the
result code, the number of evaluations, minf and the final y (hex floats); and a sha256 of the trajectory's bits
(dual_trajectories.fingerprint).  The trajectories themselves are not stored: the tests regenerate them with the
oracle port and check the fingerprint.
"""
import ctypes as C
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
sys.path.insert(0, ROOT)
sys.path.insert(0, TESTS)
import numpy as np  # noqa: E402

import dual_trajectories as DT  # noqa: E402
import nlopt_b200 as nl  # noqa: E402
import oracle_bindings as ob  # noqa: E402
from nlopt_b200 import Library  # noqa: E402

OUT = os.path.join(HERE, "reference_dual_trajectories.json")


def reference_run(lib, case):
    F, y0, lo, hi = DT.problem(case)
    m, stop = case["m"], case["stop"]
    rec = DT.Recorder(F, m)
    o = nl.opt(nl.LD_MMA, m, library=lib)
    o.set_min_objective(lambda y, grad: rec(y, grad))
    o.set_lower_bounds(lo)
    o.set_upper_bounds(hi)
    o.set_stopval(-np.inf)
    o.set_ftol_rel(stop["ftol_rel"])
    o.set_ftol_abs(stop["ftol_abs"])
    o.set_xtol_rel(stop["xtol_rel"])
    o.set_xtol_abs(float(stop["xtol_abs"]))
    o.set_maxeval(stop["maxeval"])
    y = np.array(y0, dtype=np.float64)
    minf = C.c_double(0.0)
    ret = lib.nlopt_optimize(o._h, y.ctypes.data_as(C.POINTER(C.c_double)), C.byref(minf))
    assert o._exc is None, o._exc
    ys, fs, gs = rec.arrays()
    return dict(ret=int(ret), nevals=len(fs), minf=minf.value.hex(), y=DT.hexs(y), sha256=DT.fingerprint(ys, fs, gs))


def main():
    assert os.path.exists(ob.REF_SO), "build oracle/_ref first (python __graft_entry__.py with the reference sources)"
    lib = Library(ob.REF_SO, extensions=False)
    cases = []
    for case in DT.catalogue():
        r = reference_run(lib, case)
        cases.append(dict(case=case, **r))
    with open(OUT, "w") as f:
        json.dump(dict(cases=cases), f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"{len(cases)} cases, {sum(c['nevals'] for c in cases)} evaluations -> {OUT}")


if __name__ == "__main__":
    main()
