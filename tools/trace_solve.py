"""Timeline of the persistent dual-solve kernel: where does one generation (= one dual evaluation) spend its
time?  Builds an instrumented copy of the library (-DNB200_TRACE, build/trace/) and runs bench.py's
device-resident arm against it with NLOPT_B200_TRACE_FILE set (NLOPT_B200_LIBDIR, when set, picks another
-DNB200_TRACE build, e.g. one from tools/ab_build.py).  For the TMA-staged form it also prints the generation boundary:
tail spread of the CTAs' last records, the folder's hand-off, publication -> first consumer, and how long producers sat
parked on a full ring.  Usage:
    python tools/trace_solve.py build            # here (no GPU needed)
    python tools/trace_solve.py run N [alg]      # on a GPU; prints a summary of build/trace_{alg}_N.txt"""
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402

TDIR = os.path.join(ROOT, "build", "trace")


def build():
    os.makedirs(TDIR, exist_ok=True)
    cuda_home = os.path.dirname(os.path.dirname(G.NVCC))
    G.write_jit_headers(os.path.join(G.BUILD, "jit_headers.inc"))
    objs = []
    for src in G.LIB_SOURCES_CU:
        obj = os.path.join(TDIR, src + ".o")
        G._run([G.NVCC, *G.ARCH, *G.NVCC_FLAGS, "-DNB200_TRACE", "-c", os.path.join(G.CSRC, src), "-o", obj])
        objs.append(obj)
    for src in G.LIB_SOURCES_CXX:
        obj = os.path.join(TDIR, src + ".o")
        extra = ["-I" + G.BUILD, f'-DNLOPT_B200_CUDA_LIB64="{cuda_home}/lib64"'] if src == "jit.cpp" else []      # as in build_library
        G._run(["g++", *G.CXX_FLAGS, *extra, f"-I{cuda_home}/include", "-c", os.path.join(G.CSRC, src), "-o", obj])
        objs.append(obj)
    lib = os.path.join(TDIR, "libnlopt_b200.so")
    G._run([G.NVCC, *G.ARCH, "-shared", "-o", lib, *objs, "-cudart", "shared", "-ldl", "-Xlinker", "-soname,libnlopt_b200.so",
            "-Xlinker", "-Bsymbolic-functions"])
    G._run([G.NVCC, *G.ARCH, *G.NVCC_FLAGS, "-shared", os.path.join(G.CSRC, "problems.cu"), "-o",
            os.path.join(TDIR, "libnlopt_b200_problems.so"), "-cudart", "shared", "-L" + TDIR, "-lnlopt_b200", "-Xlinker", "-rpath=$ORIGIN"])
    print("built", lib)


def run(n, alg="ccsaq", extra=()):
    out = os.path.join(ROOT, "build", f"trace_{alg}_{n}.txt")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if os.path.exists(out):
        os.remove(out)
    env = dict(os.environ, NLOPT_B200_TRACE_FILE=out)
    env.setdefault("NLOPT_B200_LIBDIR", TDIR)        # or another -DNB200_TRACE build (tools/ab_build.py)
    subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--n", str(n), "--alg", alg, "--steps", "4", "--warmup", "2",
                    "--no-cpu", "--no-e2e", *extra], env=env, check=True, stdout=subprocess.DEVNULL)
    rows = []
    head = ""
    for line in open(out):
        if line.startswith("solve"):
            head = line.strip()
        if not line.lstrip().startswith("gen "):
            continue
        r = {f"{k}_lo": int(lo) for k, lo, _ in re.findall(r"(\w+)\[(-?\d+)\.\.(-?\d+)\]", line)}
        r.update({f"{k}_hi": int(hi) for k, _, hi in re.findall(r"(\w+)\[(-?\d+)\.\.(-?\d+)\]", line)})
        r.update({k: int(v) for k, v in re.findall(r"(\w+) (-?\d+)(?= |$)", line.split("|")[0])})
        r["sweep"] = int(re.search(r"mean_group_sweep (\d+)", line).group(1))
        if r.get("next_pub", 0) > 0:
            rows.append(r)
    print(head)
    print(f"n={n} {alg}: {len(rows)} generations; medians in ns after the generation was published:")
    for k in ("seen_lo", "seen_hi", "recs_lo", "recs_hi", "rank_done", "totals", "machine", "next_pub", "sweep",
              "lastrec_lo", "lastrec_hi", "parked_lo", "parked_hi"):
        v = [r[k] for r in rows if k in r]
        print(f"  {k:10s} {statistics.median(v) if v else -1:9.0f}")
    # the TMA-staged form's boundary (rows whose generation saw parked producers); every figure is per generation
    tma = [r for r in rows if r.get("parked_hi", 0) != 0 and r.get("lastrec_hi", 0) > 0]
    if tma:
        parts = {
            "tail spread (first -> last CTA's last record)": [r["lastrec_hi"] - r["lastrec_lo"] for r in tma],
            "last record -> fold end (all shard sums in)": [r["rank_done"] - r["recs_hi"] for r in tma],
            "fold end -> publication of the next": [r["next_pub"] - r["rank_done"] for r in tma],
            "publication -> first consumer start": [r["seen_lo"] for r in tma],
            "first -> last consumer start": [r["seen_hi"] - r["seen_lo"] for r in tma],
            "HBM under-fed (first producer parked -> first consumer start)": [r["seen_lo"] - r["parked_lo"] for r in tma],
            "all producers parked -> first consumer start": [r["seen_lo"] - r["parked_hi"] for r in tma],
            "generation (publication -> next publication)": [r["next_pub"] for r in tma],
        }
        print(f"TMA-staged boundary, {len(tma)} generations; per-generation medians in ns (parked: row of the generation waited for):")
        for k, v in parts.items():
            print(f"  {k:64s} {statistics.median(v):9.0f}")


if __name__ == "__main__":
    if sys.argv[1] == "build":
        build()
    else:
        run(int(float(sys.argv[2])), *(sys.argv[3:4] or ["ccsaq"]), extra=sys.argv[4:])
