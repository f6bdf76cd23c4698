"""A/B builds of the library: the same sources with extra -D switches, written to build/ab/NAME/ (libnlopt_b200.so +
libnlopt_b200_problems.so).  A run picks one with NLOPT_B200_LIBDIR=build/ab/NAME (nlopt_b200/_capi.py), so one GPU
session can time several compile-time variants back to back -- no template explosion in the product build.
    python tools/ab_build.py NAME [-DNB200_SOLVE_MINB4=2 ...]        # no GPU needed
Switches in use: NB200_SOLVE_MINB4 (min CTAs/SM of the solve kernel with <= 4 gradient rows, default 3),
NB200_SOLVE_TMA_IDX_STAGES4 (stages of the sigma-index TMA solve kernel with 4 rows, default 3), NB200_SIGMA_PALETTE_CAP
(entries of the sigma palette, default 65535)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402


def build(name, defines):
    out = os.path.join(ROOT, "build", "ab", name)
    os.makedirs(out, exist_ok=True)
    cuda_home = os.path.dirname(os.path.dirname(G.NVCC))
    G.write_jit_headers(os.path.join(G.BUILD, "jit_headers.inc"))
    objs = []
    for src in G.LIB_SOURCES_CU:
        obj = os.path.join(out, src + ".o")
        log = G._run([G.NVCC, *G.ARCH, *G.NVCC_FLAGS, *defines, "-c", os.path.join(G.CSRC, src), "-o", obj])
        open(os.path.join(out, "ptxas.log"), "w").write(log)
        objs.append(obj)
    for src in G.LIB_SOURCES_CXX:
        obj = os.path.join(out, src + ".o")
        extra = ["-I" + G.BUILD, f'-DNLOPT_B200_CUDA_LIB64="{cuda_home}/lib64"'] if src == "jit.cpp" else []      # as in build_library
        G._run(["g++", *G.CXX_FLAGS, *extra, *defines, f"-I{cuda_home}/include", "-c", os.path.join(G.CSRC, src), "-o", obj])
        objs.append(obj)
    lib = os.path.join(out, "libnlopt_b200.so")
    G._run([G.NVCC, *G.ARCH, "-shared", "-o", lib, *objs, "-cudart", "shared", "-ldl", "-Xlinker", "-soname,libnlopt_b200.so",
            "-Xlinker", "-Bsymbolic-functions"])
    G._run([G.NVCC, *G.ARCH, *G.NVCC_FLAGS, *defines, "-shared", os.path.join(G.CSRC, "problems.cu"), "-o",
            os.path.join(out, "libnlopt_b200_problems.so"), "-cudart", "shared", "-L" + out, "-lnlopt_b200", "-Xlinker", "-rpath=$ORIGIN"])
    for o in objs:
        os.remove(o)
    print("built", lib, " ".join(defines))


if __name__ == "__main__":
    build(sys.argv[1], sys.argv[2:])
