"""The host palette of the sigma index (nlopt_b200/csrc/sigma_palette.hpp), without a GPU: the palette and its transition
table must reproduce, bit for bit, a numpy model of sigma_init_kernel and of end_outer_kernel's sigma update for every
variable under random branch sequences, and its closure sizes are pinned for the benchmark's box."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GAMMA = (0.7, 1.2, 1.0)          # branch b of end_outer_kernel: osc < 0, osc > 0, otherwise


@pytest.fixture(scope="module")
def pal_lib():
    src = os.path.join(ROOT, "tests", "cpp", "sigma_palette_probe.cpp")
    hdr = os.path.join(ROOT, "nlopt_b200", "csrc", "sigma_palette.hpp")
    out = os.path.join(ROOT, "tests", "_build", "libsigma_palette_probe.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or max(os.path.getmtime(src), os.path.getmtime(hdr)) > os.path.getmtime(out):
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", src, "-o", out], check=True)
    L = C.CDLL(out)
    L.nb200_sigma_palette.restype = C.c_int
    L.nb200_sigma_palette.argtypes = [C.c_double] * 5 + [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                                                         C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    L.nb200_sigma_palette_cap.restype = C.c_longlong
    return L


def palette(L, lb, ub, init, kappa, sigma_min, updates, want_tables=True):
    sizes = np.zeros(max(updates, 1), np.int64)
    cap = int(L.nb200_sigma_palette_cap())
    val = np.zeros(cap, np.float64) if want_tables else None
    nxt = np.zeros(3 * cap, np.uint16) if want_tables else None
    nv, nr = C.c_longlong(), C.c_longlong()
    done = L.nb200_sigma_palette(lb, ub, init, kappa, sigma_min, updates, sizes.ctypes.data,
                                 val.ctypes.data if want_tables else None, nxt.ctypes.data if want_tables else None,
                                 cap, C.byref(nv), C.byref(nr))
    out = dict(done=done, sizes=sizes[:done], nval=nv.value, nrows=nr.value)
    if want_tables:
        out["val"], out["next"] = val[:nv.value], nxt[:3 * nr.value].reshape(-1, 3)
    return out


def model_sigma0(lb, ub, init, sigma_min, n):
    """sigma_init_kernel for uniform bounds and a uniform initial step"""
    if init > 0:
        s = init
    elif np.isinf(ub) or np.isinf(lb):
        s = 1.0
    else:
        s = np.float64(0.5) * (np.float64(ub) - np.float64(lb))
    return np.full(n, s if s > sigma_min else sigma_min, np.float64)


def model_update(sig, br, lb, ub, kappa, sigma_min):
    """end_outer_kernel's sigma update, element-wise IEEE double (no fused operations in numpy)"""
    s = sig * np.asarray(GAMMA, np.float64)[br]
    if not (np.isinf(ub) or np.isinf(lb)):
        rng = np.float64(ub) - np.float64(lb)
        top, bot = np.float64(10.0) * rng, np.float64(kappa) * rng
        s = np.where(s < top, s, top)
        s = np.where(s > bot, s, bot)
    return np.where(s > sigma_min, s, sigma_min)


CASES = [  # lb, ub, initial step (<= 0: none), kappa, sigma_min
    (-2.0, 2.0, 0.0, 1e-8, 0.0),          # the benchmark's box, CCSAQ
    (-2.0, 2.0, 0.0, 0.01, 0.0),          # MMA
    (0.0, 1.0, 0.0, 0.01, 1e-3),
    (-0.3, 0.3, 0.05, 1e-8, 0.0),         # uniform initial step
    (-1.0, 1.0, 0.0, 1e-8, 0.25),         # sigma_min above sigma_0 * 0.7
    (-np.inf, np.inf, 0.0, 1e-8, 0.0),    # no clamp: sigma_0 = 1
    (-1.0, np.inf, 0.0, 0.01, 1e-6),
    (-1e-3, 1e-3, 0.0, 1e-8, 1e-300),
]


@pytest.mark.parametrize("lb,ub,init,kappa,sigma_min", CASES)
def test_palette_follows_sigma_of_every_variable(pal_lib, lb, ub, init, kappa, sigma_min):
    updates, n = 30, 4096
    p = palette(pal_lib, lb, ub, init, kappa, sigma_min, updates)
    assert p["done"] == updates
    val, nxt = p["val"], p["next"]
    assert val[0] == 0.0
    rng = np.random.default_rng(CASES.index((lb, ub, init, kappa, sigma_min)))
    sig = model_sigma0(lb, ub, init, sigma_min, n)
    idx = np.ones(n, np.int64)
    assert np.array_equal(val[idx].view(np.uint64), sig.view(np.uint64))
    # each variable takes its own branch sequence; some mostly shrink, some mostly grow, some mix
    bias = rng.integers(0, 3, n)
    for k in range(updates):
        br = np.where(rng.random(n) < 0.6, bias, rng.integers(0, 3, n))
        sig = model_update(sig, br, lb, ub, kappa, sigma_min)
        assert np.all(idx < p["nrows"]), "an index without a transition row"
        idx = nxt[idx, br].astype(np.int64)
        assert np.array_equal(val[idx].view(np.uint64), sig.view(np.uint64)), f"update {k + 1}"


def test_palette_rows_cover_every_value_but_the_newest(pal_lib):
    p = palette(pal_lib, -2.0, 2.0, 0.0, 1e-8, 0.0, 10)
    assert p["nrows"] == p["sizes"][-2]          # rows for every entry that existed before the last update
    assert np.all(p["next"] < p["nval"]) and tuple(p["next"][0]) == (0, 0, 0)
    assert len(set(p["val"][1:].view(np.uint64).tolist())) == p["nval"] - 1, "duplicate palette values"


def test_closure_sizes_of_the_benchmark_box(pal_lib):
    """|P_k| on [-2, 2]^n, sigma_min = 0, without the padding entry: polynomial growth, 68 values after the 7 updates of
    the benchmark's 8 inner iterations, and the 65535-entry cap is passed at the 79th update (CCSAQ) / 103rd (MMA)"""
    want = {1: 3, 4: 20, 7: 68, 10: 170, 20: 1112, 38: 7348, 39: 7963}
    for kappa, last in ((1e-8, 78), (0.01, 102)):
        p = palette(pal_lib, -2.0, 2.0, 0.0, kappa, 0.0, 200, want_tables=False)
        assert p["done"] == last, (kappa, p["done"])
        assert p["sizes"][-1] <= 65535
        if kappa == 1e-8:
            for k, v in want.items():
                assert p["sizes"][k - 1] - 1 == v, (k, p["sizes"][k - 1] - 1, v)
