"""Python handle on libnlopt_b200_problems.so: the BASELINE.json problems as device-resident
(__device__ functor) or host (plain C nlopt_func) callbacks.  The host callbacks are ordinary
function pointers, so they can also be registered with another NLopt-ABI library (the reference
arm of bench.py does exactly that)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from ._capi import LIB_DIR, NLOPT_FUNC, c_double_p

LIB_PATH = os.path.join(LIB_DIR, "libnlopt_b200_problems.so")


def _load():
    L = C.CDLL(LIB_PATH, mode=C.RTLD_LOCAL)
    L.nb200p_create.restype = C.c_void_p
    L.nb200p_destroy.argtypes = [C.c_void_p]
    L.nb200p_callback_seconds.restype = C.c_double
    L.nb200p_set_rosenbrock_device.argtypes = [C.c_void_p, C.c_void_p]
    L.nb200p_add_linear_device.argtypes = [C.c_void_p, C.c_void_p, c_double_p, C.c_double, C.c_double]
    L.nb200p_set_quadratic_device.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong]
    L.nb200p_add_mean_device.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double]
    L.nb200p_make_linear_data.restype = C.c_void_p
    L.nb200p_make_linear_data.argtypes = [C.c_void_p, c_double_p, C.c_double]
    L.nb200p_set_simp_device.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_double]
    L.nb200p_add_linear_device_eq.argtypes = [C.c_void_p, C.c_void_p, c_double_p, C.c_double, C.c_double, C.c_int]
    L.nb200p_add_mean_device_eq.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int]
    L.nb200p_add_sphere_device_eq.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int]
    L.nb200p_set_quadratic_device_sync.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong]
    L.nb200p_set_simp_device_sync.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_double]
    L.nb200p_add_mean_device_sync.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double]
    L.nb200p_add_linear_rows_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, c_double_p, c_double_p, c_double_p, C.c_int]
    L.nb200p_add_block_mean_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint, c_double_p, c_double_p, C.c_int]
    L.nb200p_set_quadratic_device_max.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_int]
    L.nb200p_set_simp_device_max.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_double, C.c_int]
    L.nb200p_set_rosenbrock_device_form.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.nb200p_quadratic_pointers.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.c_int, C.c_int,
                                            C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    for nm, args in (("nb200p_make_simp_data", [C.c_void_p, C.c_ulonglong, C.c_double]),
                     ("nb200p_make_mean_data", [C.c_void_p, C.c_double]), ("nb200p_make_quad_data", [C.c_void_p, C.c_ulonglong])):
        getattr(L, nm).restype = C.c_void_p
        getattr(L, nm).argtypes = args
    return L


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _load()
    return _lib


def linear_weights(k, n):
    """weight row of constraint k of the config-3 instance (SURVEY.md 8(d)); same as tests/problems.py"""
    j = np.arange(n, dtype=np.float64)
    return (1.0 + 0.5 * np.sin(0.37 * (k + 1) * j)) / n


def rosen_x0(n):
    return -1.2 + 0.001 * (np.arange(n) % 7)


class Problem:
    """Owns the functor parameters / weight rows for one opt; keep it alive while the opt runs."""

    def __init__(self):
        self.L = lib()
        self.h = self.L.nb200p_create()
        self._keep = []

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            self.L.nb200p_destroy(h)

    # ---- device-resident callbacks (product library only) ----
    def rosenbrock_device(self, opt, m, tol=1e-8):
        n = opt.get_dimension()
        opt._check(self.L.nb200p_set_rosenbrock_device(self.h, opt._h))
        for k in range(m):
            w = linear_weights(k, n)
            opt._check(self.L.nb200p_add_linear_device(self.h, opt._h, w.ctypes.data_as(c_double_p), 0.5 + 0.1 * k, tol))

    # ---- vector device constraints: m rows from one functor, m in {1, 2, 4, 8, 16} ----
    def add_linear_rows_device(self, opt, w, b, tol=0.0, equality=False):
        """m dense linear rows  w_k.x - b_k  (<= 0, or = 0 with equality=True); w: [m][n]"""
        w = np.ascontiguousarray(w, dtype=np.float64)
        m = w.shape[0]
        b = np.ascontiguousarray(np.broadcast_to(b, (m,)), dtype=np.float64)
        tol = np.ascontiguousarray(np.broadcast_to(tol, (m,)), dtype=np.float64)
        opt._check(self.L.nb200p_add_linear_rows_device(self.h, opt._h, m, w.ctypes.data_as(c_double_p),
                                                        b.ctypes.data_as(c_double_p), tol.ctypes.data_as(c_double_p), int(equality)))

    def rosenbrock_device_rows(self, opt, m, tol=1e-8):
        """rosenbrock_device with its m LinearDev rows as one LinearRowsDev<m>: the same weights and offsets"""
        n = opt.get_dimension()
        opt._check(self.L.nb200p_set_rosenbrock_device(self.h, opt._h))
        if m:
            self.add_linear_rows_device(opt, np.stack([linear_weights(k, n) for k in range(m)]),
                                        [0.5 + 0.1 * k for k in range(m)], tol)

    def add_block_mean_device(self, opt, targets, tol=0.0):
        """local volumes  mean(x over block i) - targets[i] <= 0, block i = [i n / m, (i + 1) n / m)"""
        self._block_mean(opt, targets, tol, False)

    def add_block_mean_device_eq(self, opt, targets, tol=0.0):
        """local volumes as equalities (NLOPT_AUGLAG*)"""
        self._block_mean(opt, targets, tol, True)

    def _block_mean(self, opt, targets, tol, equality):
        t = np.ascontiguousarray(targets, dtype=np.float64)
        tol = np.ascontiguousarray(np.broadcast_to(tol, t.shape), dtype=np.float64)
        opt._check(self.L.nb200p_add_block_mean_device(self.h, opt._h, t.size, t.ctypes.data_as(c_double_p),
                                                       tol.ctypes.data_as(c_double_p), int(equality)))

    def quadratic_device(self, opt, seed=0x5EED0000, offset=0.1, tol=0.0):
        opt._check(self.L.nb200p_set_quadratic_device(self.h, opt._h, seed))
        opt._check(self.L.nb200p_add_mean_device(self.h, opt._h, offset, tol))

    # ---- device functors one at a time; sync=True registers the synchronous form (nlopt_b200_dfunc) ----
    def set_quadratic_device(self, opt, seed=0x5EED0000, sync=False):
        fn = self.L.nb200p_set_quadratic_device_sync if sync else self.L.nb200p_set_quadratic_device
        opt._check(fn(self.h, opt._h, seed))

    def set_simp_device(self, opt, seed=0x5EED0000, eps=1e-3, sync=False):
        fn = self.L.nb200p_set_simp_device_sync if sync else self.L.nb200p_set_simp_device
        opt._check(fn(self.h, opt._h, seed, eps))

    # ---- maximisation: the negated functors (Negated<F> in problems.cu) through set_max_objective ----
    # A max run of the negated functor is the min run of the functor itself, bit for bit.
    def set_quadratic_device_max(self, opt, seed=0x5EED0000, sync=False):
        """maximise -(config 2 quadratic)"""
        opt._check(self.L.nb200p_set_quadratic_device_max(self.h, opt._h, seed, int(sync)))

    def set_simp_device_max(self, opt, seed=0x5EED0000, eps=1e-3, sync=False):
        """maximise -(SIMP compliance)"""
        opt._check(self.L.nb200p_set_simp_device_max(self.h, opt._h, seed, eps, int(sync)))

    def set_rosenbrock_device(self, opt, sync=False, maximize=False):
        """the chained Rosenbrock objective alone (halo 1); maximize=True registers its negation with set_max_objective"""
        opt._check(self.L.nb200p_set_rosenbrock_device_form(self.h, opt._h, int(sync), int(maximize)))

    def quadratic_pointers(self, opt, seed=0x5EED0000, negated=False, sync=False):
        """(fn, finish, data) pointers of the quadratic functor, or of its negation, as the C++ front end registers them:
        nlopt_b200_dfunc2 / nlopt_b200_dfinish, or with sync=True an nlopt_b200_dfunc (finish None)"""
        fn, fin, data = C.c_void_p(), C.c_void_p(), C.c_void_p()
        opt._check(self.L.nb200p_quadratic_pointers(self.h, opt._h, seed, int(negated), int(sync), C.byref(fn), C.byref(fin),
                                                    C.byref(data)))
        return fn, fin, data

    def simp_sharded_max(self, opt, seed=0x5EED0000, eps=1e-3, vol=0.4, tol=0.0):
        """simp_sharded with the negated objective registered by nlopt_b200_set_max_objective_sharded"""
        lib_ = opt._lib
        d = self.L.nb200p_make_simp_data(self.h, seed, eps)
        opt._check(lib_.nlopt_b200_set_max_objective_sharded(opt._h, C.cast(self.L.nb200p_simp_sharded_neg, C.c_void_p), d))
        dm = self.L.nb200p_make_mean_data(self.h, -vol)
        opt._check(lib_.nlopt_b200_add_inequality_constraint_sharded(opt._h, C.cast(self.L.nb200p_mean_sharded, C.c_void_p), dm, tol))

    def add_mean_device(self, opt, offset, tol=0.0, sync=False):
        """inequality  mean(x) + offset <= 0"""
        fn = self.L.nb200p_add_mean_device_sync if sync else self.L.nb200p_add_mean_device
        opt._check(fn(self.h, opt._h, offset, tol))

    def add_mean_device_eq(self, opt, offset, tol=0.0, sync=False):
        """equality  mean(x) + offset = 0  (NLOPT_AUGLAG*)"""
        opt._check(self.L.nb200p_add_mean_device_eq(self.h, opt._h, offset, tol, int(sync)))

    def add_linear_device_eq(self, opt, w, b, tol=0.0, sync=False):
        """equality  w.x - b = 0  (NLOPT_AUGLAG*)"""
        w = np.ascontiguousarray(w, dtype=np.float64)
        opt._check(self.L.nb200p_add_linear_device_eq(self.h, opt._h, w.ctypes.data_as(c_double_p), b, tol, int(sync)))

    def add_sphere_device_eq(self, opt, r, tol=0.0, sync=False):
        """equality  mean(x_j^2) - r = 0  (NLOPT_AUGLAG*)"""
        opt._check(self.L.nb200p_add_sphere_device_eq(self.h, opt._h, r, tol, int(sync)))

    def simp_device_eq(self, opt, seed=0x5EED0000, eps=1e-3, vol=0.4, tol=0.0):
        """config 4 with the volume constraint as an equality, device functors"""
        self.set_simp_device(opt, seed, eps)
        self.add_mean_device_eq(opt, -vol, tol)

    def simp_host_eq(self, opt, seed=0x5EED0000, eps=1e-3, vol=0.4, tol=0.0):
        """config 4 with the volume constraint as an equality, plain C host callbacks"""
        lib_ = opt._lib
        d = self.L.nb200p_make_simp_data(self.h, seed, eps)
        opt._check(lib_.nlopt_set_min_objective(opt._h, self._fn("nb200p_simp_host"), d))
        dm = self.L.nb200p_make_mean_data(self.h, -vol)
        opt._check(lib_.nlopt_add_equality_constraint(opt._h, self._fn("nb200p_mean_host"), dm, tol))

    # ---- host callbacks in C (any NLopt-ABI library) ----
    def _fn(self, name):
        return C.cast(getattr(self.L, name), NLOPT_FUNC)

    def rosenbrock_host(self, opt, m, tol=1e-8):
        n = opt.get_dimension()
        lib_ = opt._lib
        opt._check(lib_.nlopt_set_min_objective(opt._h, self._fn("nb200p_rosenbrock_host"), None))
        for k in range(m):
            w = linear_weights(k, n)
            self._keep.append(w)
            d = self.L.nb200p_make_linear_data(self.h, w.ctypes.data_as(c_double_p), 0.5 + 0.1 * k)
            opt._check(lib_.nlopt_add_inequality_constraint(opt._h, self._fn("nb200p_linear_host"), d, tol))

    def simp_host(self, opt, seed=0x5EED0000, eps=1e-3, vol=0.4, tol=0.0):
        """BASELINE config 4: synthetic SIMP compliance + volume constraint, plain C host callbacks"""
        lib_ = opt._lib
        d = self.L.nb200p_make_simp_data(self.h, seed, eps)
        opt._check(lib_.nlopt_set_min_objective(opt._h, self._fn("nb200p_simp_host"), d))
        dm = self.L.nb200p_make_mean_data(self.h, -vol)
        opt._check(lib_.nlopt_add_inequality_constraint(opt._h, self._fn("nb200p_mean_host"), dm, tol))

    def simp_sharded(self, opt, seed=0x5EED0000, eps=1e-3, vol=0.4, tol=0.0):
        """config 4 with sharded host callbacks (product library only): each rank evaluates its own variables"""
        lib_ = opt._lib
        d = self.L.nb200p_make_simp_data(self.h, seed, eps)
        opt._check(lib_.nlopt_b200_set_min_objective_sharded(opt._h, C.cast(self.L.nb200p_simp_sharded, C.c_void_p), d))
        dm = self.L.nb200p_make_mean_data(self.h, -vol)
        opt._check(lib_.nlopt_b200_add_inequality_constraint_sharded(opt._h, C.cast(self.L.nb200p_mean_sharded, C.c_void_p), dm, tol))

    def simp_device(self, opt, seed=0x5EED0000, eps=1e-3, vol=0.4, tol=0.0):
        opt._check(self.L.nb200p_set_simp_device(self.h, opt._h, seed, eps))
        opt._check(self.L.nb200p_add_mean_device(self.h, opt._h, -vol, tol))

    def quadratic_host(self, opt, seed=0x5EED0000, offset=0.1, tol=0.0):
        """BASELINE config 2 with host callbacks (the device form is quadratic_device)"""
        lib_ = opt._lib
        d = self.L.nb200p_make_quad_data(self.h, seed)
        opt._check(lib_.nlopt_set_min_objective(opt._h, self._fn("nb200p_quadratic_host"), d))
        dm = self.L.nb200p_make_mean_data(self.h, offset)
        opt._check(lib_.nlopt_add_inequality_constraint(opt._h, self._fn("nb200p_mean_host"), dm, tol))

    def callback_seconds(self):
        return self.L.nb200p_callback_seconds()

    def reset_callback_seconds(self):
        self.L.nb200p_reset_callback_seconds()
