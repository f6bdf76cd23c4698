"""nlopt_b200 -- Python face of the GPU-native (H100) MMA/CCSAQ solver.

Mirrors the reference's Python module (SWIG over nlopt.hpp: src/swig/nlopt-python.i,
src/api/nlopt-in.hpp:254-609): ``opt(algorithm, n)``, ``set_min_objective(f)`` with
``f(x, grad)`` writing ``grad`` in place when ``grad.size > 0``, ``add_inequality_constraint``,
``optimize(x)`` returning the optimum as an array, ``last_optimum_value()``,
``last_optimize_result()``, the ``LD_MMA`` / ``LD_CCSAQ`` / result-code constants and the
exception mapping of nlopt.hpp ``mythrow`` (:87-103).

All arithmetic happens in ``libnlopt_b200.so`` (CUDA, sm_90a) behind the NLopt C ABI;
this module only marshals numpy arrays.  ``opt(..., library=Library(path))`` points the same
class at another library exporting that ABI (tests use it to run the unmodified reference).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._capi import (NLOPT_B200_DFINISH, NLOPT_B200_DFUNC, NLOPT_B200_DMFINISH, NLOPT_B200_DTFUNC, NLOPT_FUNC,
                    NLOPT_PRECOND, NLOPT_MFUNC, Library, Shard, Stats, c_double_p, default_library)

# --- algorithm ids (reference nlopt.h:72-154) ---------------------------------
_ALG_NAMES = [
    "GN_DIRECT", "GN_DIRECT_L", "GN_DIRECT_L_RAND", "GN_DIRECT_NOSCAL", "GN_DIRECT_L_NOSCAL",
    "GN_DIRECT_L_RAND_NOSCAL", "GN_ORIG_DIRECT", "GN_ORIG_DIRECT_L", "GD_STOGO", "GD_STOGO_RAND",
    "LD_LBFGS_NOCEDAL", "LD_LBFGS", "LN_PRAXIS", "LD_VAR1", "LD_VAR2", "LD_TNEWTON",
    "LD_TNEWTON_RESTART", "LD_TNEWTON_PRECOND", "LD_TNEWTON_PRECOND_RESTART", "GN_CRS2_LM",
    "GN_MLSL", "GD_MLSL", "GN_MLSL_LDS", "GD_MLSL_LDS", "LD_MMA", "LN_COBYLA", "LN_NEWUOA",
    "LN_NEWUOA_BOUND", "LN_NELDERMEAD", "LN_SBPLX", "LN_AUGLAG", "LD_AUGLAG", "LN_AUGLAG_EQ",
    "LD_AUGLAG_EQ", "LN_BOBYQA", "GN_ISRES", "AUGLAG", "AUGLAG_EQ", "G_MLSL", "G_MLSL_LDS",
    "LD_SLSQP", "LD_CCSAQ", "GN_ESCH", "GN_AGS",
]
for _i, _n in enumerate(_ALG_NAMES):
    globals()[_n] = _i
NUM_ALGORITHMS = len(_ALG_NAMES)

# --- result codes (reference nlopt.h:162-176) ---------------------------------
FAILURE, INVALID_ARGS, OUT_OF_MEMORY, ROUNDOFF_LIMITED, FORCED_STOP = -1, -2, -3, -4, -5
SUCCESS, STOPVAL_REACHED, FTOL_REACHED, XTOL_REACHED, MAXEVAL_REACHED, MAXTIME_REACHED = 1, 2, 3, 4, 5, 6


class RoundoffLimited(RuntimeError):
    """nlopt.hpp roundoff_limited (:71-74)"""


class ForcedStop(RuntimeError):
    """nlopt.hpp forced_stop (:76-79)"""


def _as_f64(a, n=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if n is not None and a.size != n:
        raise ValueError(f"dimension mismatch: expected {n}, got {a.size}")
    return a


def _ptr(a):
    return a.ctypes.data_as(c_double_p)


def _cuda_f64(v, n):
    """the device pointer of `v`, an object with __cuda_array_interface__ describing n contiguous float64 values"""
    cai = v.__cuda_array_interface__
    shape, strides = tuple(cai["shape"]), cai.get("strides")
    contiguous = []
    step = 8
    for d in reversed(shape):
        contiguous.insert(0, step)
        step *= d
    if (cai["typestr"] != "<f8" or int(np.prod(shape, dtype=np.int64)) != n
            or (strides is not None and tuple(strides) != tuple(contiguous))):
        raise ValueError(f"device bounds need a contiguous float64 CUDA array of {n} values (got typestr "
                         f"{cai['typestr']}, shape {shape}, strides {strides})")
    return cai["data"][0]


class _DeviceArray:
    """float64 device memory of the library, handed to torch.as_tensor as a zero-copy view (no stream: the view is
    used on the library stream itself)"""

    def __init__(self, ptr, shape, strides):
        self.__cuda_array_interface__ = {"shape": shape, "strides": strides, "typestr": "<f8", "data": (ptr, False),
                                         "version": 2}


class CompileError(RuntimeError):
    """a CudaFunctor that did not compile or is not accepted; .log holds the compiler log"""

    def __init__(self, msg, log=""):
        super().__init__(msg)
        self.log = log


class CudaFunctor:
    """A __device__ functor given as source (the concept of include/nlopt_b200_device.cuh), compiled at run time by
    NVRTC for sm_90a with the library's map kernels, no nvcc needed.  `name` names the functor struct in `source`;
    `options` are extra NVRTC options.  .m (0 for a scalar functor), .halo, .param_bytes (sizeof the functor) and .log
    (the compiler's log).  Raises CompileError, with the compiler's message, when the source does not compile or the
    functor is not accepted (m > 16, halo > 1).  Compiled images are cached per process."""

    def __init__(self, source, name, options=(), library: Library | None = None):
        self._lib = library or default_library()
        opts = [o.encode() for o in options]
        arr = (C.c_char_p * max(len(opts), 1))(*opts)
        self._h = self._lib.nlopt_b200_jit_create(source.encode(), name.encode(), arr, len(opts))
        if not self._h:
            raise MemoryError("nlopt_b200_jit_create")
        log = self._lib.nlopt_b200_jit_log(self._h)
        self.log = log.decode(errors="replace") if log else ""
        err = self._lib.nlopt_b200_jit_errmsg(self._h)
        if err:
            raise CompileError(err.decode(errors="replace"), self.log)
        m, halo, nbytes = C.c_int(), C.c_int(), C.c_size_t()
        self._lib.nlopt_b200_jit_info(self._h, C.byref(m), C.byref(halo), C.byref(nbytes))
        self.m, self.halo, self.param_bytes = m.value, halo.value, nbytes.value

    def image(self):
        """the compiled sm_90a cubin"""
        n = C.c_size_t()
        p = self._lib.nlopt_b200_jit_image(self._h, C.byref(n))
        return C.string_at(p, n.value) if p else b""

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.nlopt_b200_jit_destroy(h)


class opt:
    """One optimisation problem; thin owner of an ``nlopt_opt`` handle."""

    def __init__(self, algorithm, n, library: Library | None = None):
        self._lib = library or default_library()
        self._h = self._lib.nlopt_create(int(algorithm), int(n))
        if not self._h:
            raise RuntimeError("nlopt failure")       # nlopt.hpp:263
        self._n = int(n)
        self._keep = []            # ctypes thunks must outlive the handle
        self._exc = None           # exception raised inside a callback
        self._tviews = {}          # torch callbacks: zero-copy views and external streams, per pointer (one run)
        self._last_result = FAILURE
        self._last_optf = float("inf")

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.nlopt_destroy(h)

    # ---- error mapping, nlopt.hpp:87-103 -------------------------------------
    def _check(self, ret):
        if ret >= 0:
            return ret
        msg = self._lib.nlopt_get_errmsg(self._h)
        msg = msg.decode() if msg else None
        if ret == FAILURE:
            raise RuntimeError(msg or "nlopt failure")
        if ret == OUT_OF_MEMORY:
            raise MemoryError(msg or "out of memory")
        if ret == INVALID_ARGS:
            raise ValueError(msg or "nlopt invalid argument")
        if ret == ROUNDOFF_LIMITED:
            raise RoundoffLimited(msg or "nlopt roundoff-limited")
        if ret == FORCED_STOP:
            raise ForcedStop(msg or "nlopt forced stop")
        raise RuntimeError(msg or "nlopt failure")

    # ---- callbacks -----------------------------------------------------------
    def _wrap_func(self, f):
        n_fixed = self._n

        def thunk(n, x, grad, _data):
            try:
                xa = np.ctypeslib.as_array(x, shape=(n,))
                ga = np.ctypeslib.as_array(grad, shape=(n,)) if grad else np.empty(0)
                return float(f(xa, ga))
            except BaseException as e:      # nlopt.hpp:149-166: exception => forced stop
                self._exc = e
                self._lib.nlopt_force_stop(self._h)
                return float("nan")

        cb = NLOPT_FUNC(thunk)
        self._keep.append(cb)
        del n_fixed
        return cb

    def _wrap_mfunc(self, f):
        def thunk(m, result, n, x, grad, _data):
            try:
                ra = np.ctypeslib.as_array(result, shape=(m,))
                xa = np.ctypeslib.as_array(x, shape=(n,))
                ga = np.ctypeslib.as_array(grad, shape=(m, n)) if grad else np.empty(0)
                f(ra, xa, ga)
            except BaseException as e:
                self._exc = e
                self._lib.nlopt_force_stop(self._h)

        cb = NLOPT_MFUNC(thunk)
        self._keep.append(cb)
        return cb

    def set_min_objective(self, f):
        self._check(self._lib.nlopt_set_min_objective(self._h, self._wrap_func(f), None))

    def set_max_objective(self, f):
        self._check(self._lib.nlopt_set_max_objective(self._h, self._wrap_func(f), None))

    # preconditioned forms (nlopt.h:70, options.c:322-337): pre(x, v, vpre) writes vpre = H(x) v
    def _wrap_precond(self, pre):
        def thunk(n, x, v, vpre, _data):
            try:
                pre(np.ctypeslib.as_array(x, shape=(n,)), np.ctypeslib.as_array(v, shape=(n,)), np.ctypeslib.as_array(vpre, shape=(n,)))
            except BaseException as e:
                self._exc = e
                self._lib.nlopt_force_stop(self._h)

        cb = NLOPT_PRECOND(thunk)
        self._keep.append(cb)
        return C.cast(cb, C.c_void_p)

    def set_precond_min_objective(self, f, pre):
        self._check(self._lib.nlopt_set_precond_min_objective(self._h, self._wrap_func(f), self._wrap_precond(pre), None))

    def add_precond_inequality_constraint(self, fc, pre, tol=0.0):
        self._check(self._lib.nlopt_add_precond_inequality_constraint(self._h, self._wrap_func(fc), self._wrap_precond(pre), None, float(tol)))

    def add_inequality_constraint(self, fc, tol=0.0):
        self._check(self._lib.nlopt_add_inequality_constraint(self._h, self._wrap_func(fc), None, float(tol)))

    def add_equality_constraint(self, h, tol=0.0):
        self._check(self._lib.nlopt_add_equality_constraint(self._h, self._wrap_func(h), None, float(tol)))

    def add_inequality_mconstraint(self, fc, tol):
        tol = _as_f64(tol)
        self._check(self._lib.nlopt_add_inequality_mconstraint(
            self._h, tol.size, self._wrap_mfunc(fc), None, _ptr(tol)))

    def add_equality_mconstraint(self, h, tol):
        tol = _as_f64(tol)
        self._check(self._lib.nlopt_add_equality_mconstraint(
            self._h, tol.size, self._wrap_mfunc(h), None, _ptr(tol)))

    def remove_inequality_constraints(self):
        self._check(self._lib.nlopt_remove_inequality_constraints(self._h))

    def remove_equality_constraints(self):
        self._check(self._lib.nlopt_remove_equality_constraints(self._h))

    # ---- extension: device-resident callbacks (raw C function pointers) -------
    def set_min_objective_device(self, fn_ptr, data_ptr=None):
        self._check(self._lib.nlopt_b200_set_min_objective_device(self._h, fn_ptr, data_ptr))

    def set_max_objective_device(self, fn_ptr, data_ptr=None):
        """maximise the function of an nlopt_b200_dfunc pointer: the library minimises its negation"""
        self._check(self._lib.nlopt_b200_set_max_objective_device(self._h, fn_ptr, data_ptr))

    # asynchronous device objectives (nlopt_b200_dfunc2 / nlopt_b200_dfinish pointers)
    def set_min_objective_device2(self, fn_ptr, finish_ptr, data_ptr=None, halo=0):
        self._check(self._lib.nlopt_b200_set_min_objective_device2(self._h, fn_ptr, finish_ptr, data_ptr, int(halo)))

    def set_max_objective_device2(self, fn_ptr, finish_ptr, data_ptr=None, halo=0):
        self._check(self._lib.nlopt_b200_set_max_objective_device2(self._h, fn_ptr, finish_ptr, data_ptr, int(halo)))

    def add_inequality_constraint_device(self, fn_ptr, data_ptr=None, tol=0.0):
        self._check(self._lib.nlopt_b200_add_inequality_constraint_device(
            self._h, fn_ptr, data_ptr, float(tol)))

    def add_equality_constraint_device(self, fn_ptr, data_ptr=None, tol=0.0):
        self._check(self._lib.nlopt_b200_add_equality_constraint_device(
            self._h, fn_ptr, data_ptr, float(tol)))

    # vector device constraints (nlopt_b200_dmfunc2 / nlopt_b200_dmfinish pointers); m = len(tol)
    def add_inequality_mconstraint_device(self, fn_ptr, finish_ptr, data_ptr, tol, halo=0):
        tol = _as_f64(tol)
        self._check(self._lib.nlopt_b200_add_inequality_mconstraint_device2(
            self._h, tol.size, fn_ptr, finish_ptr, data_ptr, _ptr(tol), int(halo)))

    def add_equality_mconstraint_device(self, fn_ptr, finish_ptr, data_ptr, tol, halo=0):
        tol = _as_f64(tol)
        self._check(self._lib.nlopt_b200_add_equality_mconstraint_device2(
            self._h, tol.size, fn_ptr, finish_ptr, data_ptr, _ptr(tol), int(halo)))

    # ---- extension: PyTorch callbacks (per-variable terms, nlopt_b200_dtfunc) ---------------------------------------
    # f(x, grad) gets zero-copy float64 CUDA views of the library's HBM: x (n_local entries; with halo=1 n_local + 2,
    # x[0] being the left neighbour x[-1]) and grad, written in place -- (n_local,), or (m, n_local) with row stride ld
    # for the vector form; empty (numel() == 0) when no gradient is wanted.  f returns the terms, whose sum is the
    # function: a float64 tensor of grad's shape.  The library reduces them on the GPU in the order of the __device__
    # functors and applies finish once per point (default: the identity; vector form: m totals -> m values, numpy).
    # f runs on the library's stream (torch.cuda.ExternalStream), so its kernels are ordered with the library's.
    def _tcached(self, key, make):
        v = self._tviews.get(key)
        if v is None:
            v = self._tviews[key] = make()
        return v

    def _wrap_terms(self, f, vector, halo):
        import torch

        def view(ptr, shape, strides):
            return self._tcached((ptr, shape, strides), lambda: torch.as_tensor(_DeviceArray(ptr, shape, strides)))

        def thunk(m, shard, x, grad, ld, terms, _data, stream):
            try:
                nl_ = Shard.from_address(shard).n_local
                shape, strides = ((m, nl_), (8 * ld, 8)) if vector else ((nl_,), (8,))
                xv = view(x - 8 * halo, (nl_ + 2 * halo,), (8,))
                tv = view(terms, shape, strides)
                gv = view(grad, shape, strides) if grad else self._tcached(
                    ("empty", xv.device), lambda: torch.empty(0, dtype=torch.float64, device=xv.device))
                s = self._tcached(("stream", stream), lambda: torch.cuda.ExternalStream(stream, device=xv.device))
                with torch.cuda.stream(s):
                    out = f(xv, gv)
                    if not (isinstance(out, torch.Tensor) and out.dtype == torch.float64 and out.device == tv.device
                            and tuple(out.shape) == shape):
                        raise ValueError(f"a torch terms callback returns a float64 tensor of shape {shape} on {tv.device}")
                    tv.copy_(out)
            except BaseException as e:
                self._exc = e
                self._lib.nlopt_force_stop(self._h)

        cb = NLOPT_B200_DTFUNC(thunk)
        self._keep.append(cb)
        return C.cast(cb, C.c_void_p)

    def _wrap_finish(self, finish):
        def thunk(total, _data):
            try:
                return float(total if finish is None else finish(total))
            except BaseException as e:
                self._exc = e
                self._lib.nlopt_force_stop(self._h)
                return float("nan")

        cb = NLOPT_B200_DFINISH(thunk)
        self._keep.append(cb)
        return C.cast(cb, C.c_void_p)

    def _wrap_mfinish(self, finish):
        def thunk(m, totals, result, _data):
            try:
                t = np.ctypeslib.as_array(totals, shape=(m,)).copy()
                np.ctypeslib.as_array(result, shape=(m,))[:] = t if finish is None else finish(t)
            except BaseException as e:
                self._exc = e
                self._lib.nlopt_force_stop(self._h)

        cb = NLOPT_B200_DMFINISH(thunk)
        self._keep.append(cb)
        return C.cast(cb, C.c_void_p)

    def set_min_objective_torch(self, f, finish=None, halo=0):
        self._check(self._lib.nlopt_b200_set_min_objective_terms(
            self._h, self._wrap_terms(f, False, halo), self._wrap_finish(finish), None, int(halo)))

    def set_max_objective_torch(self, f, finish=None, halo=0):
        self._check(self._lib.nlopt_b200_set_max_objective_terms(
            self._h, self._wrap_terms(f, False, halo), self._wrap_finish(finish), None, int(halo)))

    def add_inequality_constraint_torch(self, fc, tol=0.0, finish=None, halo=0):
        self._check(self._lib.nlopt_b200_add_inequality_constraint_terms(
            self._h, self._wrap_terms(fc, False, halo), self._wrap_finish(finish), None, float(tol), int(halo)))

    def add_equality_constraint_torch(self, h, tol=0.0, finish=None, halo=0):
        self._check(self._lib.nlopt_b200_add_equality_constraint_terms(
            self._h, self._wrap_terms(h, False, halo), self._wrap_finish(finish), None, float(tol), int(halo)))

    # m = len(tol) rows: f returns (m, n_local) terms
    def add_inequality_mconstraint_torch(self, fc, tol, finish=None, halo=0):
        tol = _as_f64(tol)
        self._check(self._lib.nlopt_b200_add_inequality_mconstraint_terms(
            self._h, tol.size, self._wrap_terms(fc, True, halo), self._wrap_mfinish(finish), None, _ptr(tol), int(halo)))

    def add_equality_mconstraint_torch(self, h, tol, finish=None, halo=0):
        tol = _as_f64(tol)
        self._check(self._lib.nlopt_b200_add_equality_mconstraint_terms(
            self._h, tol.size, self._wrap_terms(h, True, halo), self._wrap_mfinish(finish), None, _ptr(tol), int(halo)))

    # ---- extension: __device__ functors given as source (CudaFunctor, nlopt_b200_jit) ---------------------------------
    # params: the functor object's bytes (sizeof(F) of them; e.g. bytes(ctypes.Structure) or struct.pack, with
    # tensor.data_ptr() for device arrays); finish as for the torch methods (None: the identity, applied in C).  The
    # functor's kernels are the nvcc-built functor's kernels, so runs match it bit for bit.
    def _cuda_reg(self, fn, f, params, finish, vector, *tail):
        if not isinstance(f, CudaFunctor):
            raise TypeError("expected an nlopt_b200.CudaFunctor")
        buf = memoryview(params).tobytes()          # copied by the library at registration
        fin = None if finish is None else (self._wrap_mfinish(finish) if vector else self._wrap_finish(finish))
        self._keep.append(f)                    # the functor's handle owns the registration: it lives as long as this opt
        self._check(fn(self._h, f._h, buf, len(buf), fin, None, *tail))

    def set_min_objective_cuda(self, f, params=b"", finish=None):
        self._cuda_reg(self._lib.nlopt_b200_jit_set_min_objective, f, params, finish, False)

    def set_max_objective_cuda(self, f, params=b"", finish=None):
        self._cuda_reg(self._lib.nlopt_b200_jit_set_max_objective, f, params, finish, False)

    def add_inequality_constraint_cuda(self, fc, params=b"", tol=0.0, finish=None):
        self._cuda_reg(self._lib.nlopt_b200_jit_add_inequality_constraint, fc, params, finish, False, float(tol))

    def add_equality_constraint_cuda(self, h, params=b"", tol=0.0, finish=None):
        self._cuda_reg(self._lib.nlopt_b200_jit_add_equality_constraint, h, params, finish, False, float(tol))

    # m = fc.m rows; tol: m entries (None: zeros); finish maps the m totals to the m values (numpy)
    def add_inequality_mconstraint_cuda(self, fc, params=b"", tol=None, finish=None):
        tol = None if tol is None else _as_f64(tol, max(fc.m, 1))
        self._cuda_reg(self._lib.nlopt_b200_jit_add_inequality_mconstraint, fc, params, finish, True,
                       None if tol is None else _ptr(tol))

    def add_equality_mconstraint_cuda(self, h, params=b"", tol=None, finish=None):
        tol = None if tol is None else _as_f64(tol, max(h.m, 1))
        self._cuda_reg(self._lib.nlopt_b200_jit_add_equality_mconstraint, h, params, finish, True,
                       None if tol is None else _ptr(tol))

    def optimize_torch(self, x):
        """nlopt_b200_optimize_device on a torch tensor: x (contiguous float64 CUDA tensor of this rank's n_local
        variables) holds the start point on entry and the solution on return; last_optimum_value() is the optimum.
        Torch's current stream is synchronised first, so x is ready.  Returns x."""
        import torch
        j0, cnt = C.c_ulonglong(), C.c_ulonglong()
        lib = self._lib
        lib.nlopt_b200_shard_range(self._n, lib.nlopt_b200_comm_rank(), lib.nlopt_b200_comm_world(), C.byref(j0), C.byref(cnt))
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float64 and x.is_contiguous()
                and x.numel() == cnt.value):
            raise ValueError(f"optimize_torch needs a contiguous float64 CUDA tensor of this rank's {cnt.value} variables")
        f = C.c_double(0.0)
        self._exc = None
        self._tviews.clear()
        with torch.cuda.device(x.device):
            torch.cuda.current_stream().synchronize()
            try:
                ret = lib.nlopt_b200_optimize_device(self._h, x.data_ptr(), C.byref(f))
            finally:
                self._tviews.clear()
        self._last_result, self._last_optf = ret, f.value
        if ret == FORCED_STOP and self._exc is not None:
            e, self._exc = self._exc, None
            raise e
        self._check(ret)
        return x

    def optimize_device(self, x_dev_ptr):
        f = C.c_double(0.0)
        self._exc = None
        ret = self._lib.nlopt_b200_optimize_device(self._h, x_dev_ptr, C.byref(f))
        self._last_result, self._last_optf = ret, f.value
        self._check(ret)
        return ret

    def get_stats(self):
        s = Stats()
        self._check(self._lib.nlopt_b200_get_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in Stats._fields_}

    # ---- run (nlopt.hpp:299-321) ---------------------------------------------
    def optimize(self, x):
        xa = np.array(x, dtype=np.float64, copy=True).reshape(-1)
        if xa.size != self._n:
            raise ValueError("dimension mismatch")
        f = C.c_double(0.0)
        self._exc = None
        ret = self._lib.nlopt_optimize(self._h, _ptr(xa), C.byref(f))
        self._last_result, self._last_optf = ret, f.value
        if ret == FORCED_STOP and self._exc is not None:
            e, self._exc = self._exc, None
            raise e
        self._check(ret)
        return xa

    def optimize_inplace(self, xa):
        """The C call itself (nlopt.h: nlopt_optimize(opt, x, &minf)): `xa` is the caller's own contiguous float64 buffer,
        start point on entry, solution on return -- no Python-side copy of the n doubles.  Returns the nlopt_result."""
        if not (isinstance(xa, np.ndarray) and xa.dtype == np.float64 and xa.flags["C_CONTIGUOUS"] and xa.size == self._n):
            raise ValueError("optimize_inplace needs a contiguous float64 array of the problem's dimension")
        f = C.c_double(0.0)
        self._exc = None
        ret = self._lib.nlopt_optimize(self._h, _ptr(xa), C.byref(f))
        self._last_result, self._last_optf = ret, f.value
        if ret == FORCED_STOP and self._exc is not None:
            e, self._exc = self._exc, None
            raise e
        self._check(ret)
        return ret

    def last_optimize_result(self):
        return self._last_result

    def last_optimum_value(self):
        return self._last_optf

    # ---- accessors -----------------------------------------------------------
    def get_algorithm(self):
        return self._lib.nlopt_get_algorithm(self._h)

    def get_algorithm_name(self):
        return self._lib.nlopt_algorithm_name(self.get_algorithm()).decode()

    def get_dimension(self):
        return self._lib.nlopt_get_dimension(self._h)

    def get_errmsg(self):
        m = self._lib.nlopt_get_errmsg(self._h)
        return m.decode() if m else None

    def get_numevals(self):
        return self._lib.nlopt_get_numevals(self._h)

    def set_param(self, name, val):
        self._check(self._lib.nlopt_set_param(self._h, name.encode(), float(val)))

    def get_param(self, name, default):
        return self._lib.nlopt_get_param(self._h, name.encode(), float(default))

    def has_param(self, name):
        return bool(self._lib.nlopt_has_param(self._h, name.encode()))

    def num_params(self):
        return self._lib.nlopt_num_params(self._h)

    def nth_param(self, i):
        s = self._lib.nlopt_nth_param(self._h, int(i))
        return s.decode() if s else None

    def _set_vec_or_scalar(self, vec_fn, scalar_fn, v):
        if np.isscalar(v):
            self._check(scalar_fn(self._h, float(v)))
        else:
            a = _as_f64(v, self._n)
            self._check(vec_fn(self._h, _ptr(a)))

    def _get_vec(self, fn):
        a = np.empty(self._n)
        self._check(fn(self._h, _ptr(a)))
        return a

    # bounds: a scalar, a host array, or a device array (__cuda_array_interface__: a CUDA tensor, a CuPy array ...), which
    # the library copies into its own device memory (nlopt_b200_set_*_bounds_device); a torch tensor's current stream is
    # synchronised first
    def _set_bounds(self, vec_fn, scalar_fn, dev_name, v):
        if not hasattr(v, "__cuda_array_interface__"):
            self._set_vec_or_scalar(vec_fn, scalar_fn, v)
            return
        ptr = _cuda_f64(v, self._n)
        dev_fn = getattr(self._lib, dev_name)
        if type(v).__module__.split(".")[0] != "torch":
            self._check(dev_fn(self._h, ptr))
            return
        import torch
        with torch.cuda.device(v.device):          # the object's arrays go to the tensor's device
            torch.cuda.current_stream().synchronize()
            self._check(dev_fn(self._h, ptr))

    def set_lower_bounds(self, v):
        self._set_bounds(self._lib.nlopt_set_lower_bounds, self._lib.nlopt_set_lower_bounds1,
                         "nlopt_b200_set_lower_bounds_device", v)

    def set_upper_bounds(self, v):
        self._set_bounds(self._lib.nlopt_set_upper_bounds, self._lib.nlopt_set_upper_bounds1,
                         "nlopt_b200_set_upper_bounds_device", v)

    def set_lower_bound(self, i, v):
        self._check(self._lib.nlopt_set_lower_bound(self._h, int(i), float(v)))

    def set_upper_bound(self, i, v):
        self._check(self._lib.nlopt_set_upper_bound(self._h, int(i), float(v)))

    def get_lower_bounds(self):
        return self._get_vec(self._lib.nlopt_get_lower_bounds)

    def get_upper_bounds(self):
        return self._get_vec(self._lib.nlopt_get_upper_bounds)

    def set_xtol_abs(self, v):
        self._set_vec_or_scalar(self._lib.nlopt_set_xtol_abs, self._lib.nlopt_set_xtol_abs1, v)

    def get_xtol_abs(self):
        return self._get_vec(self._lib.nlopt_get_xtol_abs)

    def set_x_weights(self, v):
        self._set_vec_or_scalar(self._lib.nlopt_set_x_weights, self._lib.nlopt_set_x_weights1, v)

    def get_x_weights(self):
        return self._get_vec(self._lib.nlopt_get_x_weights)

    def set_initial_step(self, v):
        self._set_vec_or_scalar(self._lib.nlopt_set_initial_step, self._lib.nlopt_set_initial_step1, v)

    def get_initial_step(self, x):
        xa = _as_f64(x, self._n)
        a = np.empty(self._n)
        self._check(self._lib.nlopt_get_initial_step(self._h, _ptr(xa), _ptr(a)))
        return a

    def set_default_initial_step(self, x):
        xa = _as_f64(x, self._n)
        self._check(self._lib.nlopt_set_default_initial_step(self._h, _ptr(xa)))

    def set_local_optimizer(self, lo: "opt"):
        self._check(self._lib.nlopt_set_local_optimizer(self._h, lo._h))

    def force_stop(self):
        self._check(self._lib.nlopt_force_stop(self._h))

    def set_force_stop(self, v):
        self._check(self._lib.nlopt_set_force_stop(self._h, int(v)))

    def get_force_stop(self):
        return self._lib.nlopt_get_force_stop(self._h)


def _scalar_accessors():
    # nlopt.hpp NLOPT_GETSET (:546-568)
    for name, conv in (("stopval", float), ("ftol_rel", float), ("ftol_abs", float), ("xtol_rel", float),
                       ("maxeval", int), ("maxtime", float), ("population", int), ("vector_storage", int)):
        def setter(self, v, _n=name, _c=conv):
            self._check(getattr(self._lib, "nlopt_set_" + _n)(self._h, _c(v)))

        def getter(self, _n=name):
            return getattr(self._lib, "nlopt_get_" + _n)(self._h)

        setattr(opt, "set_" + name, setter)
        setattr(opt, "get_" + name, getter)


_scalar_accessors()


def algorithm_name(a):
    return default_library().nlopt_algorithm_name(int(a)).decode()


def version_major():
    v = [C.c_int() for _ in range(3)]
    default_library().nlopt_version(*[C.byref(i) for i in v])
    return v[0].value


def device_count():
    return default_library().nlopt_b200_device_count()


__all__ = ["opt", "Library", "RoundoffLimited", "ForcedStop", "CudaFunctor", "CompileError", "algorithm_name", "device_count",
           "NLOPT_B200_DFUNC"] + _ALG_NAMES
