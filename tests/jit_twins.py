"""Source twins of nlopt_b200/csrc/problem_functors.cuh's functors, for nlopt_b200.CudaFunctor (compiled at run time).

Each twin has the nvcc functor's members in the same order and the same per-variable expressions, so its parameter
bytes are the functor object's bytes and its terms are the functor's terms; the finishes are the functors' host finishes
in Python.  Device weights are passed as pointers in the parameters.  The hash is synth.cuh's (tests/synth.py).
"""
import struct

SOURCE = r"""
namespace twin {

__device__ inline unsigned long long mix64(unsigned long long z)
{
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__device__ inline double u01(unsigned long long seed, unsigned k, unsigned long long j)
{
    const unsigned long long base = (seed + k) * 0x9E3779B97F4A7C15ull;
    return (double) (mix64(base + j) >> 11) * 0x1.0p-53;
}

struct RosenbrockDev {
    static constexpr int halo = 1;
    __device__ double operator()(unsigned long long j, unsigned long long n, long long jl, long long,
                                 const double *x, double *grad_j) const
    {
        const double xj = x[jl];
        double term = 0.0, gsum = 0.0;
        if (j + 1 < n) {
            const double d = __dsub_rn(x[jl + 1], __dmul_rn(xj, xj)), e = __dsub_rn(1.0, xj);
            term = __dadd_rn(__dmul_rn(__dmul_rn(100.0, d), d), __dmul_rn(e, e));
            gsum = __dadd_rn(0.0, __dsub_rn(__dmul_rn(__dmul_rn(-400.0, xj), d), __dmul_rn(2.0, e)));
        }
        if (j > 0) {
            const double xm = x[jl - 1];
            gsum = __dadd_rn(gsum, __dmul_rn(200.0, __dsub_rn(xj, __dmul_rn(xm, xm))));
        }
        if (grad_j) *grad_j = gsum;
        return term;
    }
};

struct LinearDev {
    const double *w;
    double b;
    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double wj = w[jl];
        if (grad_j) *grad_j = wj;
        return __dmul_rn(wj, x[jl]);
    }
};

struct QuadraticDev {
    unsigned long long seed;
    __device__ double operator()(unsigned long long j, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double a = __dadd_rn(1.0, u01(seed, 0, j));
        const double b = __dsub_rn(__dmul_rn(2.0, u01(seed, 1, j)), 1.0);
        const double d = __dsub_rn(x[jl], b);
        const double ad = __dmul_rn(a, d);
        if (grad_j) *grad_j = ad;
        return __dmul_rn(ad, d);
    }
};

struct SimpDev {
    unsigned long long seed;
    double eps;
    __device__ double operator()(unsigned long long j, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double a = __dadd_rn(0.5, u01(seed, 0, j));
        const double xj = x[jl], x2 = __dmul_rn(xj, xj), x3 = __dmul_rn(x2, xj);
        const double ome = __dsub_rn(1.0, eps);
        const double d = __dadd_rn(eps, __dmul_rn(ome, x3));
        if (grad_j) *grad_j = -__ddiv_rn(__dmul_rn(__dmul_rn(a, __dmul_rn(ome, 3.0)), x2), __dmul_rn(d, d));
        return __ddiv_rn(a, d);
    }
};

struct MeanDev {
    double inv_n, offset;
    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        if (grad_j) *grad_j = inv_n;
        return x[jl];
    }
};

struct SphereDev {
    double inv_n, r;
    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double xj = x[jl];
        if (grad_j) *grad_j = __dmul_rn(2.0, xj);
        return __dmul_rn(xj, xj);
    }
};

template <int M>
struct LinearRowsDev {
    static constexpr int m = M;
    const double *w;
    long long w_ld;
    double b[M];
    __device__ void operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x, double *t,
                               double *grad, long long grad_ld) const
    {
        const double xj = x[jl];
#pragma unroll
        for (int i = 0; i < M; ++i) {
            const double wij = w[i * w_ld + jl];
            if (grad) grad[i * grad_ld] = wij;
            t[i] = __dmul_rn(wij, xj);
        }
    }
};

template <int M>
struct BlockMeanDev {
    static constexpr int m = M;
    unsigned long long edge[M + 1];
    double inv_len[M], target[M];
    __device__ void operator()(unsigned long long j, unsigned long long, long long jl, long long, const double *x, double *t,
                               double *grad, long long grad_ld) const
    {
        const double xj = x[jl];
#pragma unroll
        for (int i = 0; i < M; ++i) {
            const bool in = j >= edge[i] && j < edge[i + 1];
            if (grad) grad[i * grad_ld] = in ? inv_len[i] : 0.0;
            t[i] = in ? xj : 0.0;
        }
    }
};

// terms read from a device table (they do not depend on x): the reduction alone
struct TableDev {
    const double *t;
    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *,
                                 double *grad_j) const
    {
        if (grad_j) *grad_j = 1.0;
        return t[jl];
    }
};

template <int M>
struct TableRowsDev {
    static constexpr int m = M;
    const double *t;
    long long ld;
    __device__ void operator()(unsigned long long, unsigned long long, long long jl, long long, const double *, double *out,
                               double *grad, long long grad_ld) const
    {
#pragma unroll
        for (int i = 0; i < M; ++i) {
            if (grad) grad[i * grad_ld] = 0.0;
            out[i] = t[i * ld + jl];
        }
    }
};

}  // namespace twin
"""

_cache = {}


def functor(name):
    """the CudaFunctor of twin `name` (e.g. "SimpDev", "LinearRowsDev<4>"), compiled once per process"""
    import nlopt_b200 as nl
    if name not in _cache:
        _cache[name] = nl.CudaFunctor(SOURCE, "twin::" + name)
    return _cache[name]


def simp(seed, eps):
    return struct.pack("<Qd", seed, eps)


def quadratic(seed):
    return struct.pack("<Q", seed)


def two_doubles(a, b):                      # MeanDev(inv_n, offset), SphereDev(inv_n, r)
    return struct.pack("<dd", a, b)


def linear(w_ptr, b):
    return struct.pack("<Qd", w_ptr, b)


def linear_rows(w_ptr, w_ld, b):
    return struct.pack(f"<Qq{len(b)}d", w_ptr, w_ld, *b)


def block_means(n, target):
    m = len(target)
    edge = [i * n // m for i in range(m + 1)]
    inv_len = [1.0 / float(edge[i + 1] - edge[i]) for i in range(m)]
    return struct.pack(f"<{m + 1}Q{m}d{m}d", *edge, *inv_len, *target), inv_len
