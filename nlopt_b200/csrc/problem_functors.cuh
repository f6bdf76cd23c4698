// problem_functors.cuh -- the __device__ functors of the benchmark / test problems (problems.cu), shared with the test
// probes that feed the same per-variable terms through other callback forms.  Per-variable expressions use un-fused
// IEEE operations in the same order as tests/problems.py (numpy).
#pragma once

#include "../../include/nlopt_b200_device.cuh"
#include "synth.cuh"

namespace {

// ---- device functors ---------------------------------------------------------------------------------
struct RosenbrockDev {
    static constexpr int halo = 1;           // reads x[jl - 1] and x[jl + 1] across shard boundaries
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
    double finish(double s) const { return s; }
};

struct LinearDev {
    const double *w;        // device, this rank's shard of the weight row
    double b;
    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double wj = w[jl];
        if (grad_j) *grad_j = wj;
        return __dmul_rn(wj, x[jl]);
    }
    double finish(double s) const { return s - b; }
};

struct QuadraticDev {
    unsigned long long seed;
    __device__ double operator()(unsigned long long j, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double a = __dadd_rn(1.0, nb200::u01(seed, 0, j));
        const double b = __dsub_rn(__dmul_rn(2.0, nb200::u01(seed, 1, j)), 1.0);
        const double d = __dsub_rn(x[jl], b);
        const double ad = __dmul_rn(a, d);
        if (grad_j) *grad_j = ad;
        return __dmul_rn(ad, d);
    }
    double finish(double s) const { return 0.5 * s; }
};

// synthetic SIMP compliance (BASELINE config 4, SURVEY.md 8(d)): f(x) = sum_j a_j / (eps + (1 - eps) x_j^3),
// a_j = 0.5 + u01(seed, 0, j).  Same expression order as nb200p_simp_host below.
struct SimpDev {
    unsigned long long seed;
    double eps;
    __device__ double operator()(unsigned long long j, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double a = __dadd_rn(0.5, nb200::u01(seed, 0, j));
        const double xj = x[jl], x2 = __dmul_rn(xj, xj), x3 = __dmul_rn(x2, xj);
        const double ome = __dsub_rn(1.0, eps);
        const double d = __dadd_rn(eps, __dmul_rn(ome, x3));
        if (grad_j) *grad_j = -__ddiv_rn(__dmul_rn(__dmul_rn(a, __dmul_rn(ome, 3.0)), x2), __dmul_rn(d, d));
        return __ddiv_rn(a, d);
    }
    double finish(double s) const { return s; }
};

struct MeanDev {
    double inv_n, offset;
    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        if (grad_j) *grad_j = inv_n;
        return x[jl];
    }
    double finish(double s) const { return s * inv_n + offset; }
};

// nonlinear equality mean(x_j^2) - r: term x_j * x_j, gradient 2 x_j, each one IEEE operation
struct SphereDev {
    double inv_n, r;
    __device__ double operator()(unsigned long long, unsigned long long, long long jl, long long, const double *x,
                                 double *grad_j) const
    {
        const double xj = x[jl];
        if (grad_j) *grad_j = __dmul_rn(2.0, xj);
        return __dmul_rn(xj, xj);
    }
    double finish(double s) const { return s * inv_n - r; }
};

// -F, for maximisation: term -F(...), gradient -grad F, finish(s) = -F.finish(-s).  Negation is exact and a sum of
// negated terms in the same tree is the negated sum, so the library's minimisation of -(-F) -- value and gradient
// negated once more -- sees F's bits: a max run of Negated<F> is the min run of F.
template <class F>
struct Negated {
    static constexpr int halo = nlopt_b200::detail::halo_of<F>::value;
    F f;
    __device__ double operator()(unsigned long long j, unsigned long long n, long long jl, long long n_local,
                                 const double *x, double *grad_j) const
    {
        const double t = f(j, n, jl, n_local, x, grad_j);
        if (grad_j) *grad_j = -*grad_j;
        return -t;
    }
    double finish(double s) const { return -f.finish(-s); }
};

// ---- vector functors (one pass over x for M constraint rows) ---------------------------------------------
// M dense linear rows c_i(x) = w_i.x - b_i: the one-functor form of M LinearDev.  Component i has LinearDev's terms
// w_ij * x_j, so it has the same bits as LinearDev with row w_i.
template <int M>
struct LinearRowsDev {
    static constexpr int m = M;
    const double *w;        // device, [M][w_ld]: this rank's shard of each weight row
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
    void finish(const double *s, double *c) const
    {
        for (int i = 0; i < M; ++i) c[i] = s[i] - b[i];
    }
};

// local volumes: c_i(x) = mean of x over the block [i n / M, (i + 1) n / M) - target_i.  Component i's term is x_j
// inside block i and +0.0 outside; its gradient 1 / |block i| inside and 0 outside.
template <int M>
struct BlockMeanDev {
    static constexpr int m = M;
    unsigned long long edge[M + 1];     // block i = [edge[i], edge[i + 1])
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
    void finish(const double *s, double *c) const
    {
        for (int i = 0; i < M; ++i) c[i] = s[i] * inv_len[i] - target[i];
    }
};

}  // namespace
