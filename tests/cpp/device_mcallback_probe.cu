// device_mcallback_probe.cu -- vector test functors for the multi-row map / fold kernels of include/nlopt_b200_device.cuh.
//
// User code of the library, built like device_callback_probe.cu: tests/test_device_mconstraints_gpu.py compiles it into
// tests/_build/ and compares every component total handed to finish() with the model of the scalar summation order.
// Component i of a vector functor with first id k_id is the scalar probe functor with id k_id + i:
//
//   TermMF<M>   t_ij = x[jl] * 2^(k_id + i)                                   exact, depends on x
//   HashMF<M>   t_ij = (2 u01(seed, k_id + i, j) - 1) * 2^e_ij,  e_ij in [-40, 40]   does not depend on x
//
// Each visit of a variable is counted once, whatever M: a kernel that visits every variable once per component shows
// up as M visits.  The error and gradient-call counters are those of the scalar probe.  finish() logs component i's total
// under id k_id + i and returns total + offset.  No assert and no trap: a wrong index shows up as a failed comparison.
#include <cmath>
#include <vector>

#include "../../include/nlopt_b200_device.cuh"
#include "../../nlopt_b200/csrc/synth.cuh"

namespace {

constexpr int kMaxIds = 64;
std::vector<double> g_totals[kMaxIds];       // every component total passed to finish(), per id, in call order

struct Witness {
    unsigned *visits;            // [n_local]
    unsigned *errors;            // [1]
    unsigned *grad_calls;        // [1]
    unsigned long long n, j0;
    long long n_local;

    __device__ bool see(unsigned long long j, unsigned long long n_, long long jl, long long n_local_, const double *grad) const
    {
        const bool in = jl >= 0 && jl < n_local;
        if (!in || j != j0 + (unsigned long long) jl || n_ != n || n_local_ != n_local) atomicAdd(errors, 1u);
        if (in) atomicAdd(visits + jl, 1u);
        if (grad) atomicAdd(grad_calls, 1u);
        return in;
    }
};

template <int M>
struct Log {
    int k_id;
    double offset;
    void finish(const double *s, double *c) const
    {
        for (int i = 0; i < M; ++i) {
            g_totals[k_id + i].push_back(s[i]);
            c[i] = s[i] + offset;
        }
    }
};

template <int M>
struct TermMF : Log<M> {
    static constexpr int m = M;
    Witness w;
    __device__ void operator()(unsigned long long j, unsigned long long n, long long jl, long long n_local, const double *x,
                               double *t, double *grad, long long grad_ld) const
    {
        const bool in = w.see(j, n, jl, n_local, grad);
        const double xj = in ? x[jl] : 0.0;
#pragma unroll
        for (int i = 0; i < M; ++i) {
            const double scale = ldexp(1.0, this->k_id + i);
            if (in && grad) grad[i * grad_ld] = scale;
            t[i] = in ? __dmul_rn(xj, scale) : 0.0;
        }
    }
};

template <int M>
struct HashMF : Log<M> {
    static constexpr int m = M;
    Witness w;
    unsigned long long seed;
    __device__ void operator()(unsigned long long j, unsigned long long n, long long jl, long long n_local, const double *,
                               double *t, double *grad, long long grad_ld) const
    {
        const bool in = w.see(j, n, jl, n_local, grad);
#pragma unroll
        for (int i = 0; i < M; ++i) {
            const unsigned k = (unsigned) (this->k_id + i);
            const double u = nb200::u01(seed, k, j);
            const int e = (int) __dmul_rn(nb200::u01(seed, k + 1000u, j), 81.0) - 40;
            if (in && grad) grad[i * grad_ld] = 1.0;
            t[i] = in ? __dmul_rn(__dsub_rn(__dmul_rn(2.0, u), 1.0), ldexp(1.0, e)) : 0.0;
        }
    }
};

Witness make_witness(unsigned long long n, unsigned *visits, unsigned *errors, unsigned *grad_calls)
{
    unsigned long long j0 = 0, cnt = n;
    nlopt_b200_shard_range(n, nlopt_b200_comm_rank(), nlopt_b200_comm_world(), &j0, &cnt);
    return Witness{visits, errors, grad_calls, n, j0, (long long) cnt};
}

template <int M>
struct Ops {
    static void *make(int kind, int k_id, unsigned long long seed, double offset, const Witness &w)
    {
        if (kind == 0) {
            auto *f = new TermMF<M>;
            f->k_id = k_id; f->offset = offset; f->w = w;
            return f;
        }
        auto *f = new HashMF<M>;
        f->k_id = k_id; f->offset = offset; f->w = w; f->seed = seed;
        return f;
    }
    static void destroy(int kind, void *f)
    {
        if (kind == 0) delete static_cast<TermMF<M> *>(f);
        else delete static_cast<HashMF<M> *>(f);
    }
    template <class F>
    static int add(nlopt_opt opt, const F *f, int equality, const double *tol)
    {
        return equality ? nlopt_b200::add_equality_mconstraint(opt, f, tol) : nlopt_b200::add_inequality_mconstraint(opt, f, tol);
    }
    static int reg(nlopt_opt opt, int kind, void *f, int equality, const double *tol)
    {
        return kind == 0 ? add(opt, static_cast<const TermMF<M> *>(f), equality, tol)
                         : add(opt, static_cast<const HashMF<M> *>(f), equality, tol);
    }
    static void *fn(int kind)
    {
        return kind == 0 ? (void *) &nlopt_b200::detail::mtrampoline2<TermMF<M>> : (void *) &nlopt_b200::detail::mtrampoline2<HashMF<M>>;
    }
    static void *fin(int kind)
    {
        return kind == 0 ? (void *) &nlopt_b200::detail::mfinish2<TermMF<M>> : (void *) &nlopt_b200::detail::mfinish2<HashMF<M>>;
    }
};

#define PROBE_WITH_M(m, CALL)                       \
    switch (m) {                                    \
    case 1: return Ops<1>::CALL;                    \
    case 3: return Ops<3>::CALL;                    \
    case 4: return Ops<4>::CALL;                    \
    case 16: return Ops<16>::CALL;                  \
    default: break;                                 \
    }

}  // namespace

extern "C" {

// kind 0: TermMF, 1: HashMF; m in {1, 3, 4, 16}; ids k_id .. k_id + m - 1.  The witness buffers are device pointers.
void *probe_mnew(int kind, int m, int k_id, unsigned long long seed, double offset, unsigned long long n, unsigned *visits,
                 unsigned *errors, unsigned *grad_calls)
{
    if (k_id < 0 || m < 1 || k_id + m > kMaxIds || (kind != 0 && kind != 1)) return nullptr;
    const Witness w = make_witness(n, visits, errors, grad_calls);
    PROBE_WITH_M(m, make(kind, k_id, seed, offset, w))
    return nullptr;
}

void probe_mfree(int kind, int m, void *f)
{
    PROBE_WITH_M(m, destroy(kind, f))
}

// the functor must outlive every optimisation of `opt`; tol: m entries or NULL
int probe_mregister(nlopt_opt opt, int kind, int m, void *f, int equality, const double *tol)
{
    PROBE_WITH_M(m, reg(opt, kind, f, equality, tol))
    return NLOPT_INVALID_ARGS;
}

// the nlopt_b200_dmfunc2 / nlopt_b200_dmfinish pair of a functor type, for registration through the C ABI
void *probe_mfunc_ptr(int kind, int m)
{
    PROBE_WITH_M(m, fn(kind))
    return nullptr;
}

void *probe_mfinish_ptr(int kind, int m)
{
    PROBE_WITH_M(m, fin(kind))
    return nullptr;
}

int probe_mtotals(int k_id, double *out, int cap)
{
    if (k_id < 0 || k_id >= kMaxIds) return -1;
    const std::vector<double> &v = g_totals[k_id];
    for (int i = 0; i < cap && i < (int) v.size(); ++i) out[i] = v[i];
    return (int) v.size();
}

void probe_mreset(void)
{
    for (std::vector<double> &v : g_totals) v.clear();
}

}  // extern "C"
