// device_callback_probe.cu -- test functors for the map / reduce kernels of include/nlopt_b200_device.cuh.
//
// User code of the library, like nlopt_b200/csrc/problems.cu: it includes only the public headers (plus the counter
// hash of synth.cuh) and registers its functors through the template front ends of nlopt_b200_device.cuh, in either
// form (dfunc2: set_min_objective / add_inequality_constraint; dfunc: the _sync twins).  tests/test_device_callbacks_gpu.py
// compiles it into tests/_build/ and compares every total the library hands to finish() with a model of the kernels'
// summation order.
//
//   TermF   t_j = x[jl] * 2^k_id                                   exact, depends on x
//   HashF   t_j = (2 u01(seed, k_id, j) - 1) * 2^e_j,  e_j in [-40, 40]   does not depend on x
//
// Both functors report what they saw through device counters that the test allocates: a visit count per variable,
// an error count (wrong j, n or n_local, or jl outside [0, n_local)) and the number of calls with a gradient pointer.
// They contain no assert and no trap: a wrong index shows up as a failed comparison, never as a device fault.
#include <cmath>
#include <vector>

#include "../../include/nlopt_b200_device.cuh"
#include "../../nlopt_b200/csrc/synth.cuh"

namespace {

constexpr int kMaxIds = 64;
std::vector<double> g_totals[kMaxIds];       // every total passed to finish(), per k_id, in call order

struct Witness {
    unsigned *visits;            // [n_local]
    unsigned *errors;            // [1]
    unsigned *grad_calls;        // [1]
    unsigned long long n, j0;    // what the library must pass
    long long n_local;

    // true when jl indexes this rank's shard (x[jl] and grad_j may be touched)
    __device__ bool see(unsigned long long j, unsigned long long n_, long long jl, long long n_local_, const double *grad_j) const
    {
        const bool in = jl >= 0 && jl < n_local;
        if (!in || j != j0 + (unsigned long long) jl || n_ != n || n_local_ != n_local) atomicAdd(errors, 1u);
        if (in) atomicAdd(visits + jl, 1u);
        if (grad_j) atomicAdd(grad_calls, 1u);
        return in;
    }
};

struct TermF {
    Witness w;
    double scale;                // 2^k_id
    double offset;               // added by finish()
    int k_id;

    __device__ double operator()(unsigned long long j, unsigned long long n, long long jl, long long n_local,
                                 const double *x, double *grad_j) const
    {
        if (!w.see(j, n, jl, n_local, grad_j)) return 0.0;
        if (grad_j) *grad_j = scale;
        return __dmul_rn(x[jl], scale);
    }
    double finish(double total) const
    {
        g_totals[k_id].push_back(total);
        return total + offset;
    }
};

struct HashF {
    Witness w;
    unsigned long long seed;
    double offset;
    int k_id;

    __device__ double operator()(unsigned long long j, unsigned long long n, long long jl, long long n_local,
                                 const double *, double *grad_j) const
    {
        if (!w.see(j, n, jl, n_local, grad_j)) return 0.0;
        const double u = nb200::u01(seed, (unsigned) k_id, j);
        const int e = (int) __dmul_rn(nb200::u01(seed, (unsigned) k_id + 1000u, j), 81.0) - 40;
        if (grad_j) *grad_j = 1.0;
        return __dmul_rn(__dsub_rn(__dmul_rn(2.0, u), 1.0), ldexp(1.0, e));
    }
    double finish(double total) const
    {
        g_totals[k_id].push_back(total);
        return total + offset;
    }
};

Witness make_witness(unsigned long long n, unsigned *visits, unsigned *errors, unsigned *grad_calls)
{
    unsigned long long j0 = 0, cnt = n;
    nlopt_b200_shard_range(n, nlopt_b200_comm_rank(), nlopt_b200_comm_world(), &j0, &cnt);
    return Witness{visits, errors, grad_calls, n, j0, (long long) cnt};
}

template <class F>
int register_functor(nlopt_opt opt, const F *f, int sync, int constraint, double tol)
{
    if (sync)
        return constraint ? nlopt_b200::add_inequality_constraint_sync(opt, f, tol) : nlopt_b200::set_min_objective_sync(opt, f);
    return constraint ? nlopt_b200::add_inequality_constraint(opt, f, tol) : nlopt_b200::set_min_objective(opt, f);
}

}  // namespace

extern "C" {

// kind 0: TermF, 1: HashF.  The witness buffers are device pointers owned by the caller.
void *probe_new(int kind, int k_id, unsigned long long seed, double offset, unsigned long long n, unsigned *visits,
                unsigned *errors, unsigned *grad_calls)
{
    if (k_id < 0 || k_id >= kMaxIds) return nullptr;
    const Witness w = make_witness(n, visits, errors, grad_calls);
    if (kind == 0) return new TermF{w, ldexp(1.0, k_id), offset, k_id};
    if (kind == 1) return new HashF{w, seed, offset, k_id};
    return nullptr;
}

void probe_free(int kind, void *f)
{
    if (kind == 0) delete static_cast<TermF *>(f);
    else if (kind == 1) delete static_cast<HashF *>(f);
}

// the functor must outlive every optimisation of `opt`
int probe_register(nlopt_opt opt, int kind, void *f, int sync, int constraint, double tol)
{
    if (kind == 0) return register_functor(opt, static_cast<const TermF *>(f), sync, constraint, tol);
    if (kind == 1) return register_functor(opt, static_cast<const HashF *>(f), sync, constraint, tol);
    return NLOPT_INVALID_ARGS;
}

// copies up to `cap` logged totals of k_id into out; returns how many were logged
int probe_totals(int k_id, double *out, int cap)
{
    if (k_id < 0 || k_id >= kMaxIds) return -1;
    const std::vector<double> &v = g_totals[k_id];
    for (int i = 0; i < cap && i < (int) v.size(); ++i) out[i] = v[i];
    return (int) v.size();
}

void probe_reset(void)
{
    for (std::vector<double> &v : g_totals) v.clear();
}

}  // extern "C"
