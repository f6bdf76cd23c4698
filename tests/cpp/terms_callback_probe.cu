// terms_callback_probe.cu -- problems.cu's __device__ functors registered either as functors (nlopt_b200_device.cuh) or
// as per-variable terms callbacks (nlopt_b200_dtfunc) that call the same functor once per variable.
//
// User code of the library, built like device_callback_probe.cu: tests/test_terms_callbacks_gpu.py compiles it into
// tests/_build/ and runs each problem both ways.  A terms callback writes exactly the functor's terms and gradient
// entries, so the library's reduction must give the functor's value bits, and the two runs must agree bit for bit.
#include <memory>
#include <vector>

#include "../../nlopt_b200/csrc/problem_functors.cuh"

namespace {

constexpr int kThreads = 256;

int grid_for(unsigned long long n)
{
    const unsigned long long g = (n + kThreads - 1) / kThreads;
    return (int) (g < 1 ? 1 : g > 2048 ? 2048 : g);
}

template <class F>
__global__ void scalar_terms_kernel(F f, nlopt_b200_shard sh, const double *x, double *grad, double *terms)
{
    const long long nl = (long long) sh.n_local;
    for (long long jl = (long long) blockIdx.x * blockDim.x + threadIdx.x; jl < nl; jl += (long long) gridDim.x * blockDim.x)
        terms[jl] = f(sh.j0 + (unsigned long long) jl, sh.n, jl, nl, x, grad ? grad + jl : nullptr);
}

template <class F>
__global__ void vector_terms_kernel(F f, nlopt_b200_shard sh, const double *x, double *grad, unsigned long long ld, double *terms)
{
    const long long nl = (long long) sh.n_local;
    for (long long jl = (long long) blockIdx.x * blockDim.x + threadIdx.x; jl < nl; jl += (long long) gridDim.x * blockDim.x) {
        double t[F::m];
        f(sh.j0 + (unsigned long long) jl, sh.n, jl, nl, x, t, grad ? grad + jl : nullptr, (long long) ld);
#pragma unroll
        for (int i = 0; i < F::m; ++i) terms[(unsigned long long) i * ld + jl] = t[i];
    }
}

// nlopt_b200_dtfunc of a scalar functor F (m == 1) and of a vector functor (m == F::m)
template <class F>
void scalar_terms(unsigned, const nlopt_b200_shard *sh, const double *x, double *grad, unsigned long long, double *terms,
                  void *data, void *stream)
{
    scalar_terms_kernel<F><<<grid_for(sh->n_local), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        *static_cast<const F *>(data), *sh, x, grad, terms);
}

template <class F>
void vector_terms(unsigned, const nlopt_b200_shard *sh, const double *x, double *grad, unsigned long long ld, double *terms,
                  void *data, void *stream)
{
    vector_terms_kernel<F><<<grid_for(sh->n_local), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        *static_cast<const F *>(data), *sh, x, grad, ld, terms);
}

std::vector<std::shared_ptr<void>> g_keep;      // functors of every registration, until probe_terms_reset()
std::vector<double *> g_rows;                   // device weight rows

// role 0: min objective, 1: max objective, 2: inequality, 3: equality; form 0: functor, 1: terms
template <class F>
int reg_scalar(nlopt_opt opt, std::shared_ptr<F> f, int role, int form, double tol)
{
    g_keep.push_back(f);
    namespace d = nlopt_b200::detail;
    const F *p = f.get();
    void *data = const_cast<F *>(p);
    const int halo = d::halo_of<F>::value;
    if (form == 0) {
        switch (role) {
        case 0: return nlopt_b200::set_min_objective(opt, p);
        case 1: return nlopt_b200::set_max_objective(opt, p);
        case 2: return nlopt_b200::add_inequality_constraint(opt, p, tol);
        default: return nlopt_b200::add_equality_constraint(opt, p, tol);
        }
    }
    switch (role) {
    case 0: return nlopt_b200_set_min_objective_terms(opt, &scalar_terms<F>, &d::finish2<F>, data, halo);
    case 1: return nlopt_b200_set_max_objective_terms(opt, &scalar_terms<F>, &d::finish2<F>, data, halo);
    case 2: return nlopt_b200_add_inequality_constraint_terms(opt, &scalar_terms<F>, &d::finish2<F>, data, tol, halo);
    default: return nlopt_b200_add_equality_constraint_terms(opt, &scalar_terms<F>, &d::finish2<F>, data, tol, halo);
    }
}

template <class F>
int reg_vector(nlopt_opt opt, std::shared_ptr<F> f, int role, int form, const double *tol)
{
    g_keep.push_back(f);
    namespace d = nlopt_b200::detail;
    const F *p = f.get();
    if (form == 0)
        return role == 3 ? nlopt_b200::add_equality_mconstraint(opt, p, tol) : nlopt_b200::add_inequality_mconstraint(opt, p, tol);
    return role == 3 ? nlopt_b200_add_equality_mconstraint_terms(opt, F::m, &vector_terms<F>, &d::mfinish2<F>, const_cast<F *>(p), tol, 0)
                     : nlopt_b200_add_inequality_mconstraint_terms(opt, F::m, &vector_terms<F>, &d::mfinish2<F>, const_cast<F *>(p), tol, 0);
}

// this rank's shard of `rows` weight rows of n entries (row-major on the host) on the device
double *upload_rows(nlopt_opt opt, const double *w_host, int rows)
{
    const unsigned n = nlopt_get_dimension(opt);
    unsigned long long j0 = 0, cnt = n;
    nlopt_b200_shard_range(n, nlopt_b200_comm_rank(), nlopt_b200_comm_world(), &j0, &cnt);
    double *w = nullptr;
    if (cudaMalloc(&w, (size_t) rows * (cnt ? cnt : 1) * sizeof(double)) != cudaSuccess) return nullptr;
    g_rows.push_back(w);
    if (cnt) cudaMemcpy2D(w, cnt * sizeof(double), w_host + j0, (size_t) n * sizeof(double), cnt * sizeof(double), rows,
                          cudaMemcpyHostToDevice);
    return w;
}

}  // namespace

extern "C" {

// kind  0 SimpDev(seed, eps = p[0])      1 MeanDev(offset = p[0])       2 LinearDev(w: n, b = p[0])
//       3 SphereDev(r = p[0])            4 RosenbrockDev (halo 1)       5 QuadraticDev(seed)
//       6 LinearRowsDev<4>(w: [4][n], b = p[0..3])                      7 BlockMeanDev<4>(target = p[0..3])
// role  0 min objective, 1 max objective, 2 inequality, 3 equality (kinds 6, 7: 2 or 3 only; tol: 4 entries or NULL)
// form  0 the functor (nlopt_b200_device.cuh), 1 a terms callback calling the functor per variable
int probe_terms_register(nlopt_opt opt, int kind, int role, int form, unsigned long long seed, const double *p, const double *w,
                         const double *tol)
{
    const double n = (double) nlopt_get_dimension(opt), t0 = tol ? tol[0] : 0.0;
    switch (kind) {
    case 0: { auto f = std::make_shared<SimpDev>(); f->seed = seed; f->eps = p[0]; return reg_scalar(opt, f, role, form, t0); }
    case 1: return reg_scalar(opt, std::make_shared<MeanDev>(MeanDev{1.0 / n, p[0]}), role, form, t0);
    case 2: {
        double *wd = upload_rows(opt, w, 1);
        return wd ? reg_scalar(opt, std::make_shared<LinearDev>(LinearDev{wd, p[0]}), role, form, t0) : NLOPT_OUT_OF_MEMORY;
    }
    case 3: return reg_scalar(opt, std::make_shared<SphereDev>(SphereDev{1.0 / n, p[0]}), role, form, t0);
    case 4: return reg_scalar(opt, std::make_shared<RosenbrockDev>(), role, form, t0);
    case 5: { auto f = std::make_shared<QuadraticDev>(); f->seed = seed; return reg_scalar(opt, f, role, form, t0); }
    case 6: {
        double *wd = upload_rows(opt, w, 4);
        if (!wd) return NLOPT_OUT_OF_MEMORY;
        unsigned long long j0 = 0, cnt = 0;
        nlopt_b200_shard_range(nlopt_get_dimension(opt), nlopt_b200_comm_rank(), nlopt_b200_comm_world(), &j0, &cnt);
        auto f = std::make_shared<LinearRowsDev<4>>();
        f->w = wd;
        f->w_ld = (long long) cnt;
        for (int i = 0; i < 4; ++i) f->b[i] = p[i];
        return reg_vector(opt, f, role, form, tol);
    }
    case 7: {
        const unsigned long long nn = nlopt_get_dimension(opt);
        auto f = std::make_shared<BlockMeanDev<4>>();
        for (int i = 0; i <= 4; ++i) f->edge[i] = (unsigned long long) i * nn / 4;
        for (int i = 0; i < 4; ++i) {
            f->inv_len[i] = 1.0 / (double) (f->edge[i + 1] - f->edge[i]);
            f->target[i] = p[i];
        }
        return reg_vector(opt, f, role, form, tol);
    }
    default: return NLOPT_INVALID_ARGS;
    }
}

// frees every functor and weight row; call when no optimiser that uses them runs any more
void probe_terms_reset(void)
{
    cudaDeviceSynchronize();
    g_keep.clear();
    for (double *w : g_rows) cudaFree(w);
    g_rows.clear();
}

}  // extern "C"
