// problems.cu -> libnlopt_b200_problems.so : the benchmark / test problems of BASELINE.json as
// USER code of the library (it only uses the public headers).  Device-resident versions are
// written as __device__ functors through include/nlopt_b200_device.cuh; host versions are plain
// nlopt_func callbacks usable with any library exporting the NLopt ABI (ours or the reference).
//
//   chained Rosenbrock  (formula of reference test/testfuncs.c:124-139)   -- config 3 objective
//   dense linear inequality  c(x) = w.x - b  with a caller-supplied weight row -- config 3 constraints
//   separable quadratic 1/2 sum a_j (x_j - b_j)^2, a, b from the counter hash  -- config 2 objective
//   mean constraint  sum x / n + offset                                         -- config 2 / 4 constraint
//
// Per-variable expressions use un-fused IEEE operations in the same order as tests/problems.py
// (numpy), so device gradients are bit-identical to the host callbacks' gradients.  The device
// functors themselves are in problem_functors.cuh.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "problem_functors.cuh"

namespace {

double g_cb_seconds = 0.0;
struct Tick {
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    ~Tick() { g_cb_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); }
};

template <class F>
int set_objective(nlopt_opt opt, const F *f, int sync, int maximize)
{
    if (maximize) return sync ? nlopt_b200::set_max_objective_sync(opt, f) : nlopt_b200::set_max_objective(opt, f);
    return sync ? nlopt_b200::set_min_objective_sync(opt, f) : nlopt_b200::set_min_objective(opt, f);
}

template <class F>
int add_eq(nlopt_opt opt, const F *f, double tol, int sync)
{
    return sync ? nlopt_b200::add_equality_constraint_sync(opt, f, tol) : nlopt_b200::add_equality_constraint(opt, f, tol);
}

// Op<M>::run(args...) for M in {1, 2, 4, 8, 16}
template <template <int> class Op, class... A>
int with_m(unsigned m, A... a)
{
    switch (m) {
    case 1: return Op<1>::run(a...);
    case 2: return Op<2>::run(a...);
    case 4: return Op<4>::run(a...);
    case 8: return Op<8>::run(a...);
    case 16: return Op<16>::run(a...);
    default: return NLOPT_INVALID_ARGS;
    }
}

template <class F>
int add_m(nlopt_opt opt, const F *f, const double *tol, int equality)
{
    return equality ? nlopt_b200::add_equality_mconstraint(opt, f, tol) : nlopt_b200::add_inequality_mconstraint(opt, f, tol);
}

}  // namespace

struct nb200p_lin_data {
    const double *w;
    double b;
};
struct nb200p_quad_data {
    unsigned long long seed;
};
struct nb200p_mean_data {
    double offset;
};
struct nb200p_simp_data {
    unsigned long long seed;
    double eps;
};

struct nb200p_problem_s {
    RosenbrockDev rosen;
    QuadraticDev quad;
    std::vector<LinearDev *> lin;
    std::vector<MeanDev *> mean;
    std::vector<SphereDev *> sphere;
    std::vector<double *> dev_rows;
    std::vector<nb200p_lin_data *> lin_host;
    SimpDev simp;
    Negated<RosenbrockDev> nrosen;          // maximisation twins (nb200p_set_*_device_max)
    Negated<QuadraticDev> nquad;
    Negated<SimpDev> nsimp;
    std::vector<void *> misc_host;          // small data records of the host callbacks (freed with the problem)
    std::vector<std::shared_ptr<void>> vec; // vector functors (LinearRowsDev<M>, BlockMeanDev<M>)
};

namespace {

template <int M>
struct AddLinearRows {
    // w_host: [M][n] row-major, b: M offsets
    static int run(nb200p_problem_s *p, nlopt_opt opt, const double *w_host, const double *b, const double *tol, int equality)
    {
        const unsigned n = nlopt_get_dimension(opt);
        unsigned long long j0 = 0, cnt = n;
        nlopt_b200_shard_range(n, nlopt_b200_comm_rank(), nlopt_b200_comm_world(), &j0, &cnt);
        double *w = nullptr;
        if (cudaMalloc(&w, (size_t) M * (cnt ? cnt : 1) * sizeof(double)) != cudaSuccess) return NLOPT_OUT_OF_MEMORY;
        p->dev_rows.push_back(w);
        if (cnt && cudaMemcpy2D(w, cnt * sizeof(double), w_host + j0, (size_t) n * sizeof(double), cnt * sizeof(double), M,
                                cudaMemcpyHostToDevice) != cudaSuccess)
            return NLOPT_FAILURE;
        auto f = std::make_shared<LinearRowsDev<M>>();
        f->w = w;
        f->w_ld = (long long) cnt;
        for (int i = 0; i < M; ++i) f->b[i] = b[i];
        p->vec.push_back(f);
        return add_m(opt, f.get(), tol, equality);
    }
};

template <int M>
struct AddBlockMean {
    static int run(nb200p_problem_s *p, nlopt_opt opt, const double *target, const double *tol, int equality)
    {
        const unsigned long long n = nlopt_get_dimension(opt);
        auto f = std::make_shared<BlockMeanDev<M>>();
        for (int i = 0; i <= M; ++i) f->edge[i] = (unsigned long long) i * n / M;
        for (int i = 0; i < M; ++i) {
            f->inv_len[i] = 1.0 / (double) (f->edge[i + 1] - f->edge[i]);
            f->target[i] = target[i];
        }
        p->vec.push_back(f);
        return add_m(opt, f.get(), tol, equality);
    }
};

}  // namespace

// Tridiagonal preconditioner vpre = sign * A v, A = tridiag(-1, d_j, -1) (tests/test_host_driver.py: precond_problem;
// sign -1 for the maximisation of the negated problem), one rank.  The operations are those of the PyTorch form
// ((d_j v_j - v_{j+1}) - v_{j-1}, then the sign), so both give the same bits.
struct nb200p_tridiag_data {
    const double *d;     // device, n entries
    double sign;
};

__global__ void nb200p_tridiag_kernel(const double *__restrict__ d, const double *__restrict__ v, double sign,
                                      unsigned long long n, double *__restrict__ vpre)
{
    for (unsigned long long j = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; j < n;
         j += (unsigned long long) gridDim.x * blockDim.x) {
        double o = __dmul_rn(d[j], v[j]);
        if (j + 1 < n) o = __dsub_rn(o, v[j + 1]);
        if (j > 0) o = __dsub_rn(o, v[j - 1]);
        vpre[j] = __dmul_rn(sign, o);
    }
}

extern "C" {

nb200p_problem_s *nb200p_create(void) { return new nb200p_problem_s; }

void nb200p_destroy(nb200p_problem_s *p)
{
    if (!p) return;
    for (double *d : p->dev_rows) cudaFree(d);
    for (LinearDev *l : p->lin) delete l;
    for (MeanDev *m : p->mean) delete m;
    for (SphereDev *s : p->sphere) delete s;
    for (nb200p_lin_data *l : p->lin_host) delete l;
    for (void *q : p->misc_host) std::free(q);
    delete p;
}

double nb200p_callback_seconds(void) { return g_cb_seconds; }
void nb200p_reset_callback_seconds(void) { g_cb_seconds = 0.0; }

// ---- device registration -------------------------------------------------------------------------------
int nb200p_set_rosenbrock_device(nb200p_problem_s *p, nlopt_opt opt)
{
    return nlopt_b200::set_min_objective(opt, &p->rosen);
}

static LinearDev *make_linear(nb200p_problem_s *p, nlopt_opt opt, const double *w_host_full, double b)
{
    const unsigned n = nlopt_get_dimension(opt);
    unsigned long long j0 = 0, cnt = n;
    nlopt_b200_shard_range(n, nlopt_b200_comm_rank(), nlopt_b200_comm_world(), &j0, &cnt);
    double *w = nullptr;
    if (cudaMalloc(&w, (cnt ? cnt : 1) * sizeof(double)) != cudaSuccess) return nullptr;
    cudaMemcpy(w, w_host_full + j0, cnt * sizeof(double), cudaMemcpyHostToDevice);
    p->dev_rows.push_back(w);
    LinearDev *l = new LinearDev{w, b};
    p->lin.push_back(l);
    return l;
}

int nb200p_add_linear_device(nb200p_problem_s *p, nlopt_opt opt, const double *w_host_full, double b, double tol)
{
    LinearDev *l = make_linear(p, opt, w_host_full, b);
    return l ? nlopt_b200::add_inequality_constraint(opt, l, tol) : NLOPT_OUT_OF_MEMORY;
}

// equality constraints (NLOPT_AUGLAG*); sync != 0 registers the synchronous form (nlopt_b200_dfunc)
int nb200p_add_linear_device_eq(nb200p_problem_s *p, nlopt_opt opt, const double *w_host_full, double b, double tol, int sync)
{
    LinearDev *l = make_linear(p, opt, w_host_full, b);
    return l ? add_eq(opt, l, tol, sync) : NLOPT_OUT_OF_MEMORY;
}

int nb200p_add_mean_device_eq(nb200p_problem_s *p, nlopt_opt opt, double offset, double tol, int sync)
{
    MeanDev *m = new MeanDev{1.0 / (double) nlopt_get_dimension(opt), offset};
    p->mean.push_back(m);
    return add_eq(opt, m, tol, sync);
}

int nb200p_add_sphere_device_eq(nb200p_problem_s *p, nlopt_opt opt, double r, double tol, int sync)
{
    SphereDev *s = new SphereDev{1.0 / (double) nlopt_get_dimension(opt), r};
    p->sphere.push_back(s);
    return add_eq(opt, s, tol, sync);
}

// vector constraints, m in {1, 2, 4, 8, 16}; equality != 0 registers h(x) = 0 (NLOPT_AUGLAG*).  tol: m entries or NULL.
// m dense linear rows w_k.x - b_k, w_host_rows [m][n] row-major (copied to the device here)
int nb200p_add_linear_rows_device(nb200p_problem_s *p, nlopt_opt opt, unsigned m, const double *w_host_rows, const double *b,
                                  const double *tol, int equality)
{
    return with_m<AddLinearRows>(m, p, opt, w_host_rows, b, tol, equality);
}

// block means: c_i = mean(x over [i n / m, (i + 1) n / m)) - target_i
int nb200p_add_block_mean_device(nb200p_problem_s *p, nlopt_opt opt, unsigned m, const double *target, const double *tol,
                                 int equality)
{
    return with_m<AddBlockMean>(m, p, opt, target, tol, equality);
}

// the synchronous forms of the quadratic / SIMP objectives and the mean inequality
int nb200p_set_quadratic_device_sync(nb200p_problem_s *p, nlopt_opt opt, unsigned long long seed)
{
    p->quad.seed = seed;
    return nlopt_b200::set_min_objective_sync(opt, &p->quad);
}

int nb200p_set_simp_device_sync(nb200p_problem_s *p, nlopt_opt opt, unsigned long long seed, double eps)
{
    p->simp.seed = seed;
    p->simp.eps = eps;
    return nlopt_b200::set_min_objective_sync(opt, &p->simp);
}

int nb200p_add_mean_device_sync(nb200p_problem_s *p, nlopt_opt opt, double offset, double tol)
{
    MeanDev *m = new MeanDev{1.0 / (double) nlopt_get_dimension(opt), offset};
    p->mean.push_back(m);
    return nlopt_b200::add_inequality_constraint_sync(opt, m, tol);
}

int nb200p_set_quadratic_device(nb200p_problem_s *p, nlopt_opt opt, unsigned long long seed)
{
    p->quad.seed = seed;
    return nlopt_b200::set_min_objective(opt, &p->quad);
}

int nb200p_add_mean_device(nb200p_problem_s *p, nlopt_opt opt, double offset, double tol)
{
    MeanDev *m = new MeanDev{1.0 / (double) nlopt_get_dimension(opt), offset};
    p->mean.push_back(m);
    return nlopt_b200::add_inequality_constraint(opt, m, tol);
}

int nb200p_set_simp_device(nb200p_problem_s *p, nlopt_opt opt, unsigned long long seed, double eps)
{
    p->simp.seed = seed;
    p->simp.eps = eps;
    return nlopt_b200::set_min_objective(opt, &p->simp);
}

// ---- maximisation: Negated<F> through nlopt_b200::set_max_objective (sync != 0: set_max_objective_sync) ----------------
int nb200p_set_quadratic_device_max(nb200p_problem_s *p, nlopt_opt opt, unsigned long long seed, int sync)
{
    p->nquad.f.seed = seed;
    return set_objective(opt, &p->nquad, sync, 1);
}

int nb200p_set_simp_device_max(nb200p_problem_s *p, nlopt_opt opt, unsigned long long seed, double eps, int sync)
{
    p->nsimp.f.seed = seed;
    p->nsimp.f.eps = eps;
    return set_objective(opt, &p->nsimp, sync, 1);
}

// the chained Rosenbrock function (halo 1), minimised or, as Negated<RosenbrockDev>, maximised, in either form
int nb200p_set_rosenbrock_device_form(nb200p_problem_s *p, nlopt_opt opt, int sync, int maximize)
{
    return maximize ? set_objective(opt, &p->nrosen, sync, 1) : set_objective(opt, &p->rosen, sync, 0);
}

// The raw pointers the C++ front end registers for QuadraticDev (negated != 0: Negated<QuadraticDev>), for registration
// from another language: sync == 0: nlopt_b200_dfunc2 / nlopt_b200_dfinish and the functor; sync != 0: nlopt_b200_dfunc
// and its data record (*fin = NULL)
int nb200p_quadratic_pointers(nb200p_problem_s *p, nlopt_opt opt, unsigned long long seed, int negated, int sync, void **fn,
                              void **fin, void **data)
{
    namespace d = nlopt_b200::detail;
    p->quad.seed = seed;
    p->nquad.f.seed = seed;
    const unsigned long long n = nlopt_get_dimension(opt);
    if (sync) {
        *fin = nullptr;
        if (negated) {
            *fn = (void *) &d::trampoline<Negated<QuadraticDev>>;
            *data = new d::Bound<Negated<QuadraticDev>>{&p->nquad, n};     // lives as long as the process, as in the front end
        } else {
            *fn = (void *) &d::trampoline<QuadraticDev>;
            *data = new d::Bound<QuadraticDev>{&p->quad, n};
        }
    } else if (negated) {
        *fn = (void *) &d::trampoline2<Negated<QuadraticDev>>;
        *fin = (void *) &d::finish2<Negated<QuadraticDev>>;
        *data = &p->nquad;
    } else {
        *fn = (void *) &d::trampoline2<QuadraticDev>;
        *fin = (void *) &d::finish2<QuadraticDev>;
        *data = &p->quad;
    }
    return NLOPT_SUCCESS;
}

// ---- host callbacks (nlopt_func shape; work with any NLopt-ABI library) ----------------------------------
double nb200p_simp_host(unsigned n, const double *x, double *grad, void *data)
{
    Tick t;
    const nb200p_simp_data *sd = static_cast<const nb200p_simp_data *>(data);
    const double ome = 1.0 - sd->eps;
    double f = 0.0;
    for (unsigned j = 0; j < n; ++j) {
        const double a = 0.5 + nb200::u01(sd->seed, 0, j);
        const double x2 = x[j] * x[j], x3 = x2 * x[j];
        const double d = sd->eps + ome * x3;
        if (grad) grad[j] = -(((a * (ome * 3.0)) * x2) / (d * d));
        f += a / d;
    }
    return f;
}

// sharded forms (nlopt_b200_sfunc): this rank's variables only, additive value contribution
double nb200p_simp_sharded(unsigned n_local, unsigned long long j0, unsigned long long, const double *x, double *grad, void *data)
{
    Tick t;
    const nb200p_simp_data *sd = static_cast<const nb200p_simp_data *>(data);
    const double ome = 1.0 - sd->eps;
    double f = 0.0;
    for (unsigned jl = 0; jl < n_local; ++jl) {
        const double a = 0.5 + nb200::u01(sd->seed, 0, j0 + jl);
        const double x2 = x[jl] * x[jl], x3 = x2 * x[jl];
        const double d = sd->eps + ome * x3;
        if (grad) grad[jl] = -(((a * (ome * 3.0)) * x2) / (d * d));
        f += a / d;
    }
    return f;
}

// -nb200p_simp_sharded, value and gradient (nlopt_b200_set_max_objective_sharded)
double nb200p_simp_sharded_neg(unsigned n_local, unsigned long long j0, unsigned long long n, const double *x, double *grad,
                               void *data)
{
    const double f = nb200p_simp_sharded(n_local, j0, n, x, grad, data);
    if (grad)
        for (unsigned jl = 0; jl < n_local; ++jl) grad[jl] = -grad[jl];
    return -f;
}

double nb200p_mean_sharded(unsigned n_local, unsigned long long j0, unsigned long long n, const double *x, double *grad, void *data)
{
    Tick t;
    const double inv_n = 1.0 / (double) n;
    double s = 0.0;
    for (unsigned jl = 0; jl < n_local; ++jl) s += x[jl];
    if (grad)
        for (unsigned jl = 0; jl < n_local; ++jl) grad[jl] = inv_n;
    return s * inv_n + (j0 == 0 ? static_cast<const nb200p_mean_data *>(data)->offset : 0.0);
}

void *nb200p_make_simp_data(nb200p_problem_s *p, unsigned long long seed, double eps)
{
    nb200p_simp_data *d = static_cast<nb200p_simp_data *>(std::malloc(sizeof(nb200p_simp_data)));
    d->seed = seed;
    d->eps = eps;
    p->misc_host.push_back(d);
    return d;
}

void *nb200p_make_mean_data(nb200p_problem_s *p, double offset)
{
    nb200p_mean_data *d = static_cast<nb200p_mean_data *>(std::malloc(sizeof(nb200p_mean_data)));
    d->offset = offset;
    p->misc_host.push_back(d);
    return d;
}

void *nb200p_make_quad_data(nb200p_problem_s *p, unsigned long long seed)
{
    nb200p_quad_data *d = static_cast<nb200p_quad_data *>(std::malloc(sizeof(nb200p_quad_data)));
    d->seed = seed;
    p->misc_host.push_back(d);
    return d;
}

double nb200p_rosenbrock_host(unsigned n, const double *x, double *grad, void *)
{
    Tick t;
    double f = 0.0;
    if (grad)
        for (unsigned j = 0; j < n; ++j) grad[j] = 0.0;
    for (unsigned j = 0; j + 1 < n; ++j) {
        const double d = x[j + 1] - x[j] * x[j], e = 1.0 - x[j];
        f += 100.0 * d * d + e * e;
        if (grad) {
            grad[j] += -400.0 * x[j] * d - 2.0 * e;
            grad[j + 1] += 200.0 * d;
        }
    }
    return f;
}

double nb200p_linear_host(unsigned n, const double *x, double *grad, void *data)
{
    Tick t;
    const nb200p_lin_data *d = static_cast<const nb200p_lin_data *>(data);
    double s = 0.0;
    for (unsigned j = 0; j < n; ++j) s += d->w[j] * x[j];
    if (grad) std::memcpy(grad, d->w, (size_t) n * sizeof(double));
    return s - d->b;
}

double nb200p_quadratic_host(unsigned n, const double *x, double *grad, void *data)
{
    Tick t;
    const unsigned long long seed = static_cast<const nb200p_quad_data *>(data)->seed;
    double s = 0.0;
    for (unsigned j = 0; j < n; ++j) {
        const double a = 1.0 + nb200::u01(seed, 0, j), b = 2.0 * nb200::u01(seed, 1, j) - 1.0;
        const double d = x[j] - b, ad = a * d;
        if (grad) grad[j] = ad;
        s += ad * d;
    }
    return 0.5 * s;
}

double nb200p_mean_host(unsigned n, const double *x, double *grad, void *data)
{
    Tick t;
    const double inv_n = 1.0 / (double) n;
    double s = 0.0;
    for (unsigned j = 0; j < n; ++j) s += x[j];
    if (grad)
        for (unsigned j = 0; j < n; ++j) grad[j] = inv_n;
    return s * inv_n + static_cast<const nb200p_mean_data *>(data)->offset;
}

// data-record helpers for the host callbacks (w_host must stay alive)
void *nb200p_make_linear_data(nb200p_problem_s *p, const double *w_host, double b)
{
    nb200p_lin_data *d = new nb200p_lin_data{w_host, b};
    p->lin_host.push_back(d);
    return d;
}

// an nlopt_b200_dprecond; data: an nb200p_tridiag_data in host memory
void nb200p_tridiag_precond(const nlopt_b200_shard *shard, const double *x, const double *v, double *vpre, void *data,
                            void *stream)
{
    (void) x;
    const nb200p_tridiag_data &t = *static_cast<const nb200p_tridiag_data *>(data);
    const unsigned long long n = shard->n_local;
    const unsigned long long g = (n + 255) / 256;
    nb200p_tridiag_kernel<<<(int) (g < 1 ? 1 : g > 4096 ? 4096 : g), 256, 0, static_cast<cudaStream_t>(stream)>>>(t.d, v, t.sign, n, vpre);
}

}  // extern "C"
