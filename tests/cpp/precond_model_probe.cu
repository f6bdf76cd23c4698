// precond_model_probe.cu -- the preconditioned-CCSAQ kernels (nlopt_b200/csrc/precond.cu) and the terms reduction
// (terms_kernels.cuh) on caller-given host arrays, for tests/test_device_precond_gpu.py.
//
// The kernel source is compiled into this probe with the library's flags (--fmad=false), so each probe_* call runs the
// library's arithmetic on the test's inputs: the test compares the outputs with a numpy model of ccsa_quadratic.c:153-181
// bit for bit, and the sums with math.fsum.  Each call copies its inputs to the device, launches, and copies back;
// returns 0, or the CUDA error code.
#include <cuda_runtime.h>

#include <vector>

#include "../../nlopt_b200/csrc/precond.cu"
#include "../../nlopt_b200/csrc/terms_kernels.cuh"

namespace {

struct Dev {
    std::vector<double *> ptrs;
    cudaError_t err = cudaSuccess;
    double *in(const double *h, unsigned long long n)          // null stays null
    {
        if (!h) return nullptr;
        double *d = out(n);
        if (d && err == cudaSuccess) err = cudaMemcpy(d, h, n * sizeof(double), cudaMemcpyHostToDevice);
        return d;
    }
    double *out(unsigned long long n)
    {
        double *d = nullptr;
        if (err == cudaSuccess) err = cudaMalloc(&d, (n ? n : 1) * sizeof(double));
        ptrs.push_back(d);
        return d;
    }
    void back(double *h, const double *d, unsigned long long n)
    {
        if (h && err == cudaSuccess) err = cudaMemcpy(h, d, n * sizeof(double), cudaMemcpyDeviceToHost);
    }
    ~Dev()
    {
        for (double *p : ptrs) cudaFree(p);
    }
};

int grid(unsigned long long n)
{
    const unsigned long long g = (n + 255) / 256;
    return (int) (g < 1 ? 1 : g > 2048 ? 2048 : g);
}

}  // namespace

extern "C" {

int probe_box(unsigned long long n, const double *lb, const double *ub, double lb0, double ub0, const double *x, const double *sigma,
              double *pre_lb, double *pre_ub, double *xcur)
{
    Dev d;
    const double *dl = d.in(lb, n), *du = d.in(ub, n), *dx = d.in(x, n), *ds = d.in(sigma, n);
    double *ol = d.out(n), *ou = d.out(n), *oc = d.out(n);
    if (d.err == cudaSuccess) d.err = nb200::launch_precond_box(dl, du, lb0, ub0, dx, ds, n, ol, ou, oc, grid(n), 0);
    d.back(pre_lb, ol, n);
    d.back(pre_ub, ou, n);
    d.back(xcur, oc, n);
    return (int) d.err;
}

int probe_dx(unsigned long long n, const double *x, const double *x0, double *dx)
{
    Dev d;
    const double *a = d.in(x, n), *b = d.in(x0, n);
    double *o = d.out(n);
    if (d.err == cudaSuccess) d.err = nb200::launch_precond_dx(a, b, n, o, grid(n), 0);
    d.back(dx, o, n);
    return (int) d.err;
}

// hdx null: a row without a preconditioner (qterm is not written); grad null: values only
int probe_model(unsigned long long n, const double *dx, const double *sigma, const double *dfdx, const double *hdx, double rho,
                double *sterm, double *qterm, double *grad)
{
    Dev d;
    const double *a = d.in(dx, n), *s = d.in(sigma, n), *g = d.in(dfdx, n), *h = d.in(hdx, n);
    double *os = d.out(n), *oq = d.out(n), *og = d.out(n);
    if (d.err == cudaSuccess)
        d.err = nb200::launch_precond_model(a, s, g, h, rho, n, os, h ? oq : nullptr, grad ? og : nullptr, grid(n), 0);
    d.back(sterm, os, n);
    if (h) d.back(qterm, oq, n);
    if (grad) d.back(grad, og, n);
    return (int) d.err;
}

int probe_w(unsigned long long n, const double *xcur, const double *x, const double *sigma, double *wterm)
{
    Dev d;
    const double *a = d.in(xcur, n), *b = d.in(x, n), *s = d.in(sigma, n);
    double *o = d.out(n);
    if (d.err == cudaSuccess) d.err = nb200::launch_precond_w(a, b, s, n, o, grid(n), 0);
    d.back(wterm, o, n);
    return (int) d.err;
}

// one row of terms through terms_group_kernel + fold_groups_mkernel on the one-rank geometry of n (the reduction the
// model's sums take), then the 8 virtual-shard sums in index order, as the library's finish adds them
int probe_sum(unsigned long long n, const double *terms, double *total)
{
    nlopt_b200_shard sh;
    nlopt_b200_shard_geometry(n, 0, 1, &sh);
    Dev d;
    const double *t = d.in(terms, n);
    double *part = d.out(sh.groups_local), *vs = d.out(8);
    if (d.err == cudaSuccess) d.err = cudaMemset(vs, 0, 8 * sizeof(double));
    if (d.err == cudaSuccess && sh.groups_local) {
        nb200::terms_group_kernel<<<dim3(sh.groups_local, 1), nb200::kTermsThreads>>>(sh, t, n, part);
        nlopt_b200::detail::fold_groups_mkernel<<<dim3(sh.local_vshards, 1), nb200::kTermsThreads>>>(
            part, sh.groups_local, sh.groups_per_vshard, vs + sh.vshard0);
        d.err = cudaGetLastError();
    }
    double h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    d.back(h, vs, 8);
    double s = h[0];
    for (int v = 1; v < 8; ++v) s += h[v];
    *total = s;
    return (int) d.err;
}

}  // extern "C"
