// precond.cu -- the element-wise kernels of preconditioned CCSAQ on the device (ccsa_quadratic.c:153-206,
// :441-467; DeviceBackend::model_solve).  Each restates a loop of the host path (nlopt_api.cpp: run_ccsa_precond,
// precond_gfunc) with the same IEEE operations in the same order, written out with __dadd_rn / __dmul_rn so that no
// FMA contraction changes a bit.  Their sums go through the terms reduction (terms_kernels.cuh).  They live in a
// translation unit of their own, so that adding them leaves the code of every kernel of device_backend.cu unchanged;
// precond.hpp declares their launches.
#include "precond.hpp"

namespace nb200 {

namespace {

constexpr int kPrecondBlock = 256;

// the trust box of one model solve (:441-446): pre_lb = max(lb, x - sigma), pre_ub = min(ub, x + sigma), in the host's
// operand order (a NaN comparison takes the second operand), and xcur = x.  lb / ub null: the scalar bounds lb0 / ub0.
__global__ void __launch_bounds__(kPrecondBlock) precond_box_kernel(const double *__restrict__ lb, const double *__restrict__ ub,
                                                                    double lb0, double ub0, const double *__restrict__ x,
                                                                    const double *__restrict__ sigma, unsigned long long n,
                                                                    double *__restrict__ pre_lb, double *__restrict__ pre_ub,
                                                                    double *__restrict__ xcur)
{
    for (unsigned long long j = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; j < n;
         j += (unsigned long long) gridDim.x * blockDim.x) {
        const double xj = x[j], s = sigma[j], l = lb ? lb[j] : lb0, u = ub ? ub[j] : ub0;
        const double lo = __dsub_rn(xj, s), hi = __dadd_rn(xj, s);
        pre_lb[j] = l > lo ? l : lo;
        pre_ub[j] = u < hi ? u : hi;
        xcur[j] = xj;
    }
}

// dx = x - x0 (precond_gfunc), the vector every preconditioner of a point is applied to
__global__ void __launch_bounds__(kPrecondBlock) precond_dx_kernel(const double *__restrict__ x, const double *__restrict__ x0,
                                                                   unsigned long long n, double *__restrict__ dx)
{
    for (unsigned long long j = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; j < n;
         j += (unsigned long long) gridDim.x * blockDim.x)
        dx[j] = __dsub_rn(x[j], x0[j]);
}

// One row of the model (ccsa_quadratic.c:153-181): the separable term and the gradient of every variable,
//     sterm = dfdx dx + ((0.5 rho) (dx dx)) sigma2inv,   grad = (dfdx + (rho dx) sigma2inv) [+ Hdx],
// with sigma2inv = 1 / (sigma sigma), and, for a preconditioned row (hdx != null), the quadratic term
//     qterm = (0.5 dx) Hdx.
// grad null: values only.
__global__ void __launch_bounds__(kPrecondBlock) precond_model_kernel(const double *__restrict__ dx, const double *__restrict__ sigma,
                                                                      const double *__restrict__ dfdx, const double *__restrict__ hdx,
                                                                      double rho, unsigned long long n, double *__restrict__ sterm,
                                                                      double *__restrict__ qterm, double *__restrict__ grad)
{
    const double half_rho = __dmul_rn(0.5, rho);
    for (unsigned long long j = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; j < n;
         j += (unsigned long long) gridDim.x * blockDim.x) {
        const double d = dx[j], s = sigma[j], g = dfdx[j];
        const double sigma2inv = __ddiv_rn(1.0, __dmul_rn(s, s));
        sterm[j] = __dadd_rn(__dmul_rn(g, d), __dmul_rn(__dmul_rn(half_rho, __dmul_rn(d, d)), sigma2inv));
        double gr = __dadd_rn(g, __dmul_rn(__dmul_rn(rho, d), sigma2inv));
        if (hdx) {
            const double h = hdx[j];
            qterm[j] = __dmul_rn(__dmul_rn(0.5, d), h);
            gr = __dadd_rn(gr, h);
        }
        if (grad) grad[j] = gr;
    }
}

// the terms of w = sum 1/2 ((xcur - x) / sigma)^2 (run_ccsa_precond: the separable branch's w, :465-467)
__global__ void __launch_bounds__(kPrecondBlock) precond_w_kernel(const double *__restrict__ xcur, const double *__restrict__ x,
                                                                  const double *__restrict__ sigma, unsigned long long n,
                                                                  double *__restrict__ wterm)
{
    for (unsigned long long j = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; j < n;
         j += (unsigned long long) gridDim.x * blockDim.x) {
        const double q = __ddiv_rn(__dsub_rn(xcur[j], x[j]), sigma[j]);
        wterm[j] = __dmul_rn(__dmul_rn(0.5, q), q);
    }
}

}  // namespace

cudaError_t launch_precond_box(const double *lb, const double *ub, double lb0, double ub0, const double *x, const double *sigma,
                               unsigned long long n, double *pre_lb, double *pre_ub, double *xcur, int grid, cudaStream_t s)
{
    precond_box_kernel<<<grid, kPrecondBlock, 0, s>>>(lb, ub, lb0, ub0, x, sigma, n, pre_lb, pre_ub, xcur);
    return cudaGetLastError();
}

cudaError_t launch_precond_dx(const double *x, const double *x0, unsigned long long n, double *dx, int grid, cudaStream_t s)
{
    precond_dx_kernel<<<grid, kPrecondBlock, 0, s>>>(x, x0, n, dx);
    return cudaGetLastError();
}

cudaError_t launch_precond_model(const double *dx, const double *sigma, const double *dfdx, const double *hdx, double rho,
                                 unsigned long long n, double *sterm, double *qterm, double *grad, int grid, cudaStream_t s)
{
    precond_model_kernel<<<grid, kPrecondBlock, 0, s>>>(dx, sigma, dfdx, hdx, rho, n, sterm, qterm, grad);
    return cudaGetLastError();
}

cudaError_t launch_precond_w(const double *xcur, const double *x, const double *sigma, unsigned long long n, double *wterm, int grid,
                             cudaStream_t s)
{
    precond_w_kernel<<<grid, kPrecondBlock, 0, s>>>(xcur, x, sigma, n, wterm);
    return cudaGetLastError();
}

}  // namespace nb200
