// precond.hpp -- launches of the preconditioned-CCSAQ kernels of precond.cu (DeviceBackend::model_solve): one thread per
// variable in a grid-stride loop of `grid` CTAs on stream s; each returns the launch's error.
#pragma once

#include <cuda_runtime.h>

namespace nb200 {

// pre_lb = max(lb, x - sigma), pre_ub = min(ub, x + sigma), xcur = x; lb / ub null: the scalars lb0 / ub0
cudaError_t launch_precond_box(const double *lb, const double *ub, double lb0, double ub0, const double *x, const double *sigma,
                               unsigned long long n, double *pre_lb, double *pre_ub, double *xcur, int grid, cudaStream_t s);
// dx = x - x0
cudaError_t launch_precond_dx(const double *x, const double *x0, unsigned long long n, double *dx, int grid, cudaStream_t s);
// one model row: separable terms, gradient (grad null: none) and, with hdx, the quadratic terms
cudaError_t launch_precond_model(const double *dx, const double *sigma, const double *dfdx, const double *hdx, double rho,
                                 unsigned long long n, double *sterm, double *qterm, double *grad, int grid, cudaStream_t s);
// the terms of w = sum 1/2 ((xcur - x) / sigma)^2
cudaError_t launch_precond_w(const double *xcur, const double *x, const double *sigma, unsigned long long n, double *wterm, int grid,
                             cudaStream_t s);

}  // namespace nb200
