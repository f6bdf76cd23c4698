// closed_forms_probe.cu -- runs the per-variable closed forms of the dual evaluation (nlopt_b200/csrc/ccsa_kernels.cuh)
// and the written-out IEEE fast paths they use (nlopt_b200/csrc/pair_math.cuh) on host arrays the caller supplies, one
// thread per operand or per pair of variables.  Tests only (tests/test_closed_forms_gpu.py).
//
// cfp_primitives: div_fast, div_by with one prepared divisor for two numerators, rcp_fast and sqrt_fast, each with its
// own range flag, and the builtins __ddiv_rn(a, b), __ddiv_rn(1, b), __dsqrt_rn(a) on the same operands.
// cfp_forms: mma_pair / ccsaq_pair (form 0) or mma_point / ccsaq_point (form 1) on arrays of pairs of variables, for the
// (variant, MAXM, FULL) instantiations the library uses.  Each pair's accumulators start at +0.
// Every entry point returns 0, or -1 with the failed call in cfp_error().
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>

#include "ccsa_kernels.cuh"

namespace {

using namespace nb200;

char g_err[256] = "";

bool failed(cudaError_t e, const char *what)
{
    if (e == cudaSuccess) return false;
    std::snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    return true;
}
#define CFP(call) do { if (failed((call), #call)) return -1; } while (0)

// device copy of a host array: freed when it goes out of scope
struct Dev {
    void *p = nullptr;
    size_t bytes = 0;
    ~Dev() { if (p) cudaFree(p); }
    cudaError_t up(const void *host, size_t nbytes)
    {
        bytes = nbytes;
        cudaError_t e = cudaMalloc(&p, nbytes ? nbytes : 16);
        return e != cudaSuccess || !nbytes ? e : cudaMemcpy(p, host, nbytes, cudaMemcpyHostToDevice);
    }
    cudaError_t alloc(size_t nbytes)
    {
        bytes = nbytes;
        cudaError_t e = cudaMalloc(&p, nbytes ? nbytes : 16);
        return e != cudaSuccess ? e : cudaMemset(p, 0xff, nbytes);
    }
    cudaError_t down(void *host) const { return bytes ? cudaMemcpy(host, p, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; }
    template <class T> T *as() const { return static_cast<T *>(p); }
};

int finish_launch()
{
    CFP(cudaGetLastError());
    CFP(cudaDeviceSynchronize());
    return 0;
}

// out[k * n + i]: k = 0 div_fast(a, b), 1 div_by(a, d), 2 div_by(a2, d) with d = prep_div(b) shared, 3 rcp_fast(b),
// 4 sqrt_fast(a), 5 __ddiv_rn(a, b), 6 __ddiv_rn(a2, b), 7 __ddiv_rn(1, b), 8 __dsqrt_rn(a); bad[k * n + i], k < 5: the
// range flag of value k
__global__ void primitives_kernel(const double *a, const double *a2, const double *b, size_t n, double *out, unsigned *bad)
{
    const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double ai = a[i], a2i = a2[i], bi = b[i];
    unsigned f[5] = {0u, 0u, 0u, 0u, 0u};
    out[0 * n + i] = div_fast(ai, bi, f[0]);
    const DivBy d = prep_div(bi);
    out[1 * n + i] = div_by(ai, d, f[1]);
    out[2 * n + i] = div_by(a2i, d, f[2]);
    out[3 * n + i] = rcp_fast(bi, f[3]);
    out[4 * n + i] = sqrt_fast(ai, f[4]);
    out[5 * n + i] = __ddiv_rn(ai, bi);
    out[6 * n + i] = __ddiv_rn(a2i, bi);
    out[7 * n + i] = __ddiv_rn(1.0, bi);
    out[8 * n + i] = __dsqrt_rn(ai);
    for (int k = 0; k < 5; ++k) bad[k * n + i] = f[k];
}

// One thread per pair p.  Variable arrays are double2 (pair p = variables 2p, 2p + 1); G holds MAXM rows of 2 * npairs
// doubles.  acc_out[p * nacc + k], nacc = 3 + MAXM (at least 4), is accumulator k of pair p.
template <int VARIANT, int MAXM, bool FULL>
__global__ void forms_kernel(const __grid_constant__ DualArgs a, const double2 *x, const double2 *lb, const double2 *ub,
                             const double2 *s, const double2 *g, const double2 *G, size_t npairs, int form, double2 *xo,
                             double *acc_out)
{
    constexpr int R = MAXM > 0 ? MAXM : 1;
    constexpr int NACC = 3 + R;
    const size_t p = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npairs) return;
    double Ga[R], Gb[R], acc[NACC];
#pragma unroll
    for (int i = 0; i < R; ++i) {
        const double2 t = i < MAXM ? G[i * npairs + p] : make_double2(0.0, 0.0);
        Ga[i] = t.x;
        Gb[i] = t.y;
    }
#pragma unroll
    for (int k = 0; k < NACC; ++k) acc[k] = 0.0;
    const double2 vx = x[p], vlb = lb[p], vub = ub[p], vs = s[p], vg = g[p];
    double2 xc;
    if (form == 0) {
        if (VARIANT == 0) xc = mma_pair<MAXM, FULL>(a, vx, vlb, vub, vs, vg, Ga, Gb, acc);
        else {
            const DivBy U = prep_div(a.u_ccsaq);
            xc = ccsaq_pair<MAXM, FULL>(a, U, vx, vlb, vub, vs, vg, Ga, Gb, acc);
        }
    } else if (VARIANT == 0) {
        xc.x = mma_point<MAXM, FULL>(a, vx.x, vlb.x, vub.x, vs.x, vg.x, Ga, acc);
        xc.y = mma_point<MAXM, FULL>(a, vx.y, vlb.y, vub.y, vs.y, vg.y, Gb, acc);
    } else {
        xc.x = ccsaq_point<MAXM, FULL>(a, vx.x, vlb.x, vub.x, vs.x, vg.x, Ga, acc);
        xc.y = ccsaq_point<MAXM, FULL>(a, vx.y, vlb.y, vub.y, vs.y, vg.y, Gb, acc);
    }
    xo[p] = xc;
#pragma unroll
    for (int k = 0; k < NACC; ++k) acc_out[p * NACC + k] = acc[k];
}

typedef void (*FormsKernel)(const DualArgs, const double2 *, const double2 *, const double2 *, const double2 *,
                            const double2 *, const double2 *, size_t, int, double2 *, double *);

template <int VARIANT, bool FULL>
FormsKernel pick(int maxm)
{
    switch (maxm) {
    case 0: return forms_kernel<VARIANT, 0, FULL>;
    case 1: return forms_kernel<VARIANT, 1, FULL>;
    case 2: return forms_kernel<VARIANT, 2, FULL>;
    case 4: return forms_kernel<VARIANT, 4, FULL>;
    case 8: return forms_kernel<VARIANT, 8, FULL>;
    case 16: return forms_kernel<VARIANT, 16, FULL>;
    default: return nullptr;
    }
}

}  // namespace

extern "C" {

const char *cfp_error() { return g_err; }

// out: [9][n] doubles, bad: [5][n] unsigned (see primitives_kernel)
int cfp_primitives(const double *a, const double *a2, const double *b, size_t n, double *out, unsigned *bad)
{
    if (n == 0) return 0;
    Dev da, da2, db, dout, dbad;
    CFP(da.up(a, n * sizeof(double)));
    CFP(da2.up(a2, n * sizeof(double)));
    CFP(db.up(b, n * sizeof(double)));
    CFP(dout.alloc(9 * n * sizeof(double)));
    CFP(dbad.alloc(5 * n * sizeof(unsigned)));
    primitives_kernel<<<(unsigned) ((n + kBlock - 1) / kBlock), kBlock>>>(da.as<double>(), da2.as<double>(), db.as<double>(), n,
                                                                           dout.as<double>(), dbad.as<unsigned>());
    if (finish_launch()) return -1;
    CFP(dout.down(out));
    CFP(dbad.down(bad));
    return 0;
}

// The scalars are set as DeviceBackend::fill_dual_args sets them: half_rho = 0.5 rho, half_rhoc[i] = 0.5 rhoc[i],
// u = rho + rhoc[0] y[0] + ... (in index order); bit i of `active` switches row i on (MMA).  Variable arrays hold
// 2 * npairs entries, G holds maxm rows of 2 * npairs; xo: 2 * npairs, acc_out: npairs * (3 + max(maxm, 1)).
int cfp_forms(int variant, int maxm, int full, int form, int m, unsigned active, double rho, const double *rhoc,
              const double *y, const double *x, const double *lb, const double *ub, const double *s, const double *g,
              const double *G, size_t npairs, double *xo, double *acc_out)
{
    FormsKernel fn = variant == 0 ? (full ? pick<0, true>(maxm) : pick<0, false>(maxm))
                                  : (full ? pick<1, true>(maxm) : pick<1, false>(maxm));
    if (!fn || m < 0 || m > maxm || (form != 0 && form != 1) || npairs == 0) {
        std::snprintf(g_err, sizeof g_err, "cfp_forms: variant, maxm, m, form or npairs out of range");
        return -1;
    }
    DualArgs a;
    std::memset(&a, 0, sizeof a);
    a.m = m;
    a.active = active;
    a.rho = rho;
    a.half_rho = 0.5 * rho;
    double u = rho;
    for (int i = 0; i < m; ++i) {
        a.y[i] = y[i];
        a.rhoc[i] = rhoc[i];
        a.half_rhoc[i] = 0.5 * rhoc[i];
        u += rhoc[i] * y[i];
    }
    a.u_ccsaq = u;
    const size_t nv = 2 * npairs * sizeof(double);
    const size_t nacc = 3 + (maxm > 0 ? maxm : 1);
    Dev dx, dl, du, ds, dg, dG, dxo, dacc;
    CFP(dx.up(x, nv));
    CFP(dl.up(lb, nv));
    CFP(du.up(ub, nv));
    CFP(ds.up(s, nv));
    CFP(dg.up(g, nv));
    CFP(dG.up(G, (size_t) maxm * nv));
    CFP(dxo.alloc(nv));
    CFP(dacc.alloc(npairs * nacc * sizeof(double)));
    fn<<<(unsigned) ((npairs + kBlock - 1) / kBlock), kBlock>>>(a, dx.as<double2>(), dl.as<double2>(), du.as<double2>(),
                                                              ds.as<double2>(), dg.as<double2>(), dG.as<double2>(), npairs,
                                                              form, dxo.as<double2>(), dacc.as<double>());
    if (finish_launch()) return -1;
    CFP(dxo.down(xo));
    CFP(dacc.down(acc_out));
    return 0;
}

}  // extern "C"
