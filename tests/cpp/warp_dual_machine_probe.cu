// warp_dual_machine_probe.cu -- replays a recorded dual-optimiser trajectory into the device machine of
// nlopt_b200/csrc/ccsa_kernels.cuh (WarpDualMachine<MAXM>), on one warp, with the calls solve_folder makes: start, then
// per evaluation trial(), feed_pre(F, dF/dy_lane, time_up, lane) and step(lane) unless finished.  Tests only
// (tests/test_dual_machine_gpu.py builds it with the library's nvcc flags).
#include <cuda_runtime.h>

#include <cstdio>

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
#define WDM(call) do { if (failed((call), #call)) { rc = -1; goto out; } } while (0)

// counts[]: ret, nevals, feeds, status (0 finished on the recorded answers, 1 trial point k != ys[k], 2 wanted more than
// K evaluations), k of the mismatch.  yf[]: y (lanes < m), then fmin.
template <int MAXM>
__global__ void replay_kernel(int m, const double *y0, const double *lo, const double *hi, DualStop st, long k_time,
                              long K, const double *ys, const double *fs, const double *gs, double *yf, long long *counts)
{
    const int lane = threadIdx.x & 31;
    WarpDualMachine<MAXM> mach;
    const double y0l = lane < m ? y0[lane] : 0.0, lol = lane < m ? lo[lane] : 0.0, hil = lane < m ? hi[lane] : 0.0;
    const int rc = mach.start(m, y0l, lol, hil, st, lane);
    long feeds = 0, where = -1;
    int status = 0;
    if (rc == kRetSuccess) {
        for (long k = 0;; ++k) {
            if (k == K) { status = 2; where = k; break; }
            const double t = mach.trial();
            const bool differs = lane < m && __double_as_longlong(t) != __double_as_longlong(ys[k * m + lane]);
            if (__any_sync(0xffffffffu, differs)) { status = 1; where = k; break; }
            ++feeds;
            const double grad = lane < m ? gs[k * m + lane] : 0.0;
            if (mach.feed_pre(fs[k], grad, k_time >= 0 && k >= k_time, lane)) break;
            mach.step(lane);
        }
    }
    if (lane < m) yf[lane] = mach.y;
    if (lane == 0) {
        yf[32] = mach.fmin;
        counts[0] = mach.ret; counts[1] = mach.nevals; counts[2] = feeds; counts[3] = status; counts[4] = where;
    }
}

template <int MAXM>
void launch(int m, const double *y0, const double *lo, const double *hi, const DualStop &st, long k_time, long K,
            const double *ys, const double *fs, const double *gs, double *yf, long long *counts)
{
    replay_kernel<MAXM><<<1, 32>>>(m, y0, lo, hi, st, k_time, K, ys, fs, gs, yf, counts);
}

}  // namespace

extern "C" {

const char *wdm_error() { return g_err; }

// One replay on the device in WarpDualMachine<maxm> (1, 2, 4, 8 or 16; m <= maxm).  Host arrays as in
// tests/cpp/dual_machine_probe.cpp; yf_out[33] = y (first m), fmin; counts_out[5] = ret, nevals, feeds, status, where.
// Returns 0, or -1 with the failed call in wdm_error().
int wdm_replay(int maxm, int m, const double *y0, const double *lo, const double *hi, const double *stop5, long k_time,
               long K, const double *ys, const double *fs, const double *gs, double *yf_out, long long *counts_out)
{
    int rc = 0;
    double *d = nullptr;
    long long *dc = nullptr;
    const size_t km = (size_t) K * (size_t) m;
    const size_t total = 3 * (size_t) m + 2 * km + (size_t) K + 33;
    DualStop st{stop5[0], stop5[1], stop5[2], stop5[3], (int) stop5[4], k_time >= 0 ? 1.0 : 0.0};
    if (m < 1 || m > maxm || !(maxm == 1 || maxm == 2 || maxm == 4 || maxm == 8 || maxm == 16)) {
        std::snprintf(g_err, sizeof g_err, "m = %d does not fit MAXM = %d", m, maxm);
        return -1;
    }
    {
        WDM(cudaMalloc(&d, total * sizeof(double)));
        WDM(cudaMalloc(&dc, 5 * sizeof(long long)));
        double *dy0 = d, *dlo = d + m, *dhi = d + 2 * m, *dys = d + 3 * m, *dgs = dys + km, *dfs = dgs + km, *dyf = dfs + K;
        WDM(cudaMemcpy(dy0, y0, m * sizeof(double), cudaMemcpyHostToDevice));
        WDM(cudaMemcpy(dlo, lo, m * sizeof(double), cudaMemcpyHostToDevice));
        WDM(cudaMemcpy(dhi, hi, m * sizeof(double), cudaMemcpyHostToDevice));
        if (K) {
            WDM(cudaMemcpy(dys, ys, km * sizeof(double), cudaMemcpyHostToDevice));
            WDM(cudaMemcpy(dgs, gs, km * sizeof(double), cudaMemcpyHostToDevice));
            WDM(cudaMemcpy(dfs, fs, K * sizeof(double), cudaMemcpyHostToDevice));
        }
        WDM(cudaMemset(dyf, 0, 33 * sizeof(double)));
        switch (maxm) {
            case 1: launch<1>(m, dy0, dlo, dhi, st, k_time, K, dys, dfs, dgs, dyf, dc); break;
            case 2: launch<2>(m, dy0, dlo, dhi, st, k_time, K, dys, dfs, dgs, dyf, dc); break;
            case 4: launch<4>(m, dy0, dlo, dhi, st, k_time, K, dys, dfs, dgs, dyf, dc); break;
            case 8: launch<8>(m, dy0, dlo, dhi, st, k_time, K, dys, dfs, dgs, dyf, dc); break;
            default: launch<16>(m, dy0, dlo, dhi, st, k_time, K, dys, dfs, dgs, dyf, dc); break;
        }
        WDM(cudaGetLastError());
        WDM(cudaDeviceSynchronize());
        WDM(cudaMemcpy(yf_out, dyf, 33 * sizeof(double), cudaMemcpyDeviceToHost));
        WDM(cudaMemcpy(counts_out, dc, 5 * sizeof(long long), cudaMemcpyDeviceToHost));
    }
out:
    if (d) cudaFree(d);
    if (dc) cudaFree(dc);
    return rc;
}

}  // extern "C"
