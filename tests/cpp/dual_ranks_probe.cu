// dual_ranks_probe.cu -- launches the library's dual evaluation kernels (nlopt_b200/csrc/ccsa_kernels.cuh) as one rank
// of 1, 2, 4 or 8 on host arrays the caller supplies, and publish_kernel on the gathered virtual-shard sums, the way
// DeviceBackend::launch_dual does after its ncclAllGather.  Tests only (tests/test_dual_sums_gpu.py).
//
// Only the one-launch evaluation kernels run here: their sweeper CTAs wait for nothing and the folder CTA waits for
// its own rank's group records only.  The mailbox exchange and the persistent solve kernel wait for their peers and are
// not launched.  Every entry point returns 0, or -1 with the failed call in drp_error().
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "ccsa_kernels.cuh"

namespace {

char g_err[256] = "";

bool failed(cudaError_t e, const char *what)
{
    if (e == cudaSuccess) return false;
    std::snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    return true;
}
#define DRP(call) do { if (failed((call), #call)) return -1; } while (0)

struct Dev {
    void *p = nullptr;
    ~Dev() { if (p) cudaFree(p); }
    cudaError_t up(const void *host, size_t nbytes)
    {
        cudaError_t e = cudaMalloc(&p, nbytes);
        return e != cudaSuccess ? e : cudaMemcpy(p, host, nbytes, cudaMemcpyHostToDevice);
    }
    cudaError_t zeros(size_t nbytes)
    {
        cudaError_t e = cudaMalloc(&p, nbytes);
        return e != cudaSuccess ? e : cudaMemset(p, 0, nbytes);
    }
    double *d() const { return static_cast<double *>(p); }
};

typedef void (*DualKernel)(const nb200::DualArgs);

// the kernels of the library's default paths: the register form in its default geometry for 4 rows (device_backend.cu
// kCfgs / default_cfg: MMA {256, 1, 3}, CCSAQ {256, 1, 4}), the TMA-staged form with 4 rows and 2 stages at 3 CTAs/SM
// (kernel_cfg 11), and the wide kernel
enum { kRegister = 0, kTma = 1, kWide = 2 };
constexpr int kTmaStages = 2;

DualKernel pick(int kind, int variant)
{
    using namespace nb200;
    if (kind == kRegister)
        return variant == 0 ? (DualKernel) dual_eval_kernel<0, 4, true, true, 256, 1, 3, false>
                            : (DualKernel) dual_eval_kernel<1, 4, true, true, 256, 1, 4, false>;
    if (kind == kTma)
        return variant == 0 ? (DualKernel) dual_eval_tma_kernel<0, 4, true, kTmaStages, 3>
                            : (DualKernel) dual_eval_tma_kernel<1, 4, true, kTmaStages, 3>;
    return variant == 0 ? (DualKernel) dual_eval_wide_kernel<0, true> : (DualKernel) dual_eval_wide_kernel<1, true>;
}

size_t dyn_smem(int kind, int m)
{
    if (kind == kTma) return (size_t) kTmaStages * (5 + 4) * nb200::kChunkBytes;
    if (kind == kWide) return 12 * (size_t) ((m + nb200::kWideRows - 1) / nb200::kWideRows * nb200::kWideRows) * sizeof(double);
    return 0;
}

}  // namespace

extern "C" {

const char *drp_error() { return g_err; }

// dynamic shared memory, resident CTAs per SM and SMs of one kernel as the library sizes it
int drp_occupancy(int kind, int variant, int m, long long *smem, int *per_sm, int *sms)
{
    DualKernel fn = pick(kind, variant);
    const size_t s = dyn_smem(kind, m);
    if (s) DRP(cudaFuncSetAttribute((const void *) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) s));
    DRP(cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, fn, kind == kTma ? nb200::kTmaBlock : nb200::kBlock, s));
    int dev = 0;
    DRP(cudaGetDevice(&dev));
    DRP(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
    *smem = (long long) s;
    return 0;
}

// One rank's launch.  geo = {n_local, nchunks, chunk0, groups_total, group0, groups_per_vshard, local_vshards,
// groups_local} of nlopt_b200_shard_geometry(n, rank, world).  The arrays hold the rank's ld entries (ld a multiple of
// 512, sigma = 0 beyond n_local), grad_c m rows of ld.  y, rhoc: m entries; active: m flags (MMA: 0 where the
// constraint value is NaN).
// publish = 1: the single-rank path, the 3 + m totals land in out (nvp entries); publish = 0: the NCCL path, the
// rank's virtual-shard sums land in its rows of out_dev[8][nvp] (host, in and out).  xcur: ld entries of x*(y).
int drp_eval(int kind, int variant, int m, const unsigned long long *geo, unsigned long long ld, const double *x,
             const double *lb, const double *ub, const double *sigma, const double *g, const double *grad_c,
             const double *y, const double *rhoc, const int *active, double rho, int rank, int world, int publish,
             int nvp, double *out_dev, double *out, double *xcur)
{
    using namespace nb200;
    if ((kind != kWide && m != 4) || (kind == kWide && (m <= kMaxParamM || m > kWideMaxM)) || nvp < 3 + m || ld % 512) {
        std::snprintf(g_err, sizeof g_err, "drp_eval: the register and TMA forms take m = 4, the wide one 16 < m <= %d", kWideMaxM);
        return -1;
    }
    for (int i = 0; i < m; ++i)
        if (kind != kWide && !active[i]) {      // FULL instantiations: every row on
            std::snprintf(g_err, sizeof g_err, "drp_eval: the register and TMA forms here run with every row on");
            return -1;
        }
    const unsigned groups_local = (unsigned) geo[7];
    Dev dx, dlb, dub, ds, dg, dG, dxc, tags, od, oh, flag, wide;
    DRP(dx.up(x, ld * sizeof(double)));
    DRP(dlb.up(lb, ld * sizeof(double)));
    DRP(dub.up(ub, ld * sizeof(double)));
    DRP(ds.up(sigma, ld * sizeof(double)));
    DRP(dg.up(g, ld * sizeof(double)));
    DRP(dG.up(grad_c, (size_t) m * ld * sizeof(double)));
    DRP(dxc.zeros(ld * sizeof(double)));
    DRP(tags.zeros((size_t) groups_local * nvp * 2 * sizeof(double)));
    DRP(od.up(out_dev, (size_t) kVirtualShards * nvp * sizeof(double)));
    DRP(oh.zeros((size_t) nvp * sizeof(double)));
    DRP(flag.zeros(sizeof(unsigned long long)));

    DualArgs a;
    std::memset(&a, 0, sizeof a);
    a.x = dx.d(); a.lb = dlb.d(); a.ub = dub.d(); a.sigma = ds.d(); a.g = dg.d(); a.G = dG.d(); a.xcur = dxc.d();
    a.ld = ld;
    a.nchunks = geo[1]; a.chunk0 = geo[2];
    a.nseg_total = (unsigned) geo[3]; a.seg0 = (unsigned) geo[4]; a.segs_per_vshard = (unsigned) geo[5];
    a.local_vshards = (unsigned) geo[6];
    a.grouptags = tags.d();
    a.tag = (1ull << 63) | 1ull;
    a.out_dev = od.d(); a.out_host = oh.d(); a.flag_host = static_cast<unsigned long long *>(flag.p);
    a.seq = 1; a.publish_host = publish; a.nvp = nvp;
    a.rank = rank; a.world = world;             // box[] stays null: the NCCL path
    a.m = m;
    a.rho = rho; a.half_rho = 0.5 * rho;
    double u = rho;                             // DeviceBackend::fill_dual_args: every row, in index order
    std::vector<double> wh;
    if (kind == kWide) wh.resize(4 * (size_t) m);
    for (int i = 0; i < m; ++i) {
        if (kind == kWide) {
            wh[i] = y[i]; wh[m + i] = rhoc[i]; wh[2 * (size_t) m + i] = 0.5 * rhoc[i]; wh[3 * (size_t) m + i] = active[i] ? 1.0 : 0.0;
        } else {
            a.y[i] = y[i]; a.rhoc[i] = rhoc[i]; a.half_rhoc[i] = 0.5 * rhoc[i];
            if (active[i]) a.active |= 1u << i;
        }
        u += rhoc[i] * y[i];
    }
    a.u_ccsaq = u;
    if (kind == kWide) {
        DRP(wide.up(wh.data(), wh.size() * sizeof(double)));
        a.wide = wide.d();
    }

    long long smem = 0;
    int per_sm = 0, sms = 0;
    if (drp_occupancy(kind, variant, m, &smem, &per_sm, &sms)) return -1;
    if (per_sm < 1) {
        std::snprintf(g_err, sizeof g_err, "drp_eval: the kernel does not fit on an SM");
        return -1;
    }
    long long grid = (long long) sms * per_sm;
    if (grid > (long long) groups_local) grid = groups_local;
    if (grid < 1) grid = 1;
    pick(kind, variant)<<<(unsigned) grid + 1, kind == kTma ? kTmaBlock : kBlock, (size_t) smem>>>(a);
    DRP(cudaGetLastError());
    DRP(cudaDeviceSynchronize());
    DRP(cudaMemcpy(xcur, dxc.p, ld * sizeof(double), cudaMemcpyDeviceToHost));
    DRP(cudaMemcpy(out_dev, od.p, (size_t) kVirtualShards * nvp * sizeof(double), cudaMemcpyDeviceToHost));
    DRP(cudaMemcpy(out, oh.p, (size_t) nvp * sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
}

// publish_kernel on the assembled out_dev[8][nvp], launched as the library launches it after its all-gather
int drp_publish(const double *out_dev, int nv, int nvp, double *out)
{
    Dev od, oh, flag;
    DRP(od.up(out_dev, (size_t) nb200::kVirtualShards * nvp * sizeof(double)));
    DRP(oh.zeros((size_t) nvp * sizeof(double)));
    DRP(flag.zeros(sizeof(unsigned long long)));
    nb200::publish_kernel<<<1, 256>>>(od.d(), nv, nvp, oh.d(), static_cast<unsigned long long *>(flag.p), 1ull);
    DRP(cudaGetLastError());
    DRP(cudaDeviceSynchronize());
    DRP(cudaMemcpy(out, oh.p, (size_t) nvp * sizeof(double), cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"
