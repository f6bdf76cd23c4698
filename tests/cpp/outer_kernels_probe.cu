// outer_kernels_probe.cu -- launches the library's own outer-iteration kernels (nlopt_b200/csrc/ccsa_kernels.cuh) on
// host arrays the caller supplies: penalty_axpy_kernel, negate_kernel, fill_kernel, sigma_init_kernel,
// end_outer_kernel for one rank of 1, 2, 4 or 8 and publish_kernel.  Tests only (tests/test_outer_kernels_gpu.py).
//
// Arrays a kernel writes travel as a whole buffer {total, off}: the buffer is copied to the device, the kernel gets
// the pointer buf + off, and the whole buffer comes back, so the caller sees every byte around the target row.
// Every entry point returns 0, or -1 with the failed call in okp_error().
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>

#include "ccsa_kernels.cuh"

namespace {

char g_err[256] = "";

bool failed(cudaError_t e, const char *what)
{
    if (e == cudaSuccess) return false;
    std::snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    return true;
}
#define OKP(call) do { if (failed((call), #call)) return -1; } while (0)

// device copy of a host array (or of nothing, when host is null): freed when it goes out of scope
struct Dev {
    void *p = nullptr;
    size_t bytes = 0;
    ~Dev() { if (p) cudaFree(p); }
    cudaError_t up(const void *host, size_t nbytes)
    {
        if (!host || !nbytes) return cudaSuccess;
        bytes = nbytes;
        cudaError_t e = cudaMalloc(&p, nbytes);
        return e != cudaSuccess ? e : cudaMemcpy(p, host, nbytes, cudaMemcpyHostToDevice);
    }
    cudaError_t zeros(size_t nbytes)
    {
        bytes = nbytes;
        cudaError_t e = cudaMalloc(&p, nbytes);
        return e != cudaSuccess ? e : cudaMemset(p, 0, nbytes);
    }
    cudaError_t down(void *host) const { return p ? cudaMemcpy(host, p, bytes, cudaMemcpyDeviceToHost) : cudaSuccess; }
    double *at(size_t off) const { return p ? static_cast<double *>(p) + off : nullptr; }
};

int finish_launch()
{
    OKP(cudaGetLastError());
    OKP(cudaDeviceSynchronize());
    return 0;
}

}  // namespace

extern "C" {

const char *okp_error() { return g_err; }

int okp_sm_count(int *sms)
{
    int dev = 0;
    OKP(cudaGetDevice(&dev));
    OKP(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
    return 0;
}

// g[j] += sum_k coefs[k] * rows[row_idx[k] * ld + j], j < n_local; 0 <= count <= 16
int okp_penalty(double *g_buf, size_t g_total, size_t g_off, const double *rows, size_t rows_total, size_t ld,
                size_t n_local, const double *coefs, const int *row_idx, int count, int grid)
{
    if (count < 0 || count > nb200::kPenaltyRowsPerLaunch || n_local == 0 || grid < 1) {
        std::snprintf(g_err, sizeof g_err, "okp_penalty: count, n_local or grid out of range");
        return -1;
    }
    nb200::PenaltyCoefs pc;
    std::memset(&pc, 0, sizeof pc);
    for (int k = 0; k < count; ++k) { pc.c[k] = coefs[k]; pc.row[k] = row_idx[k]; }
    pc.count = count;
    Dev g, r;
    OKP(g.up(g_buf, g_total * sizeof(double)));
    OKP(r.up(rows, rows_total * sizeof(double)));
    nb200::penalty_axpy_kernel<<<grid, nb200::kBlock>>>(g.at(g_off), r.at(0), ld, n_local, pc);
    if (finish_launch()) return -1;
    OKP(g.down(g_buf));
    return 0;
}

int okp_negate(double *buf, size_t total, size_t off, size_t n_local, int grid, int times)
{
    if (n_local == 0 || grid < 1) {
        std::snprintf(g_err, sizeof g_err, "okp_negate: n_local or grid out of range");
        return -1;
    }
    Dev g;
    OKP(g.up(buf, total * sizeof(double)));
    for (int t = 0; t < times; ++t) nb200::negate_kernel<<<grid, nb200::kBlock>>>(g.at(off), n_local);
    if (finish_launch()) return -1;
    OKP(g.down(buf));
    return 0;
}

int okp_fill(double *buf, size_t total, size_t off, double value, size_t n_local, int grid)
{
    if (n_local == 0 || grid < 1) {
        std::snprintf(g_err, sizeof g_err, "okp_fill: n_local or grid out of range");
        return -1;
    }
    Dev g;
    OKP(g.up(buf, total * sizeof(double)));
    nb200::fill_kernel<<<grid, nb200::kBlock>>>(g.at(off), value, n_local);
    if (finish_launch()) return -1;
    OKP(g.down(buf));
    return 0;
}

// sidx_buf may be null (no sigma index); it has the same {total, off} as the sigma buffer
int okp_sigma_init(double *sigma_buf, unsigned short *sidx_buf, size_t total, size_t off, const double *lb,
                   const double *ub, const double *init, double sigma_min, size_t n_local, int grid)
{
    if (n_local == 0 || grid < 1) {
        std::snprintf(g_err, sizeof g_err, "okp_sigma_init: n_local or grid out of range");
        return -1;
    }
    Dev s, i, l, u, in;
    OKP(s.up(sigma_buf, total * sizeof(double)));
    OKP(i.up(sidx_buf, total * sizeof(unsigned short)));
    OKP(l.up(lb, n_local * sizeof(double)));
    OKP(u.up(ub, n_local * sizeof(double)));
    OKP(in.up(init, n_local * sizeof(double)));
    nb200::sigma_init_kernel<<<grid, nb200::kBlock>>>(s.at(off), l.at(0), u.at(0), in.at(0), sigma_min, n_local,
                                                      i.p ? static_cast<unsigned short *>(i.p) + off : nullptr);
    if (finish_launch()) return -1;
    OKP(s.down(sigma_buf));
    OKP(i.down(sidx_buf));
    return 0;
}

// One rank's end_outer_kernel launch.  geo = {n_local, nchunks, chunk0, groups_total, group0, groups_per_vshard,
// local_vshards, groups_local} of nlopt_b200_shard_geometry(n, rank, world); the read-only arrays hold the rank's
// n_local entries, the written ones are {total, off} buffers (xprevprev_buf null: the keep-the-point form).
// publish = 1: the kernel folds its virtual-shard sums itself into out4 (one rank); publish = 0: it writes them into
// its rows of out_dev[8][4] (host, in and out), which okp_publish folds once every rank has run.
int okp_end_outer(const unsigned long long *geo, const double *xcur, double *xprev_buf, double *xprevprev_buf,
                  double *sigma_buf, size_t total, size_t off, const double *lb, const double *ub, const double *w,
                  const double *xtol_abs, int update_sigma, double kappa, double sigma_min, int publish,
                  double *out_dev, double *out4)
{
    const size_t nl = (size_t) geo[0];
    const unsigned groups_local = (unsigned) geo[7], local_vshards = (unsigned) geo[6];
    if (nl == 0 || groups_local == 0 || (update_sigma && !xprevprev_buf)) {
        std::snprintf(g_err, sizeof g_err, "okp_end_outer: empty shard, or a sigma update without xprevprev");
        return -1;
    }
    Dev xc, xp, xpp, sg, l, u, ww, ta, partials, vsums, tickets, od, oh, flag;
    OKP(xc.up(xcur, nl * sizeof(double)));
    OKP(xp.up(xprev_buf, total * sizeof(double)));
    OKP(xpp.up(xprevprev_buf, total * sizeof(double)));
    OKP(sg.up(sigma_buf, total * sizeof(double)));
    OKP(l.up(lb, nl * sizeof(double)));
    OKP(u.up(ub, nl * sizeof(double)));
    OKP(ww.up(w, nl * sizeof(double)));
    OKP(ta.up(xtol_abs, nl * sizeof(double)));
    OKP(partials.zeros((size_t) groups_local * 4 * sizeof(double)));
    OKP(vsums.zeros((size_t) nb200::kVirtualShards * 4 * sizeof(double)));
    OKP(tickets.zeros((nb200::kVirtualShards + 1) * sizeof(unsigned)));
    OKP(od.up(out_dev, (size_t) nb200::kVirtualShards * 4 * sizeof(double)));
    OKP(oh.zeros(4 * sizeof(double)));
    OKP(flag.zeros(sizeof(unsigned long long)));
    nb200::EndOuterArgs a;
    std::memset(&a, 0, sizeof a);
    a.xcur = xc.at(0);
    a.xprev = xp.at(off); a.xprevprev = xpp.at(off); a.sigma = sg.at(off);
    a.lb = l.at(0); a.ub = u.at(0); a.w = ww.at(0); a.xtol_abs = ta.at(0);
    a.n_local = geo[0]; a.nchunks = geo[1]; a.chunk0 = geo[2];
    a.nseg_total = (unsigned) geo[3]; a.seg0 = (unsigned) geo[4]; a.segs_per_vshard = (unsigned) geo[5];
    a.local_vshards = local_vshards;
    a.partials = partials.at(0); a.vsums = vsums.at(0); a.tickets = static_cast<unsigned *>(tickets.p);
    a.out_dev = od.at(0);
    a.out_host = oh.at(0); a.flag_host = static_cast<unsigned long long *>(flag.p);
    a.seq = 1; a.publish_host = publish; a.nvp = 4;
    a.update_sigma = update_sigma; a.kappa = kappa; a.sigma_min = sigma_min;
    nb200::end_outer_kernel<<<(int) groups_local, nb200::kBlock>>>(a);
    if (finish_launch()) return -1;
    OKP(xp.down(xprev_buf));
    OKP(xpp.down(xprevprev_buf));
    OKP(sg.down(sigma_buf));
    OKP(od.down(out_dev));
    if (publish) OKP(oh.down(out4));
    return 0;
}

// publish_kernel on the assembled out_dev[8][4], launched as the library launches it after its all-gather
int okp_publish(const double *out_dev, double *out4)
{
    Dev od, oh, flag;
    OKP(od.up(out_dev, (size_t) nb200::kVirtualShards * 4 * sizeof(double)));
    OKP(oh.zeros(4 * sizeof(double)));
    OKP(flag.zeros(sizeof(unsigned long long)));
    nb200::publish_kernel<<<1, 32>>>(od.at(0), 4, 4, oh.at(0), static_cast<unsigned long long *>(flag.p), 1ull);
    if (finish_launch()) return -1;
    OKP(oh.down(out4));
    return 0;
}

}  // extern "C"
