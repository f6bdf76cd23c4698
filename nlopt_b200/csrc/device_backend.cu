// device_backend.cu -- DeviceBackend: the n-dimensional state of an MMA/CCSAQ run in HBM and the
// launches that act on it.  See device_backend.hpp for the layout and ccsa_kernels.cuh for the
// kernels.  One instance = one rank's shard (the whole problem when there is a single rank).
#include "device_backend.hpp"

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "bounds_kernels.cuh"
#include "ccsa_kernels.cuh"
#include "comm.hpp"
#include "dual_mma.hpp"
#include "nlopt_object.hpp"
#include "synth.cuh"
#include "terms_kernels.cuh"

namespace nb200 {

namespace {

#define NB_CUDA(call)                                   \
    do {                                                \
        cudaError_t e__ = (call);                       \
        if (e__ != cudaSuccess) return fail(#call, e__);\
    } while (0)

// element-wise kernels: one thread per element, at most 16 CTAs per SM (grid-stride beyond)
int grid_for(unsigned long long n, int sms)
{
    const unsigned long long g = (n + kBlock - 1) / kBlock, cap = 16ull * (unsigned long long) sms;
    return (int) (g < 1 ? 1 : (g > cap ? cap : g));
}

// launch-geometry variants of the dual kernel: {threads per CTA, chunks per sweep step, min CTAs/SM}.
// Occupancy matters most; the grid is 4x the resident CTAs (the hardware scheduler evens out the tail better
// than a strictly persistent grid).
struct KernelCfg { int block, unroll, minb; };
constexpr KernelCfg kCfgs[] = {{256, 1, 3}, {256, 1, 4}, {256, 2, 3}, {256, 1, 2}};
constexpr int kNumCfgs = (int) (sizeof(kCfgs) / sizeof(kCfgs[0]));

typedef void (*DualKernel)(const DualArgs);

// measured best geometry per (variant, rows in registers)
constexpr int default_cfg(int variant, int maxm)
{
    return maxm >= 8 ? 3 : maxm == 4 ? (variant == kMMA ? 0 : 1) : (variant == kMMA ? 1 : 2);
}

template <int VARIANT, int MAXM, bool FULL, int CFG, bool SB = false>
DualKernel kernel_for(bool store)
{
    constexpr KernelCfg c = kCfgs[CFG];
    return store ? (DualKernel) dual_eval_kernel<VARIANT, MAXM, FULL, true, c.block, c.unroll, c.minb, SB>
                 : (DualKernel) dual_eval_kernel<VARIANT, MAXM, FULL, false, c.block, c.unroll, c.minb, SB>;
}

// rows kept in registers <= 4: every geometry is built (tuning); 8 or 16 rows need the 128-register budget.
// sb (uniform bounds, no lb / ub loads): built for the default geometry only.
template <int VARIANT, int MAXM, bool FULL>
DualKernel kernel_by_cfg(int cfg, bool store, bool sb)
{
    if (sb) return kernel_for<VARIANT, MAXM, FULL, default_cfg(VARIANT, MAXM), true>(store);
    if (MAXM >= 8) return kernel_for<VARIANT, MAXM, FULL, 3>(store);
    switch (cfg) {
    case 1: return kernel_for<VARIANT, (MAXM >= 8 ? 0 : MAXM), FULL, 1>(store);
    case 2: return kernel_for<VARIANT, (MAXM >= 8 ? 0 : MAXM), FULL, 2>(store);
    case 3: return kernel_for<VARIANT, (MAXM >= 8 ? 0 : MAXM), FULL, 3>(store);
    default: return kernel_for<VARIANT, (MAXM >= 8 ? 0 : MAXM), FULL, 0>(store);
    }
}

template <int VARIANT, bool FULL>
DualKernel pick_kernel(int maxm, int cfg, bool store, bool sb)
{
    switch (maxm) {
    case 0: return kernel_by_cfg<VARIANT, 0, FULL>(cfg, store, sb);
    case 1: return kernel_by_cfg<VARIANT, 1, FULL>(cfg, store, sb);
    case 2: return kernel_by_cfg<VARIANT, 2, FULL>(cfg, store, sb);
    case 4: return kernel_by_cfg<VARIANT, 4, FULL>(cfg, store, sb);
    case 8: return kernel_by_cfg<VARIANT, 8, FULL>(cfg, store, sb);
    default: return kernel_by_cfg<VARIANT, 16, FULL>(cfg, store, sb);
    }
}

// TMA-staged variant (kernel_cfg 10/11/12 = 3/2/4 stages): full-m cases only
template <int VARIANT, int MAXM, int STAGES, int MINB>
DualKernel tma_kernel_for(bool store)
{
    return store ? (DualKernel) dual_eval_tma_kernel<VARIANT, MAXM, true, STAGES, MINB>
                 : (DualKernel) dual_eval_tma_kernel<VARIANT, MAXM, false, STAGES, MINB>;
}

template <int VARIANT>
DualKernel pick_tma_kernel(int maxm, int stages, bool store)
{
    switch (maxm) {
    case 1: return stages == 2 ? tma_kernel_for<VARIANT, 1, 2, 3>(store) : stages == 4 ? tma_kernel_for<VARIANT, 1, 4, 2>(store) : tma_kernel_for<VARIANT, 1, 3, 3>(store);
    case 4: return stages == 2 ? tma_kernel_for<VARIANT, 4, 2, 3>(store) : stages == 4 ? tma_kernel_for<VARIANT, 4, 4, 1>(store) : tma_kernel_for<VARIANT, 4, 3, 2>(store);
    case 16: return stages == 2 ? tma_kernel_for<VARIANT, 16, 2, 1>(store) : tma_kernel_for<VARIANT, 16, 2, 1>(store);
    default: return nullptr;
    }
}

// Process-wide cache of the big allocations (device state pool, pinned staging).  nlopt_optimize
// creates and destroys its state per call like the reference (mma.c:173, :450); cudaMalloc /
// cudaHostAlloc of gigabytes costs tens to hundreds of milliseconds, so freed blocks are parked here
// and handed back to the next call of a similar size.  nlopt_b200_release_cached_memory() empties it.
// Device blocks are keyed by (device ordinal, size): a process whose threads drive different GPUs must never be
// handed a block that lives on another device, and a block is freed with its owner selected.
class BlockCache {
public:
    static int current_device()
    {
        int d = 0;
        cudaGetDevice(&d);
        return d;
    }
    void *take(bool pinned, size_t bytes)
    {
        std::lock_guard<std::mutex> g(mu_);
        auto &pool = pinned ? pinned_ : device_[current_device()];
        auto it = pool.lower_bound(bytes);
        if (it != pool.end() && it->first <= bytes + bytes / 4 + 4096) {
            void *p = it->second;
            pool.erase(it);
            return p;
        }
        return nullptr;
    }
    void give(bool pinned, size_t bytes, void *p, int device = -1)
    {
        std::lock_guard<std::mutex> g(mu_);
        if (device < 0) device = current_device();
        auto &pool = pinned ? pinned_ : device_[device];
        pool.emplace(bytes, p);
        while (pool.size() > 48) {                // keep the cache bounded: drop the smallest block
            auto it = pool.begin();
            if (pinned) cudaFreeHost(it->second); else free_on(device, it->second);
            pool.erase(it);
        }
    }
    void clear()
    {
        std::lock_guard<std::mutex> g(mu_);
        for (auto &d : device_)
            for (auto &e : d.second) free_on(d.first, e.second);
        for (auto &e : pinned_) cudaFreeHost(e.second);
        device_.clear();
        pinned_.clear();
    }
    static BlockCache &get() { static BlockCache c; return c; }

private:
    static void free_on(int device, void *p)
    {
        const int cur = current_device();
        if (cur != device) cudaSetDevice(device);
        cudaFree(p);
        if (cur != device) cudaSetDevice(cur);
    }
    std::mutex mu_;
    std::map<int, std::multimap<size_t, void *>> device_;
    std::multimap<size_t, void *> pinned_;
};

cudaError_t cached_malloc(double **p, size_t bytes)
{
    if (void *q = BlockCache::get().take(false, bytes)) { *p = (double *) q; return cudaSuccess; }
    return cudaMalloc(p, bytes);
}

cudaError_t cached_host_alloc(double **p, size_t bytes)
{
    if (void *q = BlockCache::get().take(true, bytes)) { *p = (double *) q; return cudaSuccess; }
    return cudaHostAlloc(p, bytes, cudaHostAllocMapped);
}

constexpr int kEndNvp = 4;          // end_outer_kernel: record stride (4 sums)
constexpr size_t kGuard = 8;        // doubles of guard around x and xcur (halo cells)

int pick_maxm(int m) { return m == 0 ? 0 : m <= 1 ? 1 : m <= 2 ? 2 : m <= 4 ? 4 : m <= 8 ? 8 : 16; }

std::string no_device_message(cudaError_t e)
{
    return std::string("no usable CUDA device (") + cudaGetErrorString(e) +
           "); libnlopt_b200 runs NLOPT_LD_MMA/NLOPT_LD_CCSAQ on the GPU only";
}

// bounds_check_kernel over n lanes and the copy of its report into pinned host memory, on stream s
cudaError_t enqueue_bounds_check(const double *lb, const double *ub, const double *x, unsigned n, BoundsReport *rep_dev,
                                 BoundsReport *rep_host, int sms, cudaStream_t s)
{
    cudaError_t e = cudaMemsetAsync(rep_dev, 0, sizeof(BoundsReport), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(&rep_dev->first_bad, 0xff, sizeof(unsigned), s);
    if (e != cudaSuccess) return e;
    bounds_check_kernel<<<grid_for(n, sms), kBlock, 0, s>>>(lb, ub, x, n, rep_dev);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return cudaMemcpyAsync(rep_host, rep_dev, sizeof(BoundsReport), cudaMemcpyDeviceToHost, s);
}

void read_bounds_report(const BoundsReport &r, StartCheck *out)
{
    out->bad = r.first_bad == 0xffffffffu ? -1 : (long long) r.first_bad;
    out->lb = r.lb;
    out->x = r.x;
    out->ub = r.ub;
}

}  // namespace

DeviceBackend::DeviceBackend() {}

DeviceBackend::~DeviceBackend()
{
    drain_events();
    for (cudaEvent_t e : ev_pool_) cudaEventDestroy(e);
    free_state();
}

bool DeviceBackend::fail(const char *what, cudaError_t e)
{
    err_ = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
}

bool DeviceBackend::fail(const std::string &what)
{
    err_ = what;
    return false;
}

void DeviceBackend::free_state()
{
    if (stream_) cudaStreamSynchronize(stream_);
    if (copy_stream_) cudaStreamSynchronize(copy_stream_);
    if (pool_) BlockCache::get().give(false, pool_bytes_, pool_, device_);
    if (pen_rows_) BlockCache::get().give(false, (size_t) pen_total_ * geo_.ld * sizeof(double), pen_rows_, device_);
    pen_rows_ = nullptr;
    if (w_dev_) cudaFree(w_dev_);
    if (xtol_abs_dev_) cudaFree(xtol_abs_dev_);
    for (const Owned &o : owned_) BlockCache::get().give(o.pinned, o.bytes, o.p, device_);   // every small buffer
    owned_.clear();
    if (xfull_dev_) BlockCache::get().give(false, (size_t) Comm::instance().world * shard_cap_ * sizeof(double), xfull_dev_, device_);
    solve_state_ = nullptr;
    vs2_dev_ = vs2_host_ = halo_edges_ = nullptr;
    terms_ = terms_part_ = nullptr;
    halo_ptr_ = nullptr;
    grouptags_ = nullptr;
    res_host_ = nullptr;
    wide_dev_ = nullptr;
    if (h_x_) BlockCache::get().give(true, (size_t) geo_.n * sizeof(double), h_x_);
    if (h_xs_) BlockCache::get().give(true, (geo_.n_local ? geo_.n_local : 1) * sizeof(double), h_xs_);
    for (int b = 0; b < 2; ++b) {
        if (h_gs_[b]) BlockCache::get().give(true, (geo_.n_local ? geo_.n_local : 1) * sizeof(double), h_gs_[b]);
        if (h_gs_done_[b]) cudaEventDestroy(h_gs_done_[b]);
        h_gs_[b] = nullptr; h_gs_done_[b] = nullptr;
    }
    h_xs_ = nullptr;
    for (int b = 0; b < 2; ++b) {
        if (h_grad_[b]) BlockCache::get().give(true, h_grad_cap_ * sizeof(double), h_grad_[b]);
        if (h_grad_done_[b]) cudaEventDestroy(h_grad_done_[b]);
    }
    if (stream_) cudaStreamDestroy(stream_);
    if (copy_stream_) cudaStreamDestroy(copy_stream_);
    pool_ = w_dev_ = xtol_abs_dev_ = partials_ = vsums_ = out_dev_ = xfull_dev_ = scalar_dev_ = nullptr;
    tickets_ = nullptr;
    out_host_ = nullptr;
    flag_host_ = nullptr;
    h_x_ = nullptr;
    h_grad_[0] = h_grad_[1] = nullptr;
    h_grad_done_[0] = h_grad_done_[1] = nullptr;
    stream_ = copy_stream_ = nullptr;
}

bool DeviceBackend::alloc_state()
{
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return fail(no_device_message(e));
    Comm &comm = Comm::instance();
    if (comm.active()) {
        device_ = comm.device;
        NB_CUDA(cudaSetDevice(device_));
    } else {
        NB_CUDA(cudaGetDevice(&device_));
    }
    geo_ = Geometry::make(geo_.n, comm.world, comm.rank, target_chunks_, pmax_);
    shard_cap_ = 0;
    for (int r = 0; r < comm.world; ++r) {
        Geometry gr = Geometry::make(geo_.n, comm.world, r, target_chunks_, pmax_);
        if (gr.ld > shard_cap_) shard_cap_ = gr.ld;
    }
    if (m_ > (unsigned) kWideMaxM)
        return fail("more than 2048 inequality constraints: the dual kernel keeps 88 bytes of shared memory per constraint");

    NB_CUDA(cudaDeviceGetAttribute(&sm_count_, cudaDevAttrMultiProcessorCount, device_));
    NB_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    NB_CUDA(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));

    const size_t ld = geo_.ld;
    if (cfg_.values_only) {                  // x | best point
        pool_bytes_ = (2 * ld + 3 * kGuard) * sizeof(double);
        NB_CUDA(cached_malloc(&pool_, pool_bytes_));
        NB_CUDA(cudaMemsetAsync(pool_, 0, pool_bytes_, stream_));
        x_ = pool_ + kGuard;
        xprev_ = x_ + ld + kGuard;
        return alloc_workspace();
    }
    // x and xcur carry kGuard cells on either side: the halo of stencil device callbacks (x[-1], x[ld]); everything
    // stays 64-byte aligned (ld is a multiple of 512 doubles)
    const size_t total = (9 + 2 * (size_t) m_) * ld + 3 * kGuard;
    pool_bytes_ = total * sizeof(double);
    NB_CUDA(cached_malloc(&pool_, pool_bytes_));
    NB_CUDA(cudaMemsetAsync(pool_, 0, total * sizeof(double), stream_));
    double *p = pool_ + kGuard;
    x_ = p; p += ld + kGuard;  xcur_ = p; p += ld + kGuard;  xprev_ = p; p += ld;  xprevprev_ = p; p += ld;
    lb_ = p; p += ld; ub_ = p; p += ld;    sigma_ = p; p += ld;  g_ = p; p += ld;  gcur_ = p; p += ld;
    G_ = p; p += (size_t) m_ * ld;
    Gcur_ = p;
    cand_in_x_ = true;
    return alloc_workspace();
}

// small buffers go through the same cache (cudaMalloc / cudaHostAlloc / cudaFree are slow and synchronising);
// they are handed back in free_state()
bool DeviceBackend::small_dev(void **p, size_t bytes)
{
    double *q = nullptr;
    if (cached_malloc(&q, bytes) != cudaSuccess) return fail("cudaMalloc", cudaGetLastError());
    *p = q;
    owned_.push_back({q, bytes, false});
    return true;
}

bool DeviceBackend::small_pinned(void **p, size_t bytes)
{
    double *q = nullptr;
    if (cached_host_alloc(&q, bytes) != cudaSuccess) return fail("cudaHostAlloc", cudaGetLastError());
    *p = q;
    owned_.push_back({q, bytes, true});
    return true;
}

void DeviceBackend::release_small(void *p)
{
    for (size_t i = 0; i < owned_.size(); ++i)
        if (owned_[i].p == p) {
            BlockCache::get().give(owned_[i].pinned, owned_[i].bytes, p, device_);
            owned_.erase(owned_.begin() + (long) i);
            return;
        }
}

bool DeviceBackend::alloc_workspace()
{
    if (partials_) { release_small(partials_); partials_ = nullptr; }
    if (grouptags_) { release_small(grouptags_); grouptags_ = nullptr; }
    if (vsums_) { release_small(vsums_); vsums_ = nullptr; }
    if (m_ <= (unsigned) kMaxParamM) {
        const int maxm = pick_maxm((int) m_);
        const int nv = 3 + (maxm > 0 ? maxm : 1);
        nvp_ = (nv + 3) / 4 * 4;                  // records are multiples of 32 bytes
    } else {
        nvp_ = (3 + (int) m_ + 3) / 4 * 4;        // wide kernel: 3 + m sums
    }
    const size_t ng = geo_.nseg_local;
    const size_t rec = (size_t) (nvp_ > 24 ? nvp_ : 24);
    if (!small_dev((void **) &partials_, ng * kEndNvp * sizeof(double))) return false;   // end_outer_kernel: one record (4 sums) per group
    // tagged group records {value, tag} of the dual kernels: [nvp][local groups]; tags never repeat (launch ids), so
    // the slots only have to start from zero once
    {
        const size_t bytes = ng * (size_t) nvp_ * 2 * sizeof(double);
        if (!small_dev((void **) &grouptags_, bytes)) return false;
        NB_CUDA(cudaMemsetAsync(grouptags_, 0, bytes, stream_));
    }
    if (!small_dev((void **) &vsums_, (size_t) kV * 24 * sizeof(double))) return false;
    if (out_dev_ && out_rec_ < rec) { release_small(out_dev_); out_dev_ = nullptr; release_small((void *) out_host_); out_host_ = nullptr; }
    if (!out_dev_ && !small_dev((void **) &out_dev_, (size_t) kV * rec * sizeof(double) + 64)) return false;
    if (!tickets_) {
        if (!small_dev((void **) &tickets_, 256)) return false;
        NB_CUDA(cudaMemsetAsync(tickets_, 0, (kV + 1) * sizeof(unsigned), stream_));
    }
    if (!out_host_ && !small_pinned((void **) &out_host_, rec * sizeof(double))) return false;
    out_rec_ = rec;
    if (!flag_host_) {
        if (!small_pinned((void **) &flag_host_, 128)) return false;
        *flag_host_ = 0;
    }
    if (m_ > (unsigned) kMaxParamM && !wide_dev_ && !small_dev((void **) &wide_dev_, 4 * (size_t) m_ * sizeof(double))) return false;
    pend_val_.assign(1 + (size_t) m_, 0.0);
    pend_set_.assign(1 + (size_t) m_, 0);
    NB_CUDA(cudaStreamSynchronize(stream_));
    return true;
}

bool DeviceBackend::setup_raw(Variant v, unsigned n, unsigned m)
{
    variant_ = v;
    m_ = m;
    geo_.n = n;
    cfg_ = BackendConfig();
    cfg_.variant = v;
    cfg_.n = n;
    return alloc_state();
}

bool DeviceBackend::setup(const BackendConfig &cfg)
{
    cfg_ = cfg;
    variant_ = cfg.variant;
    geo_.n = cfg.n;
    m_ = 0;
    max_cdim_ = 1;
    for (const FuncSpec &c : cfg.constraints) {
        m_ += c.m;
        if (c.m > max_cdim_) max_cdim_ = c.m;
    }
    pen_total_ = 0;
    if (cfg.penalty)
        for (int pass = 0; pass < 2; ++pass)
            for (const FuncSpec &c : (pass == 0 ? cfg.penalty->eq : cfg.penalty->ineq)) {
                pen_total_ += c.m;
                if (c.m > max_cdim_) max_cdim_ = c.m;
            }
    terms_rows_ = cfg.objective.dtf ? 1 : 0;
    auto terms_rows_of = [this](const std::vector<FuncSpec> &list) {
        for (const FuncSpec &c : list)
            if (c.dtf && c.m > terms_rows_) terms_rows_ = c.m;
    };
    terms_rows_of(cfg.constraints);
    if (cfg.penalty) {
        terms_rows_of(cfg.penalty->eq);
        terms_rows_of(cfg.penalty->ineq);
    }
    if (cfg.stats) stats_ = cfg.stats;
    if (!alloc_state()) return false;
    const size_t nl = geo_.n_local, j0 = geo_.j0;
    if (cfg.values_only) {
        bool any_host_cb = cfg.objective.f != nullptr;
        for (const FuncSpec &c : cfg.constraints) any_host_cb = any_host_cb || c.f || c.mf;
        if (any_host_cb) NB_CUDA(cached_host_alloc(&h_x_, (size_t) geo_.n * sizeof(double)));
        if (cfg.x0_host) {
            NB_CUDA(cudaMemcpyAsync(x_, cfg.x0_host + j0, nl * sizeof(double), cudaMemcpyHostToDevice, stream_));
            stats_->h2d_bytes += nl * sizeof(double);
        } else if (cfg.x_dev) {
            NB_CUDA(cudaMemcpyAsync(x_, cfg.x_dev, nl * sizeof(double), cudaMemcpyDeviceToDevice, stream_));
        } else
            return fail("no start point");
        NB_CUDA(cudaMemcpyAsync(xprev_, x_, nl * sizeof(double), cudaMemcpyDeviceToDevice, stream_));
        return set_norm_arrays(cfg.x_weights, cfg.xtol_abs);
    }
    if (pen_total_) {
        NB_CUDA(cached_malloc(&pen_rows_, (size_t) pen_total_ * geo_.ld * sizeof(double)));
        NB_CUDA(cudaMemsetAsync(pen_rows_, 0, (size_t) pen_total_ * geo_.ld * sizeof(double), stream_));
    }
    // bounds and start point
    if (cfg.lb_dev) {                         // device bounds: uniformity is known after the check below
        if (Comm::instance().active()) return fail("device bounds run on one rank");
        NB_CUDA(cudaMemcpyAsync(lb_, cfg.lb_dev, nl * sizeof(double), cudaMemcpyDeviceToDevice, stream_));
        NB_CUDA(cudaMemcpyAsync(ub_, cfg.ub_dev, nl * sizeof(double), cudaMemcpyDeviceToDevice, stream_));
    } else {
        if (cfg.lb_uniform) {
            fill_kernel<<<grid_for(nl, sm_count_), kBlock, 0, stream_>>>(lb_, cfg.lb[0], nl);
            ++stats_->kernel_launches;
        } else {
            NB_CUDA(cudaMemcpyAsync(lb_, cfg.lb + j0, nl * sizeof(double), cudaMemcpyHostToDevice, stream_));
            stats_->h2d_bytes += nl * sizeof(double);
        }
        if (cfg.ub_uniform) {
            fill_kernel<<<grid_for(nl, sm_count_), kBlock, 0, stream_>>>(ub_, cfg.ub[0], nl);
            ++stats_->kernel_launches;
        } else {
            NB_CUDA(cudaMemcpyAsync(ub_, cfg.ub + j0, nl * sizeof(double), cudaMemcpyHostToDevice, stream_));
            stats_->h2d_bytes += nl * sizeof(double);
        }
        scalar_bounds_ = cfg.lb_uniform && cfg.ub_uniform;
        lb_u_ = scalar_bounds_ ? cfg.lb[0] : 0.0;
        ub_u_ = scalar_bounds_ ? cfg.ub[0] : 0.0;
    }
    sidx_valid_ = false;
    bool any_host_cb = cfg.objective.f != nullptr;
    for (const FuncSpec &c : cfg.constraints) any_host_cb = any_host_cb || c.f || c.mf;
    if (cfg.penalty)
        for (int pass = 0; pass < 2; ++pass)
            for (const FuncSpec &c : (pass == 0 ? cfg.penalty->eq : cfg.penalty->ineq)) any_host_cb = any_host_cb || c.f || c.mf;
    bool any_sharded_cb = cfg.objective.sf != nullptr;
    for (const FuncSpec &c : cfg.constraints) any_sharded_cb = any_sharded_cb || c.sf;
    if (any_sharded_cb) {
        const size_t cap = geo_.n_local ? geo_.n_local : 1;
        NB_CUDA(cached_host_alloc(&h_xs_, cap * sizeof(double)));
        for (int b = 0; b < 2; ++b) {
            NB_CUDA(cached_host_alloc(&h_gs_[b], cap * sizeof(double)));
            NB_CUDA(cudaEventCreateWithFlags(&h_gs_done_[b], cudaEventDisableTiming));
        }
    }
    if (any_host_cb) {
        NB_CUDA(cached_host_alloc(&h_x_, (size_t) geo_.n * sizeof(double)));
        h_grad_cap_ = (size_t) max_cdim_ * geo_.n;
        for (int b = 0; b < 2; ++b) {
            NB_CUDA(cached_host_alloc(&h_grad_[b], h_grad_cap_ * sizeof(double)));
            NB_CUDA(cudaEventCreateWithFlags(&h_grad_done_[b], cudaEventDisableTiming));
        }
        if (Comm::instance().active())
            NB_CUDA(cached_malloc(&xfull_dev_, (size_t) Comm::instance().world * shard_cap_ * sizeof(double)));
    }
    if (Comm::instance().active()) {
        scalar_cap_ = 1 + (size_t) m_;
        if (!small_dev((void **) &scalar_dev_, (scalar_cap_ + 64) * sizeof(double))) return false;
    }
    if (cfg.x0_host) {
        NB_CUDA(cudaMemcpyAsync(x_, cfg.x0_host + j0, nl * sizeof(double), cudaMemcpyHostToDevice, stream_));
        stats_->h2d_bytes += nl * sizeof(double);
    } else if (cfg.x_dev) {
        NB_CUDA(cudaMemcpyAsync(x_, cfg.x_dev, nl * sizeof(double), cudaMemcpyDeviceToDevice, stream_));
    } else
        return fail("no start point");
    BoundsReport *rep_host = nullptr;
    if (cfg.lb_dev) {                         // before any callback; read back with the synchronisation below
        BoundsReport *rep_dev = nullptr;
        if (!small_dev((void **) &rep_dev, sizeof(BoundsReport))) return false;
        if (!small_pinned((void **) &rep_host, sizeof(BoundsReport))) return false;
        NB_CUDA(enqueue_bounds_check(lb_, ub_, x_, (unsigned) nl, rep_dev, rep_host, sm_count_, stream_));
        ++stats_->kernel_launches;
    }
    if (!set_norm_arrays(cfg.x_weights, cfg.xtol_abs)) return false;
    NB_CUDA(cudaStreamSynchronize(stream_));
    if (rep_host) {
        if (cfg.start_check) read_bounds_report(*rep_host, cfg.start_check);
        scalar_bounds_ = rep_host->nonuniform == 0;
        lb_u_ = scalar_bounds_ ? rep_host->lb0 : 0.0;
        ub_u_ = scalar_bounds_ ? rep_host->ub0 : 0.0;
    }
    if (scalar_bounds_ && m_ == 4) {          // the sigma index and its palette (device + pinned staging), sized for the cap once
        if (!small_dev((void **) &sidx_, geo_.ld * sizeof(unsigned short))) return false;
        if (!small_dev((void **) &pal_, SigmaPalette::kCap * sizeof(double))) return false;
        if (!small_dev((void **) &next_, SigmaPalette::kCap * 3 * sizeof(unsigned short))) return false;
        if (!small_pinned((void **) &pal_pinned_, SigmaPalette::kCap * sizeof(double))) return false;
        if (!small_pinned((void **) &next_pinned_, SigmaPalette::kCap * 3 * sizeof(unsigned short))) return false;
        NB_CUDA(cudaMemsetAsync(sidx_, 0, geo_.ld * sizeof(unsigned short), stream_));
    }
    cand_in_x_ = true;                       // xcur == x at the start (mma.c:220)
    return true;
}

bool DeviceBackend::set_norm_arrays(const double *w_host, const double *xtol_abs_host)
{
    const size_t nl = geo_.n_local, j0 = geo_.j0;
    if (w_dev_) { cudaFree(w_dev_); w_dev_ = nullptr; }
    if (xtol_abs_dev_) { cudaFree(xtol_abs_dev_); xtol_abs_dev_ = nullptr; }
    if (w_host) {
        NB_CUDA(cudaMalloc(&w_dev_, geo_.ld * sizeof(double)));
        NB_CUDA(cudaMemcpyAsync(w_dev_, w_host + j0, nl * sizeof(double), cudaMemcpyHostToDevice, stream_));
    }
    if (xtol_abs_host) {
        NB_CUDA(cudaMalloc(&xtol_abs_dev_, geo_.ld * sizeof(double)));
        NB_CUDA(cudaMemcpyAsync(xtol_abs_dev_, xtol_abs_host + j0, nl * sizeof(double), cudaMemcpyHostToDevice, stream_));
    }
    NB_CUDA(cudaStreamSynchronize(stream_));
    return true;
}

// ------------------------------------------------------------------------------------------------
// sigma

bool DeviceBackend::sigma_init_from(const double *sigma_init_host, double sigma_min)
{
    const size_t nl = geo_.n_local;
    const double *init_dev = nullptr;
    if (sigma_init_host) {           // xprevprev is free until the second outer iteration: use it as scratch
        NB_CUDA(cudaMemcpyAsync(xprevprev_, sigma_init_host + geo_.j0, nl * sizeof(double), cudaMemcpyHostToDevice, stream_));
        stats_->h2d_bytes += nl * sizeof(double);
        init_dev = xprevprev_;
    }
    // the sigma index needs one sigma_0: uniform bounds, and no initial step or the same one for every variable (all of
    // them, so that every rank decides alike); it is kept only when the solve kernel that reads it will run
    sidx_valid_ = sidx_ != nullptr && sigma_index_runs();
    if (sidx_valid_ && sigma_init_host)
        for (size_t j = 1; j < (size_t) geo_.n && sidx_valid_; ++j)
            sidx_valid_ = std::memcmp(sigma_init_host + j, sigma_init_host, sizeof(double)) == 0;
    if (sidx_valid_) {
        palette_.reset(SigmaPalette::sigma0(lb_u_, ub_u_, sigma_init_host ? sigma_init_host[0] : 0.0, sigma_min), lb_u_, ub_u_,
                       variant_ == kMMA ? 0.01 : 1e-8, sigma_min);
        sidx_sigma_min_ = sigma_min;
        pal_uploaded_ = rows_uploaded_ = 0;
        if (!upload_palette()) return false;
    }
    stats_->sigma_palette = sidx_valid_ ? (long long) palette_.val.size() : 0;
    sigma_init_kernel<<<grid_for(nl, sm_count_), kBlock, 0, stream_>>>(sigma_, lb_, ub_, init_dev, sigma_min, nl,
                                                                        sidx_valid_ ? sidx_ : nullptr);
    ++stats_->kernel_launches;
    NB_CUDA(cudaGetLastError());
    return true;
}

bool DeviceBackend::init_sigma(double sigma_min) { return sigma_init_from(cfg_.sigma_init, sigma_min); }

// The sigma-index form of the TMA-staged solve kernel runs -- and only then is the index kept -- with uniform bounds,
// 4 rows, the TMA form chosen by the default rule (knob b200_solve_tma = 1 forces the TMA form with the fp64 sigma),
// no L2 policy, the fused solve, and an fp64 operand set of more than NB200_SIGMA_INDEX_MIN_MB (DESIGN.md section 3.2:
// below it the palette lookup is not paid back).
bool DeviceBackend::sigma_index_runs() const
{
    const size_t operand_bytes = (3 + (size_t) m_) * geo_.ld * sizeof(double);
    return scalar_bounds_ && m_ == 4 && solve_tma_ < 0 && l2_keep_bytes_ == 0 && supports_dual_solve() &&
           operand_bytes > ((size_t) NB200_SIGMA_INDEX_MIN_MB << 20);
}

// the palette entries and transition rows added since the last upload, through pinned staging on the library stream
// (entries are append-only: a slot of the staging is never rewritten while its copy may be in flight)
bool DeviceBackend::upload_palette()
{
    const size_t nv = palette_.val.size(), nr = palette_.rows();
    if (nv > pal_uploaded_) {
        std::memcpy(pal_pinned_ + pal_uploaded_, palette_.val.data() + pal_uploaded_, (nv - pal_uploaded_) * sizeof(double));
        NB_CUDA(cudaMemcpyAsync(pal_ + pal_uploaded_, pal_pinned_ + pal_uploaded_, (nv - pal_uploaded_) * sizeof(double),
                                cudaMemcpyHostToDevice, stream_));
    }
    if (nr > rows_uploaded_) {
        std::memcpy(next_pinned_ + 3 * rows_uploaded_, palette_.next.data() + 3 * rows_uploaded_,
                    3 * (nr - rows_uploaded_) * sizeof(unsigned short));
        NB_CUDA(cudaMemcpyAsync(next_ + 3 * rows_uploaded_, next_pinned_ + 3 * rows_uploaded_,
                                3 * (nr - rows_uploaded_) * sizeof(unsigned short), cudaMemcpyHostToDevice, stream_));
    }
    pal_uploaded_ = nv;
    rows_uploaded_ = nr;
    return true;
}

// ------------------------------------------------------------------------------------------------
// user functions

double *DeviceBackend::staging(unsigned rows)
{
    (void) rows;
    const int b = h_grad_next_;
    h_grad_next_ ^= 1;
    cudaEventSynchronize(h_grad_done_[b]);    // the previous upload out of this buffer has finished
    return h_grad_[b];
}

bool DeviceBackend::host_x_for(Slot slot)
{
    // Host callbacks see the full x.  Single rank: one D2H of the shard (= everything).
    // Several ranks: every rank copies its shard into host memory shared by the ranks of the node (Comm::shared_host);
    // without that, all-gather the shards on the device and copy all of it down on every rank.
    if (h_x_slot_ == (int) slot && h_x_epoch_ == x_epoch_) return true;    // already mirrored
    double *src = slot == kBase ? x_ : xcur_view();
    Comm &comm = Comm::instance();
    if (!comm.active()) {
        h_x_view_ = h_x_;
        NB_CUDA(cudaMemcpyAsync(h_x_, src, geo_.n_local * sizeof(double), cudaMemcpyDeviceToHost, stream_));
        stats_->d2h_bytes += geo_.n_local * sizeof(double);
    } else if (double *shared = comm.shared_host(geo_.n, &err_)) {
        // every rank copies ITS shard into host memory shared by all ranks of the node: n / world doubles per PCIe link
        if (!comm.host_barrier()) return fail("host barrier timed out (a peer rank died?)");    // the previous x has been read by everyone
        NB_CUDA(cudaMemcpyAsync(shared + geo_.j0, src, geo_.n_local * sizeof(double), cudaMemcpyDeviceToHost, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        if (!comm.host_barrier()) return fail("host barrier timed out (a peer rank died?)");    // every shard has landed
        stats_->d2h_bytes += geo_.n_local * sizeof(double);
        h_x_view_ = shared;
        h_x_slot_ = (int) slot;
        h_x_epoch_ = x_epoch_;
        return true;
    } else {
        h_x_view_ = h_x_;
        NB_CUDA(cudaMemcpyAsync(xfull_dev_ + (size_t) comm.rank * shard_cap_, src, geo_.n_local * sizeof(double),
                                cudaMemcpyDeviceToDevice, stream_));
        if (comm.all_gather_inplace(xfull_dev_, shard_cap_, stream_, &err_)) return false;
        for (int r = 0; r < comm.world; ++r) {
            Geometry gr = Geometry::make(geo_.n, comm.world, r, target_chunks_, pmax_);
            NB_CUDA(cudaMemcpyAsync(h_x_ + gr.j0, xfull_dev_ + (size_t) r * shard_cap_, gr.n_local * sizeof(double),
                                    cudaMemcpyDeviceToHost, stream_));
        }
        stats_->d2h_bytes += geo_.n * sizeof(double);
    }
    NB_CUDA(cudaStreamSynchronize(stream_));
    h_x_slot_ = (int) slot;
    h_x_epoch_ = x_epoch_;
    return true;
}

bool DeviceBackend::push_grad_rows(Slot slot, int row0, unsigned rows, bool is_objective, const double *host_grad)
{
    double *dst = is_objective ? (slot == kBase ? g_ : gcur_) : (slot == kBase ? G_ : Gcur_) + (size_t) row0 * geo_.ld;
    return push_rows_to(dst, rows, host_grad);
}

bool DeviceBackend::eval_objective(Slot slot, bool want_grad, double *value)
{
    return cfg_.penalty ? eval_penalty_objective(slot, want_grad, value) : eval_user_objective(slot, want_grad, value);
}

// The augmented-Lagrangian objective (PenaltySpec, backend_factory.hpp; auglag.c:25-65).  The constraint gradients
// go to scratch rows in HBM (uploaded through the same pinned staging pipeline as everything else, or written by
// device callbacks); one kernel then adds the active ones to grad f.  Only the m' + p' values visit the host.
// Asynchronous device callbacks (the objective and nlopt_b200_dfunc2 constraints) are enqueued back to back and settled
// by one finish_evals; the penalty rows take the value slots 1 + m + row of that block.
bool DeviceBackend::eval_penalty_objective(Slot slot, bool want_grad, double *value)
{
    const PenaltySpec &ps = *cfg_.penalty;
    double L = 0;
    if (!eval_user_objective(slot, want_grad, &L)) return false;
    std::vector<double> settled(m_ + (size_t) pen_total_ + 1);   // finish_evals' view: [m] constraints | [pen_total_] rows
    {
        unsigned row = 0;
        for (int pass = 0; pass < 2; ++pass)
            for (const FuncSpec &fs : (pass == 0 ? ps.eq : ps.ineq)) {
                if (fs.async_device() && !enqueue_df2(fs, slot, want_grad ? pen_rows_ + (size_t) row * geo_.ld : nullptr, 1 + m_ + row))
                    return false;
                row += fs.m;
            }
    }
    if (!finish_evals(&L, settled.data())) return false;
    if (ps.nevals_p) ++*ps.nevals_p;
    *value = L;
    if (ps.force_stop && *ps.force_stop) return true;               // auglag.c:39
    std::vector<double> vals(pen_total_ ? pen_total_ : 1);
    double *xs = slot == kBase ? x_ : xcur_view();
    Comm &comm = Comm::instance();
    std::vector<char> partial(pen_total_ ? pen_total_ : 1, 0);
    unsigned row = 0;
    bool any_partial = false;
    for (int pass = 0; pass < 2; ++pass)
        for (const FuncSpec &fs : (pass == 0 ? ps.eq : ps.ineq)) {
            if (fs.async_device()) {
                for (unsigned r = 0; r < fs.m; ++r) vals[row + r] = settled[m_ + row + r];
            } else if (fs.df) {
                const double t0 = wall_seconds();
                vals[row] = fs.df((unsigned) geo_.n_local, geo_.j0, xs, want_grad ? pen_rows_ + (size_t) row * geo_.ld : nullptr, fs.data, stream_);
                cb_seconds_ += wall_seconds() - t0;
                if (comm.active()) { partial[row] = 1; any_partial = true; }
            } else {
                if (!host_x_for(slot)) return false;
                double *grad = want_grad ? staging(fs.m) : nullptr;
                const double t0 = wall_seconds();
                if (fs.f) vals[row] = fs.f((unsigned) geo_.n, h_x_view_, grad, fs.data);        // nlopt_eval_constraint, stop.c:178-184
                else fs.mf(fs.m, &vals[row], (unsigned) geo_.n, h_x_view_, grad, fs.data);
                cb_seconds_ += wall_seconds() - t0;
                if (want_grad && !push_rows_to(pen_rows_ + (size_t) row * geo_.ld, fs.m, grad)) return false;
            }
            row += fs.m;
            if (ps.force_stop && *ps.force_stop) return true;
        }
    if (any_partial) {                 // shard-local values of device callbacks: one all-reduce for all of them
        std::vector<double> buf(pen_total_);
        for (unsigned k = 0; k < pen_total_; ++k) buf[k] = partial[k] ? vals[k] : 0.0;
        double *tmp = nullptr;
        NB_CUDA(cached_malloc(&tmp, pen_total_ * sizeof(double)));
        NB_CUDA(cudaMemcpyAsync(tmp, buf.data(), pen_total_ * sizeof(double), cudaMemcpyHostToDevice, stream_));
        if (comm.all_reduce_sum(tmp, pen_total_, stream_, &err_)) return false;
        NB_CUDA(cudaMemcpyAsync(buf.data(), tmp, pen_total_ * sizeof(double), cudaMemcpyDeviceToHost, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        BlockCache::get().give(false, pen_total_ * sizeof(double), tmp, device_);
        for (unsigned k = 0; k < pen_total_; ++k)
            if (partial[k]) vals[k] = buf[k];
    }
    // values -> L and the coefficients of the gradient rows, in the reference's order (auglag.c:41-62)
    PenaltyCoefs pc;
    pc.count = 0;
    double *gdst = slot == kBase ? g_ : gcur_;
    auto flush = [&]() -> bool {
        if (pc.count && want_grad) {
            penalty_axpy_kernel<<<grid_for(geo_.n_local, sm_count_), kBlock, 0, stream_>>>(gdst, pen_rows_, geo_.ld, geo_.n_local, pc);
            ++stats_->kernel_launches;
            NB_CUDA(cudaGetLastError());
        }
        pc.count = 0;
        return true;
    };
    unsigned neq = 0;
    for (const FuncSpec &fs : ps.eq) neq += fs.m;
    for (unsigned k = 0; k < pen_total_; ++k) {
        double coef = 0;
        bool active = true;
        if (k < neq) {
            const double h = vals[k] + ps.lambda[k] / ps.rho;
            L += 0.5 * ps.rho * h * h;
            coef = ps.rho * h;
        } else {
            const double fc = vals[k] + ps.mu[k - neq] / ps.rho;
            active = fc > 0;
            if (active) { L += 0.5 * ps.rho * fc * fc; coef = ps.rho * fc; }
        }
        if (active) {
            pc.c[pc.count] = coef;
            pc.row[pc.count] = (int) k;
            if (++pc.count == kPenaltyRowsPerLaunch && !flush()) return false;
        }
    }
    if (!flush()) return false;
    *value = L;
    return true;
}

bool DeviceBackend::push_rows_to(double *dst, unsigned rows, const double *host_grad)
{
    const int b = host_grad == h_grad_[0] ? 0 : 1;
    NB_CUDA(cudaMemcpy2DAsync(dst, geo_.ld * sizeof(double), host_grad + geo_.j0, (size_t) geo_.n * sizeof(double),
                              geo_.n_local * sizeof(double), rows, cudaMemcpyHostToDevice, copy_stream_));
    NB_CUDA(cudaEventRecord(h_grad_done_[b], copy_stream_));
    NB_CUDA(cudaStreamWaitEvent(stream_, h_grad_done_[b], 0));     // kernels wait for the upload, the host does not
    stats_->h2d_bytes += (size_t) rows * geo_.n_local * sizeof(double);
    return true;
}

// A maximised device or sharded objective (FuncSpec::negate): the gradient the callback has just written or enqueued on
// the library stream changes sign in place, in stream order before any kernel that reads it.
bool DeviceBackend::negate_gradient(double *g)
{
    if (!g || geo_.n_local == 0) return true;
    negate_kernel<<<grid_for((geo_.n_local + 1) / 2, sm_count_), kBlock, 0, stream_>>>(g, geo_.n_local);
    ++stats_->kernel_launches;
    NB_CUDA(cudaGetLastError());
    return true;
}

// With FuncSpec::negate the objective's value changes sign once it is final: here for one rank, in finish_evals() for
// shard contributions and for the asynchronous form.
bool DeviceBackend::eval_user_objective(Slot slot, bool want_grad, double *value)
{
    const FuncSpec &fs = cfg_.objective;
    if (fs.sf) {
        double *gs = want_grad ? (slot == kBase ? g_ : gcur_) : nullptr;
        if (!eval_sharded(fs, slot, gs, 0, value)) return false;
        if (fs.negate && !Comm::instance().active()) *value = -*value;
        return !fs.negate || negate_gradient(gs);
    }
    if (fs.async_device()) {
        double *gs = want_grad ? (slot == kBase ? g_ : gcur_) : nullptr;
        *value = 0.0;                                  // settled in finish_evals()
        if (!enqueue_df2(fs, slot, gs, 0)) return false;
        return !fs.negate || negate_gradient(gs);
    }
    if (fs.df) {
        double *xs = slot == kBase ? x_ : xcur_view();
        double *gs = want_grad ? (slot == kBase ? g_ : gcur_) : nullptr;
        const double t0 = wall_seconds();
        double v = fs.df((unsigned) geo_.n_local, geo_.j0, xs, gs, fs.data, stream_);
        cb_seconds_ += wall_seconds() - t0;
        if (Comm::instance().active()) {           // shard contributions add up: settled in finish_evals()
            pend_val_[0] = v;
            pend_set_[0] = 1;
            pend_any_ = true;
        } else if (fs.negate)
            v = -v;
        *value = v;
        return !fs.negate || negate_gradient(gs);
    }
    if (!fs.f) return fail("no objective function");
    if (!host_x_for(slot)) return false;
    double *grad = want_grad ? staging(1) : nullptr;
    const double t0 = wall_seconds();
    *value = fs.f((unsigned) geo_.n, h_x_view_, grad, fs.data);
    cb_seconds_ += wall_seconds() - t0;
    if (want_grad) return push_grad_rows(slot, 0, 1, true, grad);
    return true;
}

bool DeviceBackend::eval_constraint(Slot slot, unsigned ic, unsigned row0, bool want_grad, double *values)
{
    const FuncSpec &fs = cfg_.constraints[ic];
    if (fs.sf) return eval_sharded(fs, slot, want_grad ? (slot == kBase ? G_ : Gcur_) + (size_t) row0 * geo_.ld : nullptr, 1 + row0, values);
    if (fs.async_device()) {
        double *gs = want_grad ? (slot == kBase ? G_ : Gcur_) + (size_t) row0 * geo_.ld : nullptr;
        for (unsigned r = 0; r < fs.m; ++r) values[r] = 0.0;
        return enqueue_df2(fs, slot, gs, 1 + row0);
    }
    if (fs.df) {
        double *xs = slot == kBase ? x_ : xcur_view();
        double *gs = want_grad ? (slot == kBase ? G_ : Gcur_) + (size_t) row0 * geo_.ld : nullptr;
        const double t0 = wall_seconds();
        double v = fs.df((unsigned) geo_.n_local, geo_.j0, xs, gs, fs.data, stream_);
        cb_seconds_ += wall_seconds() - t0;
        if (Comm::instance().active()) {
            pend_val_[1 + row0] = v;
            pend_set_[1 + row0] = 1;
            pend_any_ = true;
        }
        values[0] = v;
        return true;
    }
    if (!host_x_for(slot)) return false;       // usually a no-op: the objective call mirrored x already
    double *grad = want_grad ? staging(fs.m) : nullptr;
    const double t0 = wall_seconds();
    if (fs.f) values[0] = fs.f((unsigned) geo_.n, h_x_view_, grad, fs.data);        // nlopt_eval_constraint, stop.c:178-184
    else fs.mf(fs.m, values, (unsigned) geo_.n, h_x_view_, grad, fs.data);
    cb_seconds_ += wall_seconds() - t0;
    if (want_grad) return push_grad_rows(slot, (int) row0, fs.m, false, grad);
    return true;
}

// Device callbacks on several ranks return shard-local values; one all-reduce settles every value of the point
// (1 + m doubles; entries from host callbacks are global already and are not touched).
// Sharded host callbacks (nlopt_b200_sfunc): this rank's n_local variables down, its n_local gradient entries up, the
// additive value contribution settled with the others in finish_evals().
bool DeviceBackend::eval_sharded(const FuncSpec &fs, Slot slot, double *grad_dst, unsigned index, double *value)
{
    const size_t nl = geo_.n_local;
    const double *src = slot == kBase ? x_ : xcur_view();
    if (!(h_xs_slot_ == (int) slot && h_xs_epoch_ == x_epoch_)) {
        NB_CUDA(cudaMemcpyAsync(h_xs_, src, nl * sizeof(double), cudaMemcpyDeviceToHost, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        stats_->d2h_bytes += nl * sizeof(double);
        h_xs_slot_ = (int) slot;
        h_xs_epoch_ = x_epoch_;
    }
    double *grad = nullptr;
    int b = 0;
    if (grad_dst) {
        b = h_gs_next_;
        h_gs_next_ ^= 1;
        cudaEventSynchronize(h_gs_done_[b]);      // the previous upload out of this buffer has finished
        grad = h_gs_[b];
    }
    const double t0 = wall_seconds();
    const double v = fs.sf((unsigned) nl, geo_.j0, geo_.n, h_xs_, grad, fs.data);
    cb_seconds_ += wall_seconds() - t0;
    if (grad_dst) {
        NB_CUDA(cudaMemcpyAsync(grad_dst, grad, nl * sizeof(double), cudaMemcpyHostToDevice, copy_stream_));
        NB_CUDA(cudaEventRecord(h_gs_done_[b], copy_stream_));
        NB_CUDA(cudaStreamWaitEvent(stream_, h_gs_done_[b], 0));
        stats_->h2d_bytes += nl * sizeof(double);
    }
    if (Comm::instance().active()) {
        pend_val_[index] = v;
        pend_set_[index] = 1;
        pend_any_ = true;
    }
    *value = v;
    return true;
}

// Asynchronous device callbacks (nlopt_b200_dfunc2): enqueue, remember which value is pending.  A vector callback
// (nlopt_b200_dmfunc2) takes the m slots [index, index + m) and the m gradient rows from grad_dst on, stride ld; so does
// a terms callback (nlopt_b200_dtfunc, reduce_terms) of m rows.
bool DeviceBackend::enqueue_df2(const FuncSpec &fs, Slot slot, double *grad_dst, unsigned index)
{
    Comm &comm = Comm::instance();
    if (!vs2_dev_) {
        vs2_cap_ = 1 + (size_t) m_ + pen_total_;       // objective | constraints | penalty rows (eval_penalty_objective)
        if (!small_dev((void **) &vs2_dev_, vs2_cap_ * kV * sizeof(double))) return false;
        if (!small_pinned((void **) &vs2_host_, vs2_cap_ * kV * sizeof(double))) return false;
        shard_.n = geo_.n; shard_.n_local = geo_.n_local; shard_.j0 = geo_.j0;
        shard_.nchunks = geo_.nchunks; shard_.chunk0 = geo_.chunk0;
        shard_.groups_total = geo_.S; shard_.group0 = geo_.seg0; shard_.groups_local = geo_.nseg_local; shard_.groups_per_vshard = geo_.P;
        shard_.vshard0 = geo_.seg0 / geo_.P; shard_.local_vshards = geo_.local_vshards;
        shard_.rank = comm.rank; shard_.world = comm.world;
        pend2_.assign(vs2_cap_, nullptr);
    }
    if (!pend2_any_) NB_CUDA(cudaMemsetAsync(vs2_dev_, 0, vs2_cap_ * kV * sizeof(double), stream_));   // first callback of this point
    if (fs.halo > 0 && !ensure_halo(slot)) return false;
    double *xs = slot == kBase ? x_ : xcur_view();
    double *vsums = vs2_dev_ + (size_t) index * kV;
    if (fs.dtf) {
        if (!reduce_terms(fs, xs, grad_dst, vsums)) return false;
    } else {
        const double t0 = wall_seconds();
        if (fs.dmf2) fs.dmf2(fs.m, &shard_, xs, grad_dst, geo_.ld, vsums, fs.data, stream_);
        else fs.df2(&shard_, xs, grad_dst, vsums, fs.data, stream_);
        cb_seconds_ += wall_seconds() - t0;
        NB_CUDA(cudaGetLastError());
    }
    for (unsigned r = 0; r < fs.m; ++r) pend2_[index + r] = &fs;
    pend2_any_ = true;
    return true;
}

// A terms callback (nlopt_b200_dtfunc): the user fills the library's [m][ld] terms buffer on the stream, then
// terms_group_kernel + fold_groups_mkernel reduce each row into its 8 virtual-shard slots at vsums (row i at vsums + 8 i)
// in the order of the __device__ functors' kernels.  One buffer serves every terms callback of the backend: each
// callback's reduction is enqueued before the next callback can write it.
bool DeviceBackend::reduce_terms(const FuncSpec &fs, const double *xs, double *grad_dst, double *vsums)
{
    if (fs.m > 65535) return fail("a terms callback takes at most 65535 rows (one grid row of the reduction each)");
    if (!terms_) {
        const size_t groups = shard_.groups_local ? shard_.groups_local : 1;
        if (!small_dev((void **) &terms_, (size_t) terms_rows_ * geo_.ld * sizeof(double))) return false;
        if (!small_dev((void **) &terms_part_, (size_t) terms_rows_ * groups * sizeof(double))) return false;
    }
    const double t0 = wall_seconds();
    fs.dtf(fs.m, &shard_, xs, grad_dst, geo_.ld, terms_, fs.data, stream_);
    cb_seconds_ += wall_seconds() - t0;
    NB_CUDA(cudaGetLastError());
    if (shard_.groups_local == 0) return true;              // a rank without variables: its slots stay +0.0
    terms_group_kernel<<<dim3(shard_.groups_local, fs.m), kTermsThreads, 0, stream_>>>(shard_, terms_, geo_.ld, terms_part_);
    nlopt_b200::detail::fold_groups_mkernel<<<dim3(shard_.local_vshards, fs.m), kTermsThreads, 0, stream_>>>(
        terms_part_, shard_.groups_local, shard_.groups_per_vshard, vsums + shard_.vshard0);
    stats_->kernel_launches += 2;
    NB_CUDA(cudaGetLastError());
    return true;
}

// The fold of nlopt_b200_device.cuh's trampoline2 (m == 0) / mtrampoline2 (m rows) for the functors compiled at run
// time (jit.cu): the header's fold kernels are defined in this translation unit, and a second one may not define them.
void fold_functor_sums(unsigned m, const double *partials, const nlopt_b200_shard &sh, double *vsums, cudaStream_t s)
{
    if (m == 0)
        nlopt_b200::detail::fold_groups_kernel<<<sh.local_vshards, nlopt_b200::detail::kThreads, 0, s>>>(
            partials, sh.groups_per_vshard, vsums + sh.vshard0);
    else
        nlopt_b200::detail::fold_groups_mkernel<<<dim3(sh.local_vshards, m), nlopt_b200::detail::kThreads, 0, s>>>(
            partials, sh.groups_local, sh.groups_per_vshard, vsums + sh.vshard0);
}

// The halo cells of the slot's x for stencil callbacks: once per point (x_epoch_), only with several ranks.
bool DeviceBackend::ensure_halo(Slot slot)
{
    Comm &comm = Comm::instance();
    if (!comm.active()) return true;
    double *xs = slot == kBase ? x_ : xcur_view();
    if (halo_ptr_ == xs && halo_epoch_ == x_epoch_) return true;
    if (geo_.n_local == 0) return fail("halo exchange: a rank owns no variables (n too small for this many ranks)");
    if (comm.use_p2p()) {
        HaloArgs a;
        std::memset(&a, 0, sizeof a);
        a.x = xs; a.n_local = geo_.n_local; a.right_cell = geo_.n_local;
        for (int r = 0; r < comm.world; ++r) a.box[r] = comm.box_peer[r];
        a.rank = comm.rank; a.world = comm.world;
        a.seq = comm.next_seq();
        halo_exchange_kernel<<<1, 32, 0, stream_>>>(a);
    } else {
        if (!halo_edges_ && !small_dev((void **) &halo_edges_, 2 * 8 * sizeof(double))) return false;
        halo_pack_kernel<<<1, 32, 0, stream_>>>(xs, geo_.n_local, halo_edges_, comm.rank);
        if (comm.all_gather_inplace(halo_edges_, 2, stream_, &err_)) return false;
        halo_apply_kernel<<<1, 32, 0, stream_>>>(xs, geo_.n_local, halo_edges_, comm.rank, comm.world);
    }
    ++stats_->kernel_launches;
    NB_CUDA(cudaGetLastError());
    halo_ptr_ = xs;
    halo_epoch_ = x_epoch_;
    return true;
}

bool DeviceBackend::finish_evals(double *fvalue, double *cvalues)
{
    if (pend2_any_) {
        // one exchange + one copy + one synchronisation for all values of the point.  Every slot of the [1+m][8] block
        // is non-zero on exactly one rank, so the all-reduce is exact whatever its internal order; the 8 shard sums are
        // then added in index order: the value does not depend on the number of ranks.
        Comm &comm = Comm::instance();
        if (comm.active() && comm.all_reduce_sum(vs2_dev_, vs2_cap_ * kV, stream_, &err_)) return false;
        NB_CUDA(cudaMemcpyAsync(vs2_host_, vs2_dev_, vs2_cap_ * kV * sizeof(double), cudaMemcpyDeviceToHost, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        size_t step = 1;
        for (size_t i = 0; i < vs2_cap_; i += step) {
            const FuncSpec *fs = pend2_[i];
            step = 1;
            if (!fs) continue;
            if (fs->dmfin) {           // a vector constraint: its m rows, one finish call (never the objective's slot 0)
                step = fs->m;
                if (!cvalues) continue;
                std::vector<double> tots(fs->m);
                for (unsigned r = 0; r < fs->m; ++r) {
                    const double *vs = vs2_host_ + (i + r) * kV;
                    double tot = vs[0];
                    for (unsigned v = 1; v < kV; ++v) tot += vs[v];
                    tots[r] = tot;
                }
                fs->dmfin(fs->m, tots.data(), cvalues + i - 1, fs->data);
                for (unsigned r = 0; r < fs->m; ++r) pend2_[i + r] = nullptr;
                continue;
            }
            double tot = vs2_host_[i * kV];
            for (unsigned v = 1; v < kV; ++v) tot += vs2_host_[i * kV + v];
            const double val = fs->dfin(tot, fs->data);
            if (i == 0) { if (fvalue) *fvalue = fs->negate ? -val : val; else continue; }
            else { if (cvalues) cvalues[i - 1] = val; else continue; }
            pend2_[i] = nullptr;
        }
        pend2_any_ = false;
        for (const FuncSpec *q : pend2_) pend2_any_ = pend2_any_ || q != nullptr;
    }
    if (!pend_any_) return true;
    Comm &comm = Comm::instance();
    const size_t cnt = 1 + (size_t) m_;
    std::vector<double> buf(cnt);
    for (size_t i = 0; i < cnt; ++i) buf[i] = pend_set_[i] ? pend_val_[i] : 0.0;
    if (cnt > scalar_cap_) {
        if (scalar_dev_) release_small(scalar_dev_);
        scalar_dev_ = nullptr;
        if (!small_dev((void **) &scalar_dev_, (cnt + 64) * sizeof(double))) return false;
        scalar_cap_ = cnt;
    }
    NB_CUDA(cudaMemcpyAsync(scalar_dev_, buf.data(), cnt * sizeof(double), cudaMemcpyHostToDevice, stream_));
    if (comm.all_reduce_sum(scalar_dev_, cnt, stream_, &err_)) return false;
    NB_CUDA(cudaMemcpyAsync(buf.data(), scalar_dev_, cnt * sizeof(double), cudaMemcpyDeviceToHost, stream_));
    NB_CUDA(cudaStreamSynchronize(stream_));
    if (fvalue && pend_set_[0]) { *fvalue = cfg_.objective.negate ? -buf[0] : buf[0]; pend_set_[0] = 0; }
    if (cvalues)
        for (unsigned i = 0; i < m_; ++i)
            if (pend_set_[1 + i]) { cvalues[i] = buf[1 + i]; pend_set_[1 + i] = 0; }
    pend_any_ = false;
    for (size_t i = 0; i < cnt; ++i) pend_any_ = pend_any_ || pend_set_[i];
    return true;
}

// Collective OR of a rank-local decision (the time limit): one 8-byte all-reduce.  Every rank calls it at the same
// points of the driver loop (ccsa_driver.cpp: Loop::timed_out), so the ranks cannot disagree about MAXTIME.
bool DeviceBackend::agree_any(bool local)
{
    Comm &comm = Comm::instance();
    if (!comm.active()) return local;
    double v = local ? 1.0 : 0.0;
    double *slot = scalar_dev_ + scalar_cap_;          // the spare doubles behind the value buffer
    if (cudaMemcpyAsync(slot, &v, sizeof v, cudaMemcpyHostToDevice, stream_) != cudaSuccess) return local;
    if (comm.all_reduce_sum(slot, 1, stream_, &err_)) return local;
    if (cudaMemcpyAsync(&v, slot, sizeof v, cudaMemcpyDeviceToHost, stream_) != cudaSuccess) return local;
    if (cudaStreamSynchronize(stream_) != cudaSuccess) return local;
    return v > 0.0;
}

// ------------------------------------------------------------------------------------------------
// dual evaluation

bool DeviceBackend::wait_flag()
{
    // The kernel's last CTA writes the sums and then the sequence number into mapped pinned
    // memory; polling it is a few microseconds cheaper than a stream synchronise per evaluation.
    const auto t0 = std::chrono::steady_clock::now();
    unsigned long spins = 0;
    for (;;) {
        if (__atomic_load_n(flag_host_, __ATOMIC_ACQUIRE) == seq_) return true;
        if ((++spins & 0x3fff) == 0) {
            cudaError_t q = cudaStreamQuery(stream_);
            if (q != cudaSuccess && q != cudaErrorNotReady) return fail("dual kernel", q);
            if (q == cudaSuccess) {
                if (__atomic_load_n(flag_host_, __ATOMIC_ACQUIRE) == seq_) return true;
                return fail("dual kernel finished without publishing its result");
            }
            // a whole dual solve (up to dual_maxeval evaluations) can legitimately run for minutes at n = 1e8;
            // in-kernel timeouts cover dead peers, this one only a kernel that never ends
            if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > 3600.0)
                return fail("timed out waiting for the dual kernel");
        }
    }
}

// operand arrays to load evict_last (DualArgs::l2_keep), in order of preference: the arrays that never move
// (sigma, lb, ub), then x, grad f and the gradient rows -- as many as fit into l2_keep_bytes_
unsigned DeviceBackend::l2_keep_mask() const
{
    if (l2_keep_bytes_ == 0) return 0u;
    const size_t per = geo_.ld * sizeof(double);
    size_t budget = l2_keep_bytes_ / (per ? per : 1);
    static const int order[5] = {3, 1, 2, 0, 4};
    unsigned mask = 0;
    for (int k = 0; k < 5 && budget > 0; ++k, --budget) mask |= 1u << order[k];
    for (unsigned i = 0; i < m_ && i < (unsigned) kMaxParamM && budget > 0; ++i, --budget) mask |= 1u << (5 + i);
    return mask;
}

void DeviceBackend::fill_dual_args(DualArgs &a, const double *y, const DualScalars &sc)
{
    std::memset(&a, 0, sizeof a);
    a.x = x_; a.lb = lb_; a.ub = ub_; a.sigma = sigma_; a.g = g_; a.G = G_;
    a.lb_u = lb_u_; a.ub_u = ub_u_;
    a.sidx = sidx_valid_ ? sidx_ : nullptr; a.pal = pal_;
    a.xcur = xcur_;
    a.ld = geo_.ld;
    a.nchunks = geo_.nchunks; a.chunk0 = geo_.chunk0;
    a.nseg_total = geo_.S; a.seg0 = geo_.seg0; a.segs_per_vshard = geo_.P; a.local_vshards = geo_.local_vshards;
    a.grouptags = grouptags_;
    a.tag = (1ull << 63) | ++eval_tag_;          // the solve kernel's tags (launch id << 40 | generation) stay below 2^63
    a.out_dev = out_dev_;
    a.out_host = out_host_; a.flag_host = flag_host_;
    a.seq = seq_ = Comm::instance().active() ? Comm::instance().next_seq() : seq_ + 1;
    a.publish_host = Comm::instance().active() ? 0 : 1;
    a.nvp = nvp_;
    const bool wide = m_ > (unsigned) kMaxParamM;
    {
        Comm &cm = Comm::instance();
        a.rank = cm.rank;
        a.world = cm.world;
        // the mailbox holds records of <= 19 sums: the wide kernel exchanges through ncclAllGather
        for (int r = 0; r < 8; ++r) a.box[r] = (cm.active() && cm.use_p2p() && !wide && r < cm.world) ? cm.box_peer[r] : nullptr;
    }
    a.l2_keep = l2_keep_mask();
    a.m = (int) m_;
    a.rho = sc.rho;
    a.half_rho = 0.5 * sc.rho;
    a.active = 0;
    double u = sc.rho;                                   // ccsa_quadratic.c:116-120, j-independent
    if (wide) wide_host_.resize(4 * (size_t) m_);
    for (unsigned i = 0; i < m_; ++i) {
        const bool on = !(variant_ == kMMA && std::isnan(sc.fcval[i]));
        if (wide) {
            wide_host_[i] = y[i];
            wide_host_[m_ + i] = sc.rhoc[i];
            wide_host_[2 * (size_t) m_ + i] = 0.5 * sc.rhoc[i];
            wide_host_[3 * (size_t) m_ + i] = on ? 1.0 : 0.0;
        } else {
            a.y[i] = y[i];
            a.rhoc[i] = sc.rhoc[i];
            a.half_rhoc[i] = 0.5 * sc.rhoc[i];
            if (on) a.active |= 1u << i;
        }
        u += sc.rhoc[i] * y[i];
    }
    a.u_ccsaq = u;
    a.wide = wide_dev_;
}

// what `evals` dual evaluations asked HBM for: 3 + m operand arrays with scalar bounds, 5 + m without, + the x* store;
// with the sigma index (si) 2 bytes per variable replace the sigma array
void DeviceBackend::count_operand_bytes(long long evals, bool sb, bool si, bool store)
{
    const long long per = (long long) (8 * geo_.ld);
    stats_->dual_operand_bytes += evals * (per * ((sb ? 3 : 5) - (si ? 1 : 0) + (long long) m_) + (si ? per / 4 : 0)) + (store ? per : 0);
}

bool DeviceBackend::launch_dual(const double *y, const DualScalars &sc, bool store, bool wait)
{
    DualArgs a;
    fill_dual_args(a, y, sc);

    const bool wide = m_ > (unsigned) kMaxParamM;
    const int maxm = pick_maxm((int) m_);
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (time_kernels_) {
        if (ev_used_ + 2 > ev_pool_.size()) {
            if (ev_pool_.size() >= 8192) drain_events();
            else
                for (int k = 0; k < 512; ++k) { cudaEvent_t e; cudaEventCreate(&e); ev_pool_.push_back(e); }
        }
        e0 = ev_pool_[ev_used_++];
        e1 = ev_pool_[ev_used_++];
        cudaEventRecord(e0, stream_);
    }
    const bool full_m = !wide && (int) m_ == maxm && (variant_ == kCCSAQ || a.active == ((1u << m_) - 1u));
    // MMA with 16 gradient rows is register-starved in the register form; the TMA-staged form is the default
    // there.  Everywhere else the register form is faster and the TMA form is opt-in (kernel_cfg 10 / 11 / 12 = 3 / 2 / 4 stages).
    const bool tma_default = kernel_cfg_ < 0 && variant_ == kMMA && maxm == 16 && full_m;
    bool sb = false;
    if (wide) {
        // any number of constraints: rows streamed in blocks of 8, per-row scalars in dynamic shared memory
        NB_CUDA(cudaMemcpyAsync(wide_dev_, wide_host_.data(), 4 * (size_t) m_ * sizeof(double), cudaMemcpyHostToDevice, stream_));
        DualKernel fn = variant_ == kMMA ? (store ? (DualKernel) dual_eval_wide_kernel<0, true> : (DualKernel) dual_eval_wide_kernel<0, false>)
                                         : (store ? (DualKernel) dual_eval_wide_kernel<1, true> : (DualKernel) dual_eval_wide_kernel<1, false>);
        const size_t mp = ((size_t) m_ + kWideRows - 1) / kWideRows * kWideRows;
        const size_t smem = 12 * mp * sizeof(double);
        NB_CUDA(cudaFuncSetAttribute((const void *) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
        int per_sm = 0;
        NB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kBlock, smem));
        if (per_sm < 1) return fail("dual_eval_wide_kernel does not fit on an SM");
        long long pgrid = (long long) sm_count_ * (ctas_per_sm_ > 0 ? ctas_per_sm_ : per_sm);
        if (pgrid > (long long) geo_.nseg_local) pgrid = geo_.nseg_local;
        fn<<<(unsigned) (pgrid < 1 ? 1 : pgrid) + 1, kBlock, smem, stream_>>>(a);
    } else if ((tma_default || (kernel_cfg_ >= 10 && kernel_cfg_ <= 12)) && full_m && (maxm == 1 || maxm == 4 || maxm == 16)) {
        // TMA-staged form: producer warp + 8 consumer warps, dynamic shared memory = stages x (5+m) x 4 KB
        int stages = kernel_cfg_ == 10 ? 3 : kernel_cfg_ == 11 ? 2 : kernel_cfg_ == 12 ? 4 : 2;
        if (maxm == 16) stages = 2;
        DualKernel fn = variant_ == kMMA ? pick_tma_kernel<0>(maxm, stages, store) : pick_tma_kernel<1>(maxm, stages, store);
        const size_t smem = (size_t) stages * (5 + maxm) * kChunkBytes;
        NB_CUDA(cudaFuncSetAttribute((const void *) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
        int per_sm = 0;
        NB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kTmaBlock, smem));
        if (per_sm < 1) return fail("dual_eval_tma_kernel does not fit on an SM");
        long long pgrid = (long long) sm_count_ * (ctas_per_sm_ > 0 ? ctas_per_sm_ : 6);     // oversubscribed 2-3x: evens out the tail
        if (pgrid > (long long) geo_.nseg_local) pgrid = geo_.nseg_local;
        fn<<<(unsigned) (pgrid < 1 ? 1 : pgrid) + 1, kTmaBlock, smem, stream_>>>(a);
    } else {
        // persistent kernel: the grid is sized to the machine, not to the problem (+ the folder CTA)
        int cfg = kernel_cfg_ >= 0 && kernel_cfg_ < kNumCfgs ? kernel_cfg_ : default_cfg(variant_, maxm);
        if (maxm >= 8) cfg = 3;
        sb = scalar_bounds_ && cfg == default_cfg(variant_, maxm);
        const KernelCfg c = kCfgs[cfg];
        DualKernel fn = variant_ == kMMA ? (full_m ? pick_kernel<0, true>(maxm, cfg, store, sb) : pick_kernel<0, false>(maxm, cfg, store, sb))
                                         : (full_m ? pick_kernel<1, true>(maxm, cfg, store, sb) : pick_kernel<1, false>(maxm, cfg, store, sb));
        const long long want = (long long) geo_.nseg_local;
        const long long cap = (long long) sm_count_ * (ctas_per_sm_ > 0 ? ctas_per_sm_ : 4 * c.minb);
        const int pgrid = (int) (want < cap ? want : cap);
        fn<<<(pgrid < 1 ? 1 : pgrid) + 1, c.block, 0, stream_>>>(a);
    }
    if (time_kernels_) cudaEventRecord(e1, stream_);
    ++stats_->kernel_launches;
    NB_CUDA(cudaGetLastError());
    count_operand_bytes(1, sb, false, store);
    if (!a.publish_host && a.box[0] == nullptr) {
        const int nv = wide ? 3 + (int) m_ : 3 + (maxm > 0 ? maxm : 1);
        if (Comm::instance().all_gather_inplace(out_dev_, (size_t) geo_.local_vshards * nvp_, stream_, &err_)) return false;
        publish_kernel<<<1, 256, 0, stream_>>>(out_dev_, nv, nvp_, out_host_, flag_host_, a.seq);
        ++stats_->kernel_launches;
        NB_CUDA(cudaGetLastError());
    }
    return wait ? wait_flag() : true;
}

bool DeviceBackend::dual_eval(const double *y, const DualScalars &sc, bool materialize, DualSums *out)
{
    if (materialize) { cand_in_x_ = false; ++x_epoch_; }   // xcur_ is about to hold the candidate
    if (!launch_dual(y, sc, materialize, true)) return false;
    if (Comm::instance().active() && std::isnan(out_host_[0]) && std::isnan(out_host_[1]) && std::isnan(out_host_[2]))
        return fail("the cross-rank exchange of the dual sums timed out or produced NaN (is every rank running the same calls?)");
    out->val = out_host_[0];
    out->gval = out_host_[1];
    out->wval = out_host_[2];
    for (unsigned k = 0; k < m_; ++k) out->gc[k] = out_host_[3 + k];
    return true;
}

// ------------------------------------------------------------------------------------------------
// one launch per dual solve (persistent cooperative kernel, ccsa_kernels.cuh: dual_solve_kernel)

namespace {
typedef void (*SolveKernel)(const SolveArgs);

// One configuration per row count.  Two alternatives were measured and removed:
// two chunks in flight per sweep step (slower at n = 1e7 over 8 GPUs) and 4 CTAs/SM at 64 registers (spills).
#ifndef NB200_SOLVE_MINB4
#define NB200_SOLVE_MINB4 3      // A/B switch (tools/ab_build.py): resident CTAs per SM of the solve kernel with <= 4 rows
#endif
// `roomy`: the 2-CTAs/SM instantiation (128 registers, no spills in the sweep or in the folder's optimiser turn) -- used
// when the grid does not need a third CTA per SM anyway (small and mid-size shards), see DeviceBackend::dual_solve
// SB: uniform bounds as two scalars (never combined with POL)
template <int VARIANT, bool FULL, bool POL, bool SB>
SolveKernel pick_solve_kernel(int maxm, bool roomy)
{
    if (roomy) switch (maxm) {
        case 1: return dual_solve_kernel<VARIANT, 1, FULL, POL, 256, 2, SB>;
        case 2: return dual_solve_kernel<VARIANT, 2, FULL, POL, 256, 2, SB>;
        case 4: return dual_solve_kernel<VARIANT, 4, FULL, POL, 256, 2, SB>;
        default: break;
        }
    switch (maxm) {
    case 1: return dual_solve_kernel<VARIANT, 1, FULL, POL, 256, NB200_SOLVE_MINB4, SB>;
    case 2: return dual_solve_kernel<VARIANT, 2, FULL, POL, 256, NB200_SOLVE_MINB4, SB>;
    case 4: return dual_solve_kernel<VARIANT, 4, FULL, POL, 256, NB200_SOLVE_MINB4, SB>;
    case 8: return dual_solve_kernel<VARIANT, 8, FULL, POL, 256, 2, SB>;
    default: return dual_solve_kernel<VARIANT, 16, FULL, POL, 256, 2, SB>;
    }
}
// TMA-staged form (full-m, 1 / 2 / 4 rows): {stages, bytes of dynamic shared memory}.  A stage is (5 + m) x 4 KB,
// (3 + m) x 4 KB with uniform bounds (kScalarBounds), (2 + m) x 4 KB + 1 KB with the sigma index (kSigmaIndex).
// 3 CTAs per SM, except 4 rows with uniform bounds: 3 stages of 28 KB (25 KB with the sigma index) at 2 CTAs/SM
// (96 registers, no spills for CCSAQ) -- on the H100 at n = 1e7 198-206 us per evaluation against 236-241 us for
// 2 stages at 3 CTAs/SM (72 registers, 88 B of spills), DESIGN.md section 3.2.
#ifndef NB200_SOLVE_TMA_IDX_STAGES4
#define NB200_SOLVE_TMA_IDX_STAGES4 3   // A/B switch (tools/ab_build.py): stages of the sigma-index form with 4 rows
#endif
template <int VARIANT, int BM>
SolveKernel pick_solve_tma_kernel(int maxm, size_t *smem)
{
    constexpr size_t stage = (BM == kBoundArrays ? 5 : BM == kScalarBounds ? 3 : 2) * (size_t) kChunkBytes + (BM == kSigmaIndex ? kIdxChunkBytes : 0);
    if constexpr (BM == kSigmaIndex) {      // 4 rows only (DeviceBackend::sigma_index_runs)
        *smem = NB200_SOLVE_TMA_IDX_STAGES4 * (stage + 4 * kChunkBytes);
        return maxm == 4 ? dual_solve_tma_kernel<VARIANT, 4, NB200_SOLVE_TMA_IDX_STAGES4, 2, BM> : nullptr;
    } else {
        switch (maxm) {
        case 1: *smem = 3 * (stage + 1 * kChunkBytes); return dual_solve_tma_kernel<VARIANT, 1, 3, 3, BM>;
        case 2: *smem = 2 * (stage + 2 * kChunkBytes); return dual_solve_tma_kernel<VARIANT, 2, 2, 3, BM>;
        case 4:
            if constexpr (BM == kScalarBounds) { *smem = 3 * (stage + 4 * kChunkBytes); return dual_solve_tma_kernel<VARIANT, 4, 3, 2, BM>; }
            else { *smem = 2 * (stage + 4 * kChunkBytes); return dual_solve_tma_kernel<VARIANT, 4, 2, 3, BM>; }
        default: *smem = 0; return nullptr;
        }
    }
}
template <int VARIANT>
SolveKernel pick_solve_tma_kernel1(int bm, int maxm, size_t *smem)
{
    return bm == kSigmaIndex ? pick_solve_tma_kernel<VARIANT, kSigmaIndex>(maxm, smem)
         : bm == kScalarBounds ? pick_solve_tma_kernel<VARIANT, kScalarBounds>(maxm, smem)
                               : pick_solve_tma_kernel<VARIANT, kBoundArrays>(maxm, smem);
}

// asynchronous operand pipeline (dual_solve_async_kernel): {stages} x (5 + rows) x 4 KB of dynamic shared memory per CTA.
// <= 2 rows: 3 CTAs/SM at 80 registers; 4 or 8 rows: the ring leaves room for 2 CTAs/SM, which get 128 registers.
template <int VARIANT, bool FULL, int STAGES>
SolveKernel pick_solve_async_kernel(int maxm)
{
    switch (maxm) {
    case 1: return dual_solve_async_kernel<VARIANT, 1, FULL, STAGES, 3>;
    case 2: return dual_solve_async_kernel<VARIANT, 2, FULL, STAGES, 3>;
    case 4: return dual_solve_async_kernel<VARIANT, 4, FULL, STAGES, 2>;
    case 8: return dual_solve_async_kernel<VARIANT, 8, FULL, STAGES, 2>;
    default: return nullptr;
    }
}
template <int VARIANT>
SolveKernel pick_solve_async_kernel2(int maxm, bool full, int stages)
{
    if (stages == 2) return full ? pick_solve_async_kernel<VARIANT, true, 2>(maxm) : pick_solve_async_kernel<VARIANT, false, 2>(maxm);
    return full ? pick_solve_async_kernel<VARIANT, true, 3>(maxm) : pick_solve_async_kernel<VARIANT, false, 3>(maxm);
}

template <int VARIANT, bool FULL>
SolveKernel pick_solve_kernel1(int maxm, bool pol, bool sb, bool roomy)
{
    if (pol) return pick_solve_kernel<VARIANT, FULL, true, false>(maxm, roomy);
    return sb ? pick_solve_kernel<VARIANT, FULL, false, true>(maxm, roomy) : pick_solve_kernel<VARIANT, FULL, false, false>(maxm, roomy);
}
template <int VARIANT>
SolveKernel pick_solve_kernel2(int maxm, bool full, bool pol, bool sb, bool roomy)
{
    return full ? pick_solve_kernel1<VARIANT, true>(maxm, pol, sb, roomy) : pick_solve_kernel1<VARIANT, false>(maxm, pol, sb, roomy);
}
}  // namespace

bool DeviceBackend::supports_dual_solve() const
{
    // several ranks: the in-kernel optimiser needs the in-kernel (mailbox) exchange
    const Comm &cm = Comm::instance();
    if (cm.active() && !cm.use_p2p()) return false;
    if (variant_ == kMMA && m_ > 8) return false;      // the TMA-staged evaluation kernel wins there (see launch_dual)
    return fused_solve_ok_ && m_ >= 1 && m_ <= (unsigned) kMaxParamM;
}

bool DeviceBackend::dual_solve(double *y, const double *lo, const double *hi, const double *stop6, const DualScalars &sc,
                               DualSums *out, int *ret, long *nevals)
{
    if (!solve_state_) {
        if (!small_dev(&solve_state_, (sizeof(SolveState) + 255) / 256 * 256)) return false;
        NB_CUDA(cudaMemsetAsync(solve_state_, 0, sizeof(SolveState), stream_));
        if (!small_pinned((void **) &res_host_, 64 * sizeof(double))) return false;
        static_assert(kResCounts + 3 <= 64, "result record");
    }
    SolveArgs sa;
    fill_dual_args(sa.d, y, sc);
    sa.st = static_cast<SolveState *>(solve_state_);
    if (solve_launch_id_ >= (1ull << 22)) {       // tags are (launch id, generation): start from a clean slate
        const size_t bytes = (size_t) geo_.nseg_local * nvp_ * 2 * sizeof(double);
        NB_CUDA(cudaMemsetAsync(grouptags_, 0, bytes, stream_));
        NB_CUDA(cudaMemsetAsync(solve_state_, 0, sizeof(SolveState), stream_));
        solve_launch_id_ = 0;
    }
    sa.tag0 = ++solve_launch_id_ << 40;
    sa.fval = sc.fval;
    for (unsigned i = 0; i < (unsigned) kMaxParamM; ++i) {
        sa.cval[i] = i < m_ ? ((variant_ == kMMA && std::isnan(sc.fcval[i])) ? 0.0 : sc.fcval[i]) : 0.0;
        sa.lo[i] = i < m_ ? lo[i] : 0.0;
        sa.hi[i] = i < m_ ? hi[i] : 0.0;
    }
    sa.stop.ftol_rel = stop6[0]; sa.stop.ftol_abs = stop6[1]; sa.stop.xtol_rel = stop6[2]; sa.stop.xtol_abs = stop6[3];
    sa.stop.maxeval = (int) stop6[4]; sa.stop.maxtime = stop6[5];
    sa.res_host = res_host_;
#ifdef NB200_TRACE
    static unsigned long long *trace_buf = nullptr;
    if (!trace_buf) NB_CUDA(cudaMalloc(&trace_buf, sizeof(unsigned long long) * 16 * kTraceGens));
    NB_CUDA(cudaMemsetAsync(trace_buf, 0, sizeof(unsigned long long) * 16 * kTraceGens, stream_));
    sa.trace = trace_buf;
#endif

    const int maxm = pick_maxm((int) m_);
    const bool full = (int) m_ == maxm && (variant_ == kCCSAQ || sa.d.active == ((1u << m_) - 1u));
    const bool use_pol = sa.d.l2_keep != 0u;
    // With uniform bounds the TMA-staged form, whose producer warp keeps the next chunks in flight during the arithmetic
    // and across group and generation boundaries, is the default for 4 rows at every size measured (n = 1.25e6 .. 5e7,
    // MMA and CCSAQ) and for 1 row up to 80 MB of operands (n <= 2.5e6); above that the two forms tie with 1 row, and
    // CCSAQ lost 8 % at n = 5e7.  2 rows (not measured), bound arrays and L2 policies keep the register form
    // (DESIGN.md section 3.2; knob b200_solve_tma: 1 always, 0 never).
    const size_t operand_bytes = (3 + (size_t) m_) * geo_.ld * sizeof(double);
    const bool tma_auto = solve_tma_ < 0 && scalar_bounds_ && (maxm == 4 || (maxm == 1 && operand_bytes <= ((size_t) 80 << 20)));
    size_t smem = 0;
    int block = 256;
    SolveKernel fn = nullptr;
    bool sb = false, si = false;
    if ((solve_tma_ > 0 || tma_auto) && full && !use_pol && (maxm == 1 || maxm == 2 || maxm == 4)) {
        sb = scalar_bounds_;
        si = sidx_valid_ && maxm == 4;             // see sigma_index_runs()
        const int bm = si ? kSigmaIndex : sb ? kScalarBounds : kBoundArrays;
        fn = variant_ == kMMA ? pick_solve_tma_kernel1<0>(bm, maxm, &smem) : pick_solve_tma_kernel1<1>(bm, maxm, &smem);
        block = kTmaBlock;
        NB_CUDA(cudaFuncSetAttribute((const void *) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    } else if (solve_async_ >= 2 && !use_pol && maxm <= 8) {
        const int stages = solve_async_ >= 3 ? 3 : 2;
        fn = variant_ == kMMA ? pick_solve_async_kernel2<0>(maxm, full, stages) : pick_solve_async_kernel2<1>(maxm, full, stages);
        smem = (size_t) stages * (5 + (size_t) maxm) * kChunkBytes;
        NB_CUDA(cudaFuncSetAttribute((const void *) fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
    } else {
        // 2 CTAs/SM with 128 registers when that many CTAs already cover the rank's groups (knob b200_solve_minb: 2 / 3 force)
        const bool roomy = solve_minb_ == 2 || (solve_minb_ != 3 && (long long) geo_.nseg_local + 1 <= 2ll * sm_count_);
        sb = scalar_bounds_ && !use_pol;
        fn = variant_ == kMMA ? pick_solve_kernel2<0>(maxm, full, use_pol, sb, roomy) : pick_solve_kernel2<1>(maxm, full, use_pol, sb, roomy);
    }
    int per_sm = 0;
    NB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, block, smem));
    if (per_sm < 1) return fail("dual_solve_kernel does not fit on an SM");
    long long grid = (long long) per_sm * sm_count_;          // all co-resident: sweepers + the folder CTA (the last one)
    if (grid > (long long) geo_.nseg_local + 1) grid = (long long) geo_.nseg_local + 1;
    if (grid < 2) return fail("dual_solve_kernel needs two co-resident CTAs");

    // the head of the state (claim counter, done flag) starts from zero every launch
    NB_CUDA(cudaMemsetAsync(solve_state_, 0, offsetof(SolveState, pub), stream_));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (time_kernels_) {
        if (ev_used_ + 2 > ev_pool_.size()) {
            if (ev_pool_.size() >= 8192) drain_events();
            else
                for (int k = 0; k < 512; ++k) { cudaEvent_t e; cudaEventCreate(&e); ev_pool_.push_back(e); }
        }
        e0 = ev_pool_[ev_used_++];
        e1 = ev_pool_[ev_used_++];
        cudaEventRecord(e0, stream_);
    }
    void *params[] = {&sa};
    {
        cudaError_t le = cudaLaunchCooperativeKernel((const void *) fn, dim3((unsigned) grid), dim3((unsigned) block), params, smem, stream_);
        if (le != cudaSuccess) {
            // e.g. co-residency not available (MPS, another context): not fatal -- switch this object to one
            // launch per evaluation; the caller sees supports_dual_solve() == false and takes the host loop
            cudaGetLastError();
            fused_solve_ok_ = false;
            if (ev_used_ >= 2 && time_kernels_) ev_used_ -= 2;
            return fail("cooperative launch of dual_solve_kernel", le);
        }
    }
    if (time_kernels_) cudaEventRecord(e1, stream_);
    ++stats_->kernel_launches;
    cand_in_x_ = false;                              // the final pass stores x*(y) into xcur_
    ++x_epoch_;
    if (!wait_flag()) return false;
#ifdef NB200_TRACE
    if (const char *tf = std::getenv("NLOPT_B200_TRACE_FILE")) {      // one line per generation, ns relative to publication
        static std::vector<unsigned long long> h(16 * kTraceGens);
        cudaStreamSynchronize(stream_);
        cudaMemcpy(h.data(), trace_buf, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
        std::string tfn = tf;
        if (Comm::instance().active()) tfn += ".r" + std::to_string(Comm::instance().rank);      // one file per rank
        if (FILE *f = std::fopen(tfn.c_str(), "a")) {
            const unsigned long long t00 = ~h[1];
            std::fprintf(f, "solve n_local=%llu m=%u grid=%lld groups=%u cta_start_spread_ns=%llu first_publish_ns=%llu\n", (unsigned long long) geo_.n_local, m_, grid,
                         geo_.nseg_local, h[2] - t00, h[16] - t00);
            for (int g = 1; g < kTraceGens && h[16 * g]; ++g) {
                const unsigned long long *r = &h[16 * g];
                const unsigned long long p = r[0];
                // lastrec / parked: TMA-staged form only (0 otherwise)
                std::fprintf(f, "  gen %d lastrec[%lld..%lld] parked[%lld..%lld] seen[%lld..%lld] recs[%lld..%lld] rank_done %lld totals %lld machine %lld next_pub %lld | mean_group_sweep %llu ns x %llu\n", g,
                             r[11] ? (long long) (~r[10] - p) : 0ll, r[11] ? (long long) (r[11] - p) : 0ll,
                             r[12] ? (long long) (~r[13] - p) : 0ll, r[12] ? (long long) (r[12] - p) : 0ll,
                             (long long) (~r[1] - p), (long long) (r[2] - p), (long long) (~r[3] - p), (long long) (r[4] - p),
                             (long long) (r[5] - p), (long long) (r[6] - p), (long long) (r[7] - p),
                             (long long) (h[16 * (g + 1)] ? h[16 * (g + 1)] - p : 0), r[9] ? r[8] / r[9] : 0ull, r[9]);
            }
            std::fclose(f);
        }
    }
#endif
    const long gens = (long) res_host_[kResCounts + 2];
    *ret = (int) res_host_[kResCounts + 1];
    *nevals = (long) res_host_[kResCounts];
    if (Comm::instance().active() && gens > 0) Comm::instance().advance_seq((unsigned long long) gens);
    if (*ret == kRetInvalid) return true;            // nothing ran; the caller reports it
    if (*ret == kRetFailure) return fail("the cross-rank exchange inside the dual solve timed out");
    count_operand_bytes(gens, sb, si, true);         // the last generation stored x*(y)
    out->val = res_host_[0];
    out->gval = res_host_[1];
    out->wval = res_host_[2];
    for (unsigned i = 0; i < m_; ++i) {
        out->gc[i] = res_host_[3 + i];
        y[i] = res_host_[kResY + i];
    }
    return true;
}

void DeviceBackend::drain_events()
{
    if (!ev_used_) return;
    cudaStreamSynchronize(stream_);
    double ms = 0;
    for (size_t i = 0; i + 1 < ev_used_; i += 2) {
        float t = 0;
        if (cudaEventElapsedTime(&t, ev_pool_[i], ev_pool_[i + 1]) == cudaSuccess) ms += t;
    }
    stats_->seconds_dual_kernel += ms * 1e-3;
    ev_used_ = 0;
}

bool DeviceBackend::time_dual(const double *y, const DualScalars &sc, bool materialize, int iters, double *ms_avg)
{
    cudaEvent_t e0, e1;
    NB_CUDA(cudaEventCreate(&e0));
    NB_CUDA(cudaEventCreate(&e1));
    NB_CUDA(cudaEventRecord(e0, stream_));
    for (int it = 0; it < iters; ++it)
        if (!launch_dual(y, sc, materialize, false)) return false;
    NB_CUDA(cudaEventRecord(e1, stream_));
    NB_CUDA(cudaStreamSynchronize(stream_));
    float ms = 0;
    NB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (materialize) cand_in_x_ = false;
    *ms_avg = (double) ms / iters;
    return true;
}

// ------------------------------------------------------------------------------------------------
// acceptance and outer-iteration bookkeeping

void DeviceBackend::accept_candidate()
{
    // mma.c:374-377 copies xcur, dfdx_cur, dfcdx_cur over x, dfdx, dfcdx: here three pointer swaps
    std::swap(x_, xcur_);
    std::swap(g_, gcur_);
    std::swap(G_, Gcur_);
    cand_in_x_ = true;
    if (h_x_slot_ == (int) kCandidate && h_x_epoch_ == x_epoch_) h_x_slot_ = (int) kBase;   // same values, new name
    if (h_xs_slot_ == (int) kCandidate && h_xs_epoch_ == x_epoch_) h_xs_slot_ = (int) kBase;
}

bool DeviceBackend::first_outer()
{
    NB_CUDA(cudaMemcpyAsync(xprev_, xcur_view(), geo_.ld * sizeof(double), cudaMemcpyDeviceToDevice, stream_));
    return true;
}

bool DeviceBackend::end_outer(unsigned k, double sigma_min, double *dnorm, double *xnorm, bool *all_below_abs)
{
    EndOuterArgs a;
    std::memset(&a, 0, sizeof a);
    a.xcur = xcur_view();
    a.xprev = xprev_; a.xprevprev = xprevprev_; a.sigma = sigma_;
    a.lb = lb_; a.ub = ub_;
    a.update_sigma = k > 1;
    a.kappa = variant_ == kMMA ? 0.01 : 1e-8;
    a.sigma_min = sigma_min;
    if (a.update_sigma && sidx_valid_) {
        // the palette one update further: the same on every rank, as nothing in it depends on the data
        sidx_valid_ = sigma_min == sidx_sigma_min_ && palette_.step();
        if (sidx_valid_ && !upload_palette()) return false;
        if (sidx_valid_) { a.sidx = sidx_; a.next = next_; a.pal = pal_; }
    }
    if (!end_outer_pass(a, dnorm, xnorm, all_below_abs)) return false;
    if (out_host_[3] != 0.0) {             // a palette value differs from the fp64 sigma: stay on the fp64 path
        stats_->sigma_index_mismatches += (long long) out_host_[3];
        sidx_valid_ = false;
    }
    stats_->sigma_palette = sidx_valid_ ? (long long) palette_.val.size() : 0;
    return true;
}

// end_outer_kernel over this rank's groups with the caller's arrays and sigma fields; the three stop sums come back
bool DeviceBackend::end_outer_pass(EndOuterArgs &a, double *dnorm, double *xnorm, bool *all_below_abs)
{
    a.w = w_dev_; a.xtol_abs = xtol_abs_dev_;
    a.n_local = geo_.n_local; a.nchunks = geo_.nchunks; a.chunk0 = geo_.chunk0;
    a.nseg_total = geo_.S; a.seg0 = geo_.seg0; a.segs_per_vshard = geo_.P; a.local_vshards = geo_.local_vshards;
    a.partials = partials_; a.vsums = vsums_; a.tickets = tickets_; a.out_dev = out_dev_;
    a.out_host = out_host_; a.flag_host = flag_host_;
    a.seq = seq_ = Comm::instance().active() ? Comm::instance().next_seq() : seq_ + 1;
    a.publish_host = Comm::instance().active() ? 0 : 1;
    a.nvp = kEndNvp;               // records of this kernel: 4 sums (its own stride: nvp_ belongs to the dual kernels)
    end_outer_kernel<<<(int) geo_.nseg_local, kBlock, 0, stream_>>>(a);
    ++stats_->kernel_launches;
    NB_CUDA(cudaGetLastError());
    if (!a.publish_host) {
        if (Comm::instance().all_gather_inplace(out_dev_, (size_t) geo_.local_vshards * kEndNvp, stream_, &err_)) return false;
        publish_kernel<<<1, 32, 0, stream_>>>(out_dev_, 4, kEndNvp, out_host_, flag_host_, a.seq);
        ++stats_->kernel_launches;
        NB_CUDA(cudaGetLastError());
    }
    if (!wait_flag()) return false;
    *dnorm = out_host_[0];
    *xnorm = out_host_[1];
    *all_below_abs = out_host_[2] == 0.0;
    return true;
}

// The AUGLAG outer loop's acceptance (auglag.c:270-285): the sums of nlopt_stop_x between x and the best point, then
// best <- x, in one read of both arrays (the end-of-iteration kernel without its sigma update and rotation)
bool DeviceBackend::stop_x_keep(double *dnorm, double *xnorm, bool *all_below_abs)
{
    EndOuterArgs a;
    std::memset(&a, 0, sizeof a);
    a.xcur = x_;
    a.xprev = xprev_;
    return end_outer_pass(a, dnorm, xnorm, all_below_abs);
}

int DeviceBackend::ranks() const { return Comm::instance().active() ? Comm::instance().world : 1; }

bool DeviceBackend::fetch_x(double *x_out)
{
    drain_events();
    if (cfg_.values_only) {
        NB_CUDA(cudaMemcpyAsync(x_out, xprev_, geo_.n_local * sizeof(double), cfg_.x_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        if (!cfg_.x_dev) stats_->d2h_bytes += geo_.n_local * sizeof(double);
        return true;
    }
    if (cfg_.x_dev && x_out == cfg_.x_dev) {
        NB_CUDA(cudaMemcpyAsync(x_out, x_, geo_.n_local * sizeof(double), cudaMemcpyDeviceToDevice, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        return true;
    }
    Comm &comm = Comm::instance();
    if (!comm.active()) {
        NB_CUDA(cudaMemcpyAsync(x_out, x_, geo_.n_local * sizeof(double), cudaMemcpyDeviceToHost, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        stats_->d2h_bytes += geo_.n_local * sizeof(double);
        return true;
    }
    if (!h_x_) NB_CUDA(cached_host_alloc(&h_x_, (size_t) geo_.n * sizeof(double)));
    if (!xfull_dev_) NB_CUDA(cached_malloc(&xfull_dev_, (size_t) comm.world * shard_cap_ * sizeof(double)));
    h_x_slot_ = -1;
    if (!host_x_for(kBase)) return false;
    std::memcpy(x_out, h_x_view_, (size_t) geo_.n * sizeof(double));
    return true;
}

// ------------------------------------------------------------------------------------------------
// kernel-level access

double *DeviceBackend::array(const char *which)
{
    const std::string w = which;
    if (w == "x") return x_;
    if (w == "xcur") return xcur_view();
    if (w == "xprev") return xprev_;
    if (w == "xprevprev") return xprevprev_;
    if (w == "lb") return lb_;
    if (w == "ub") return ub_;
    if (w == "sigma") return sigma_;
    if (w == "grad_f") return g_;
    if (w == "grad_f_cur") return gcur_;
    return nullptr;
}

bool DeviceBackend::upload(const char *which, const double *host)
{
    double *dst = array(which);
    if (std::string(which) == "xcur") { dst = xcur_; cand_in_x_ = false; }
    if (!dst) return fail(std::string("unknown array ") + which);
    if (dst == sigma_) sidx_valid_ = false;
    NB_CUDA(cudaMemcpyAsync(dst, host + geo_.j0, geo_.n_local * sizeof(double), cudaMemcpyHostToDevice, stream_));
    NB_CUDA(cudaStreamSynchronize(stream_));
    return true;
}

bool DeviceBackend::upload_grad_c(const double *host)
{
    if (!m_) return true;
    NB_CUDA(cudaMemcpy2DAsync(G_, geo_.ld * sizeof(double), host + geo_.j0, (size_t) geo_.n * sizeof(double),
                              geo_.n_local * sizeof(double), m_, cudaMemcpyHostToDevice, stream_));
    NB_CUDA(cudaStreamSynchronize(stream_));
    return true;
}

bool DeviceBackend::download(const char *which, double *host)
{
    const std::string w = which;
    if (w == "grad_c") {
        if (!m_) return true;
        NB_CUDA(cudaMemcpy2DAsync(host + geo_.j0, (size_t) geo_.n * sizeof(double), G_, geo_.ld * sizeof(double),
                                  geo_.n_local * sizeof(double), m_, cudaMemcpyDeviceToHost, stream_));
        NB_CUDA(cudaStreamSynchronize(stream_));
        return true;
    }
    double *src = array(which);
    if (!src) return fail(std::string("unknown array ") + which);
    NB_CUDA(cudaMemcpyAsync(host + geo_.j0, src, geo_.n_local * sizeof(double), cudaMemcpyDeviceToHost, stream_));
    NB_CUDA(cudaStreamSynchronize(stream_));
    return true;
}

bool DeviceBackend::fill_synthetic(unsigned long long seed)
{
    SynthArgs a;
    a.x = x_; a.lb = lb_; a.ub = ub_; a.sigma = sigma_; a.g = g_; a.G = G_;
    a.ld = geo_.ld; a.n_local = geo_.n_local; a.j0 = geo_.j0; a.seed = seed; a.m = (int) m_;
    synth_fill_kernel<<<grid_for(geo_.n_local, sm_count_), kBlock, 0, stream_>>>(a);
    NB_CUDA(cudaGetLastError());
    NB_CUDA(cudaStreamSynchronize(stream_));
    cand_in_x_ = true;
    return true;
}

bool DeviceBackend::configure(const char *key, long long value)
{
    const std::string k = key;
    if (k == "time_kernels") { time_kernels_ = value != 0; return true; }
    if (k == "kernel_cfg") { kernel_cfg_ = (int) value; return true; }
    if (k == "ctas_per_sm") { ctas_per_sm_ = (int) value; return true; }
    if (k == "fused_solve") { fused_solve_ok_ = value != 0; return true; }
    if (k == "solve_tma") { solve_tma_ = (int) value; return true; }
    if (k == "solve_async") { solve_async_ = (int) value; return true; }
    if (k == "solve_minb") { solve_minb_ = (int) value; return true; }
    if (k == "l2_keep_mb") {
        l2_keep_bytes_ = value <= 0 ? 0 : (size_t) value << 20;
        // evict_last lines are only protected inside the persisting carve-out of the L2: size it to the request
        int maxp = 0;
        if (cudaDeviceGetAttribute(&maxp, cudaDevAttrMaxPersistingL2CacheSize, device_) == cudaSuccess && maxp > 0) {
            size_t want = l2_keep_bytes_ < (size_t) maxp ? l2_keep_bytes_ : (size_t) maxp;
            cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want);
            cudaGetLastError();
        }
        return true;
    }
    if (k == "pmax" || k == "target_chunks" || k == "fill_div" || k == "group_base" || k == "geometry_rule" || k == "group_min_chunks") {
        if (value < 1 && k != "geometry_rule") return fail("bad value");
        if (k == "pmax") pmax_ = (unsigned) value;
        else if (k == "target_chunks") target_chunks_ = (unsigned) value;
        else if (k == "group_base") Geometry::group_base() = (unsigned) value;
        else if (k == "group_min_chunks") Geometry::min_group_chunks() = (unsigned) value;
        else if (k == "geometry_rule") Geometry::rule() = (int) value;
        else Geometry::fill_div() = (unsigned) value;
        if (pool_) {
            Geometry g2 = Geometry::make(geo_.n, geo_.world, geo_.rank, target_chunks_, pmax_);
            if (g2.ld != geo_.ld || g2.j0 != geo_.j0)
                return fail("changing the segment geometry of a sharded, allocated problem is not supported");
            geo_ = g2;
            return alloc_workspace();
        }
        return true;
    }
    return fail(std::string("unknown key ") + key);
}

long long DeviceBackend::query(const char *key) const
{
    const std::string k = key;
    if (k == "kernel_ns") {            // accumulated device time of timed dual launches, nanoseconds
        const_cast<DeviceBackend *>(this)->drain_events();
        return (long long) (stats_->seconds_dual_kernel * 1e9);
    }
    if (k == "segments") return geo_.S;
    if (k == "segments_local") return geo_.nseg_local;
    if (k == "P") return geo_.P;
    if (k == "n_local") return (long long) geo_.n_local;
    if (k == "j0") return (long long) geo_.j0;
    if (k == "ld") return (long long) geo_.ld;
    if (k == "launches") return stats_->kernel_launches;
    if (k == "maxm") return pick_maxm((int) m_);
    if (k == "l2_keep_mask") return (long long) l2_keep_mask();
    return -1;
}

void release_cached_blocks() { BlockCache::get().clear(); }

// ------------------------------------------------------------------------------------------------
// bounds of an object in device mode.  The work goes to the per-thread default stream and is complete on return, so a
// caller may reuse its buffers at once (NLopt's copy semantics).

namespace {

bool cuda_ok(cudaError_t e, const char *what, std::string *err)
{
    if (e == cudaSuccess) return true;
    *err = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
}

// makes `device` current for the lifetime of the guard
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int device)
    {
        if (cudaGetDevice(&prev) != cudaSuccess || prev == device || cudaSetDevice(device) != cudaSuccess) prev = -1;
    }
    ~DeviceGuard()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

class DeviceBoundsImpl : public DeviceBounds {
public:
    explicit DeviceBoundsImpl(unsigned n) : n_(n) {}
    ~DeviceBoundsImpl() override
    {
        if (p_) {
            DeviceGuard g(device_);
            cudaFree(p_);
        }
    }
    const double *lb() const override { return p_; }
    const double *ub() const override { return p_ + n_; }

    // both arrays on the current device
    bool alloc(std::string *err)
    {
        int ndev = 0;
        const cudaError_t e = cudaGetDeviceCount(&ndev);
        if (e != cudaSuccess || ndev == 0) {
            *err = no_device_message(e);
            return false;
        }
        return cuda_ok(cudaGetDevice(&device_), "cudaGetDevice", err) &&
               cuda_ok(cudaMalloc(&p_, 2 * bytes()), "cudaMalloc", err);
    }
    // lb / ub <- lb_src / ub_src (any memory CUDA can read; null: keep)
    bool upload(const double *lb_src, const double *ub_src, std::string *err)
    {
        return (!lb_src || cuda_ok(cudaMemcpyAsync(p_, lb_src, bytes(), cudaMemcpyDefault, cudaStreamPerThread), "cudaMemcpyAsync", err)) &&
               (!ub_src || cuda_ok(cudaMemcpyAsync(p_ + n_, ub_src, bytes(), cudaMemcpyDefault, cudaStreamPerThread), "cudaMemcpyAsync", err)) &&
               cuda_ok(cudaStreamSynchronize(cudaStreamPerThread), "cudaStreamSynchronize", err);
    }
    // the caller's n doubles into the lower (or upper) array, then the setters' snap against the other one
    bool set(bool lower, const double *src, std::string *err)
    {
        DeviceGuard g(device_);
        double *dst = lower ? p_ : p_ + n_;
        int sms = 0;
        if (!cuda_ok(cudaMemcpyAsync(dst, src, bytes(), cudaMemcpyDefault, cudaStreamPerThread), "cudaMemcpyAsync", err) ||
            !cuda_ok(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device_), "cudaDeviceGetAttribute", err))
            return false;
        snap_bounds_kernel<<<grid_for(n_, sms), kBlock, 0, cudaStreamPerThread>>>(dst, lower ? p_ + n_ : p_, lower, n_);
        return cuda_ok(cudaGetLastError(), "snap_bounds_kernel", err) &&
               cuda_ok(cudaStreamSynchronize(cudaStreamPerThread), "cudaStreamSynchronize", err);
    }
    bool download(double *lb_host, double *ub_host, std::string *err) const override
    {
        return cuda_ok(cudaMemcpyAsync(lb_host, p_, bytes(), cudaMemcpyDefault, cudaStreamPerThread), "cudaMemcpyAsync", err) &&
               cuda_ok(cudaMemcpyAsync(ub_host, p_ + n_, bytes(), cudaMemcpyDefault, cudaStreamPerThread), "cudaMemcpyAsync", err) &&
               cuda_ok(cudaStreamSynchronize(cudaStreamPerThread), "cudaStreamSynchronize", err);
    }
    bool copy_into(DeviceBounds **dst, std::string *err) const override
    {
        DeviceGuard g(device_);
        if (!*dst) {
            DeviceBoundsImpl *d = new DeviceBoundsImpl(n_);
            if (!d->alloc(err)) {
                delete d;
                return false;
            }
            *dst = d;
        }
        DeviceBoundsImpl *d = static_cast<DeviceBoundsImpl *>(*dst);
        return cuda_ok(cudaMemcpyAsync(d->p_, p_, 2 * bytes(), cudaMemcpyDefault, cudaStreamPerThread), "cudaMemcpyAsync", err) &&
               cuda_ok(cudaStreamSynchronize(cudaStreamPerThread), "cudaStreamSynchronize", err);
    }
    bool runs_here(std::string *err) const override
    {
        if (Comm::instance().active()) {
            *err = "device bounds (nlopt_b200_set_*_bounds_device) run on one rank in this library";
            return false;
        }
        int d = -1;
        cudaGetDevice(&d);
        if (d != device_) {
            *err = "the device bounds live on CUDA device " + std::to_string(device_) + " but device " + std::to_string(d) +
                   " is current";
            return false;
        }
        return true;
    }
    bool check(const double *x_host, const double *x_dev, StartCheck *out, std::string *err) const override
    {
        DeviceGuard g(device_);
        const cudaStream_t s = cudaStreamPerThread;
        BoundsReport *rep_dev = nullptr, *rep_host = nullptr;
        double *x_stage = nullptr;
        int sms = 0;
        bool good = cuda_ok(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device_), "cudaDeviceGetAttribute", err) &&
                    cuda_ok(cached_malloc((double **) &rep_dev, sizeof(BoundsReport)), "cudaMalloc", err) &&
                    cuda_ok(cached_host_alloc((double **) &rep_host, sizeof(BoundsReport)), "cudaHostAlloc", err);
        if (good && x_host) {
            good = cuda_ok(cached_malloc(&x_stage, bytes()), "cudaMalloc", err) &&
                   cuda_ok(cudaMemcpyAsync(x_stage, x_host, bytes(), cudaMemcpyHostToDevice, s), "cudaMemcpyAsync", err);
            x_dev = x_stage;
        }
        good = good && cuda_ok(enqueue_bounds_check(lb(), ub(), x_dev, n_, rep_dev, rep_host, sms, s), "bounds_check_kernel", err) &&
               cuda_ok(cudaStreamSynchronize(s), "cudaStreamSynchronize", err);
        if (good) read_bounds_report(*rep_host, out);
        cudaStreamSynchronize(s);
        if (x_stage) BlockCache::get().give(false, bytes(), x_stage, device_);
        if (rep_dev) BlockCache::get().give(false, sizeof(BoundsReport), rep_dev, device_);
        if (rep_host) BlockCache::get().give(true, sizeof(BoundsReport), rep_host);
        return good;
    }

private:
    size_t bytes() const { return (size_t) n_ * sizeof(double); }
    unsigned n_;
    int device_ = -1;
    double *p_ = nullptr;            // lb | ub
};

}  // namespace

Backend *make_backend(const BackendConfig &cfg, std::string *err)
{
    DeviceBackend *be = new DeviceBackend();
    if (!be->setup(cfg)) {
        if (err) *err = be->error();
        delete be;
        return nullptr;
    }
    return be;
}

}  // namespace nb200

// ================================================================================================
// C ABI: kernel-level access (include/nlopt_b200.h).  A handle is a DeviceBackend without user
// callbacks; the functions below are what the reference's static dual_func (mma.c:59,
// ccsa_quadratic.c:79) and the O(n) loops around it (mma.c:202-210, :264-265, :418-442) would
// bind to.
// ================================================================================================

struct nlopt_b200_dual_s {
    nb200::DeviceBackend be;
    std::vector<double> c0, rhoc, gc;
    double f0 = 0, rho = 1;
    std::string err;
};

namespace {
int ok(nlopt_b200_dual h, bool good)
{
    if (!good) h->err = h->be.error();
    return good ? 0 : -1;
}
}  // namespace

extern "C" {

nlopt_b200_dual nlopt_b200_dual_create(int variant, unsigned n, unsigned m)
{
    nlopt_b200_dual h = new nlopt_b200_dual_s;
    h->c0.assign(m, 0.0);
    h->rhoc.assign(m, 1.0);
    h->gc.assign(m > 0 ? m : 1, 0.0);
    if (!h->be.setup_raw(variant == NLOPT_B200_MMA ? nb200::kMMA : nb200::kCCSAQ, n, m)) {
        std::fprintf(stderr, "nlopt_b200_dual_create: %s\n", h->be.error().c_str());
        delete h;
        return nullptr;
    }
    return h;
}

void nlopt_b200_dual_destroy(nlopt_b200_dual h) { delete h; }

const char *nlopt_b200_dual_errmsg(nlopt_b200_dual h) { return h ? h->err.c_str() : "null handle"; }

int nlopt_b200_dual_upload(nlopt_b200_dual h, const double *x, const double *lb, const double *ub,
                           const double *sigma, const double *grad_f, const double *grad_c)
{
    bool good = true;
    if (x) good = good && h->be.upload("x", x);
    if (lb) good = good && h->be.upload("lb", lb);
    if (ub) good = good && h->be.upload("ub", ub);
    if (sigma) good = good && h->be.upload("sigma", sigma);
    if (grad_f) good = good && h->be.upload("grad_f", grad_f);
    if (grad_c) good = good && h->be.upload_grad_c(grad_c);
    return ok(h, good);
}

int nlopt_b200_dual_fill_synthetic(nlopt_b200_dual h, unsigned long long seed) { return ok(h, h->be.fill_synthetic(seed)); }

int nlopt_b200_dual_set_scalars(nlopt_b200_dual h, double f0, double rho, const double *c0, const double *rhoc)
{
    h->f0 = f0;
    h->rho = rho;
    for (size_t i = 0; i < h->c0.size(); ++i) {
        h->c0[i] = c0[i];
        h->rhoc[i] = rhoc[i];
    }
    return 0;
}

int nlopt_b200_dual_eval(nlopt_b200_dual h, const double *y, int want_xcur, double *out, double *grad)
{
    nb200::DualScalars sc;
    sc.fval = h->f0;
    sc.rho = h->rho;
    sc.fcval = h->c0.data();
    sc.rhoc = h->rhoc.data();
    nb200::DualSums s;
    s.gc = h->gc.data();
    if (!h->be.dual_eval(y, sc, want_xcur != 0, &s)) return ok(h, false);
    // add the O(m) constants exactly as the driver does (mma.c:75-78)
    const unsigned m = h->be.m();
    double val = h->f0;
    for (unsigned i = 0; i < m; ++i) {
        const double ci = (h->be.is_mma() && std::isnan(h->c0[i])) ? 0.0 : h->c0[i];
        val += y[i] * ci;
        out[3 + i] = ci + s.gc[i];
        if (grad) grad[i] = -out[3 + i];
    }
    val += s.val;
    out[0] = -val;
    out[1] = h->f0 + s.gval;
    out[2] = s.wval;
    return 0;
}

int nlopt_b200_dual_solve(nlopt_b200_dual h, double *y, const double *lo, const double *hi, double ftol_rel, int maxeval,
                          double *out, int *result, long *nevals, double *kernel_ms)
{
    nb200::DualScalars sc;
    sc.fval = h->f0;
    sc.rho = h->rho;
    sc.fcval = h->c0.data();
    sc.rhoc = h->rhoc.data();
    nb200::DualSums s;
    s.gc = h->gc.data();
    const unsigned m = h->be.m();
    h->be.configure("time_kernels", 1);
    const long long ns0 = h->be.query("kernel_ns");
    auto add_constants = [&](const double *yy, double *grad) {      // mma.c:75-78, :135
        double val = h->f0;
        for (unsigned i = 0; i < m; ++i) {
            const double ci = (h->be.is_mma() && std::isnan(h->c0[i])) ? 0.0 : h->c0[i];
            val += yy[i] * ci;
            if (out) out[3 + i] = ci + s.gc[i];
            if (grad) grad[i] = -(ci + s.gc[i]);
        }
        val += s.val;
        if (out) { out[0] = -val; out[1] = h->f0 + s.gval; out[2] = s.wval; }
        return -val;
    };
    if (m >= 1 && h->be.supports_dual_solve()) {
        const double stop6[6] = {ftol_rel, 0.0, 0.0, 0.0, (double) maxeval, 0.0};
        if (!h->be.dual_solve(y, lo, hi, stop6, sc, &s, result, nevals)) return ok(h, false);
        ++*nevals;
        add_constants(y, nullptr);
    } else {
        nb200::DualMMA dual(m);
        nb200::DualStop ds;
        ds.ftol_rel = ftol_rel; ds.ftol_abs = 0; ds.xtol_rel = 0; ds.xtol_abs = 0; ds.maxeval = maxeval; ds.maxtime = 0;
        double dmin = 0;
        bool good = true;
        *result = m ? dual.solve([&](const double *yy, double *grad, bool *okp) {
            if (!h->be.dual_eval(yy, sc, false, &s)) { *okp = false; good = false; return 0.0; }
            return add_constants(yy, grad);
        }, y, lo, hi, ds, &dmin, nevals) : 1;
        if (!good) return ok(h, false);
        if (!h->be.dual_eval(y, sc, true, &s)) return ok(h, false);
        ++*nevals;
        add_constants(y, nullptr);
    }
    if (kernel_ms) *kernel_ms = (double) (h->be.query("kernel_ns") - ns0) * 1e-6;
    return 0;
}

int nlopt_b200_dual_download_xcur(nlopt_b200_dual h, double *xcur_host) { return ok(h, h->be.download("xcur", xcur_host)); }

int nlopt_b200_dual_download(nlopt_b200_dual h, const char *which, double *host) { return ok(h, h->be.download(which, host)); }

int nlopt_b200_dual_sigma_init(nlopt_b200_dual h, const double *sigma_init_host, double sigma_min)
{
    return ok(h, h->be.sigma_init_from(sigma_init_host, sigma_min));
}

int nlopt_b200_dual_set_prev(nlopt_b200_dual h, const double *xcur, const double *xprev, const double *xprevprev)
{
    bool good = true;
    if (xcur) good = good && h->be.upload("xcur", xcur);
    if (xprev) good = good && h->be.upload("xprev", xprev);
    if (xprevprev) good = good && h->be.upload("xprevprev", xprevprev);
    return ok(h, good);
}

int nlopt_b200_dual_end_outer(nlopt_b200_dual h, int k, double sigma_min, const double *x_weights_host,
                              const double *xtol_abs_host, double *norms, int *all_below_xtol_abs)
{
    if (!h->be.set_norm_arrays(x_weights_host, xtol_abs_host)) return ok(h, false);
    bool below = false;
    if (!h->be.end_outer((unsigned) k, sigma_min, &norms[0], &norms[1], &below)) return ok(h, false);
    *all_below_xtol_abs = below ? 1 : 0;
    return 0;
}

int nlopt_b200_dual_time(nlopt_b200_dual h, const double *y, int want_xcur, int iters, double *ms_avg)
{
    nb200::DualScalars sc;
    sc.fval = h->f0;
    sc.rho = h->rho;
    sc.fcval = h->c0.data();
    sc.rhoc = h->rhoc.data();
    return ok(h, h->be.time_dual(y, sc, want_xcur != 0, iters, ms_avg));
}

int nlopt_b200_dual_configure(nlopt_b200_dual h, const char *key, long long value) { return ok(h, h->be.configure(key, value)); }

long long nlopt_b200_dual_query(nlopt_b200_dual h, const char *key) { return h->be.query(key); }

void nlopt_b200_shard_geometry(unsigned long long n, int rank, int world, nlopt_b200_shard *out)
{
    nb200::Geometry g = nb200::Geometry::make(n, world, rank, nb200::kDefaultTargetChunks, nb200::kDefaultPmax);
    out->n = n; out->n_local = g.n_local; out->j0 = g.j0;
    out->nchunks = g.nchunks; out->chunk0 = g.chunk0;
    out->groups_total = g.S; out->group0 = g.seg0; out->groups_local = g.nseg_local; out->groups_per_vshard = g.P;
    out->vshard0 = g.seg0 / g.P; out->local_vshards = g.local_vshards;
    out->rank = rank; out->world = world;
}

void nlopt_b200_shard_range(unsigned long long n, int rank, int world, unsigned long long *j0, unsigned long long *count)
{
    nb200::Geometry g = nb200::Geometry::make(n, world, rank, nb200::kDefaultTargetChunks, nb200::kDefaultPmax);
    *j0 = g.j0;
    *count = g.n_local;
}

int nlopt_b200_device_count(void)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) return 0;
    return e == cudaSuccess ? n : -1;
}

void nlopt_b200_release_cached_memory(void) { nb200::release_cached_blocks(); }

/* device bounds (the rest of the bounds API is in nlopt_api.cpp).  An object whose first device setter fails keeps its
   host bounds. */
static nlopt_result set_bounds_device(nlopt_opt opt, const double *src, bool lower)
{
    if (!opt) return NLOPT_INVALID_ARGS;
    opt->errmsg.clear();
    opt->has_errmsg = false;
    if (!src) return NLOPT_INVALID_ARGS;
    if (opt->n == 0) return NLOPT_SUCCESS;
    auto refuse = [opt](nlopt_result r, const std::string &msg) {
        opt->errmsg = msg;
        opt->has_errmsg = true;
        return r;
    };
    if (nb200::Comm::instance().active())
        return refuse(NLOPT_INVALID_ARGS, "device bounds (nlopt_b200_set_*_bounds_device) run on one rank in this library");
    std::string err;
    std::unique_ptr<nb200::DeviceBoundsImpl> fresh;
    nb200::DeviceBoundsImpl *b = static_cast<nb200::DeviceBoundsImpl *>(opt->dbounds);
    if (!b) {                                /* entering device mode: the other array goes up once */
        fresh.reset(new nb200::DeviceBoundsImpl(opt->n));
        if (!fresh->alloc(&err) || !fresh->upload(lower ? nullptr : opt->lb.data(), lower ? opt->ub.data() : nullptr, &err))
            return refuse(NLOPT_FAILURE, err);
        b = fresh.get();
    }
    if (!b->set(lower, src, &err)) return refuse(NLOPT_FAILURE, err);
    if (fresh) opt->dbounds = fresh.release();
    opt->lb_ub_mirror = false;
    (lower ? opt->lb_uniform : opt->ub_uniform) = false;
    return NLOPT_SUCCESS;
}

nlopt_result nlopt_b200_set_lower_bounds_device(nlopt_opt opt, const double *lb_dev) { return set_bounds_device(opt, lb_dev, true); }
nlopt_result nlopt_b200_set_upper_bounds_device(nlopt_opt opt, const double *ub_dev) { return set_bounds_device(opt, ub_dev, false); }

const char *nlopt_b200_build_info(void)
{
    return "nlopt_b200: NLOPT_LD_MMA / NLOPT_LD_CCSAQ on CUDA sm_90a, fp64, exact-rounding (no FMA contraction); "
           "built " __DATE__;
}

}  // extern "C"
