// device_backend.hpp -- HBM-resident state + kernel launches of the MMA/CCSAQ path.
#pragma once

#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "backend_factory.hpp"
#include "geometry.hpp"
#include "sigma_palette.hpp"

#ifndef NB200_SIGMA_INDEX_MIN_MB
#define NB200_SIGMA_INDEX_MIN_MB 50   // fp64 operand set above which the sigma-index form runs: the L2 (DESIGN.md section 3.2)
#endif

namespace nb200 {

// Data layout in HBM (per rank): one cudaMalloc carved into (9 + 2m) arrays of `ld` doubles,
//   x xcur xprev xprevprev lb ub sigma grad_f grad_f_cur | grad_c[m][ld] | grad_c_cur[m][ld]
// ld = shard length rounded up to 32 doubles, so every array and every row is 256-byte aligned.
// Padding lanes carry sigma = 0, which both dual formulas skip (mma.c:96-99).
// A values-only backend (BackendConfig::values_only) allocates x (with its guard cells) and xprev (the best point) only.
class DeviceBackend : public Backend {
public:
    DeviceBackend();
    ~DeviceBackend() override;

    bool setup(const BackendConfig &cfg);           // allocate + upload bounds/start point
    bool setup_raw(Variant v, unsigned n, unsigned m);   // kernel-level handle: arrays only

    // ---- Backend ----
    unsigned n() const override { return (unsigned) geo_.n; }
    unsigned m() const override { return m_; }
    unsigned num_constraint_objects() const override { return (unsigned) cfg_.constraints.size(); }
    unsigned constraint_dim(unsigned ic) const override { return cfg_.constraints[ic].m; }
    bool init_sigma(double sigma_min) override;
    bool eval_objective(Slot slot, bool want_grad, double *value) override;
    bool eval_constraint(Slot slot, unsigned ic, unsigned row0, bool want_grad, double *values) override;
    bool finish_evals(double *fvalue, double *cvalues) override;
    bool agree_any(bool local) override;
    bool enqueue_df2(const FuncSpec &fs, Slot slot, double *grad_dst, unsigned index);
    bool reduce_terms(const FuncSpec &fs, const double *xs, double *grad_dst, double *vsums);
    bool ensure_halo(Slot slot);
    bool eval_sharded(const FuncSpec &fs, Slot slot, double *grad_dst, unsigned index, double *value);
    bool eval_user_objective(Slot slot, bool want_grad, double *value);
    bool negate_gradient(double *g);
    bool push_rows_to(double *dst, unsigned rows, const double *host_grad);
    bool eval_penalty_objective(Slot slot, bool want_grad, double *value);
    bool dual_eval(const double *y, const DualScalars &sc, bool materialize, DualSums *out) override;
    bool supports_dual_solve() const override;
    bool dual_solve(double *y, const double *lo, const double *hi, const double *stop6, const DualScalars &sc, DualSums *out,
                    int *ret, long *nevals) override;
    void accept_candidate() override;
    bool first_outer() override;
    bool end_outer(unsigned k, double sigma_min, double *dnorm, double *xnorm, bool *all_below_abs) override;
    bool fetch_x(double *x_out) override;
    double *point_device() override { return cfg_.values_only ? x_ : nullptr; }
    void point_moved() override { ++x_epoch_; }
    bool stop_x_keep(double *dnorm, double *xnorm, bool *all_below_abs) override;
    int ranks() const override;
    const std::string &error() const override { return err_; }
    double seconds_in_callbacks() const override { return cb_seconds_; }

    // ---- kernel-level access (nlopt_b200_dual_* C ABI) ----
    bool upload(const char *which, const double *host);          // which: x lb ub sigma grad_f xcur xprev xprevprev
    bool upload_grad_c(const double *host_rowmajor_m_by_n);
    bool download(const char *which, double *host);
    bool fill_synthetic(unsigned long long seed);
    bool sigma_init_from(const double *sigma_init_host, double sigma_min);
    bool set_norm_arrays(const double *x_weights_host, const double *xtol_abs_host);
    bool time_dual(const double *y, const DualScalars &sc, bool materialize, int iters, double *ms_avg);
    bool configure(const char *key, long long value) override;
    long long query(const char *key) const;
    const Geometry &geometry() const { return geo_; }
    bool is_mma() const { return variant_ == kMMA; }

private:
    bool fail(const char *what, cudaError_t e);
    bool fail(const std::string &what);
    bool alloc_state();
    void free_state();
    bool alloc_workspace();
    double *array(const char *which);
    double *xcur_view() { return cand_in_x_ ? x_ : xcur_; }
    void fill_dual_args(struct DualArgs &a, const double *y, const DualScalars &sc);
    bool launch_dual(const double *y, const DualScalars &sc, bool store, bool wait);
    bool end_outer_pass(struct EndOuterArgs &a, double *dnorm, double *xnorm, bool *all_below_abs);
    unsigned l2_keep_mask() const;
    void count_operand_bytes(long long evals, bool sb, bool si, bool store);     // nlopt_b200_stats::dual_operand_bytes
    bool upload_palette();
    bool sigma_index_runs() const;
    bool wait_flag();
    bool host_x_for(Slot slot);                      // bring the slot's x to pinned host memory (cached per epoch)
    bool push_grad_rows(Slot slot, int row0, unsigned rows, bool is_objective, const double *host_grad);
    double *staging(unsigned rows);
    struct Owned { void *p; size_t bytes; bool pinned; };
    std::vector<Owned> owned_;                       // small buffers borrowed from the block cache
    bool small_dev(void **p, size_t bytes);
    bool small_pinned(void **p, size_t bytes);
    void release_small(void *p);

    BackendConfig cfg_;
    Variant variant_ = kMMA;
    unsigned m_ = 0;
    Geometry geo_;
    unsigned target_chunks_ = kDefaultTargetChunks, pmax_ = kDefaultPmax;
    int device_ = 0;
    int sm_count_ = 132, ctas_per_sm_ = 0;
    void *solve_state_ = nullptr;     // SolveState (device) of the persistent dual-solve kernel
    double *res_host_ = nullptr;      // its mapped pinned result record
    double *grouptags_ = nullptr;     // tagged group-record slots {value, tag} of the dual kernels, [nvp][local groups]
    unsigned long long eval_tag_ = 0;  // tags of the one-evaluation kernels: 1 << 63 | counter
    double *wide_dev_ = nullptr;      // m > 16: y | rhoc | rhoc/2 | active flags of the evaluation in flight
    std::vector<double> wide_host_;
    size_t l2_keep_bytes_ = 0;        // operand bytes to load evict_last (knob b200_l2_keep_mb)
    int solve_tma_ = -1;              // knob b200_solve_tma: -1 by rows, bounds and size (DeviceBackend::dual_solve), 0 register form, 1 TMA-staged form
    int solve_async_ = 0;             // knob b200_solve_async: 0 register form, 2 / 3: per-thread cp.async operand ring of 2 / 3 stages
    int solve_minb_ = 0;              // knob b200_solve_minb: 0 by size, 2 / 3: force the 2- / 3-CTAs-per-SM instantiation of the solve kernel
    size_t out_rec_ = 0;              // doubles per result record (>= 24, >= 3 + m)
    unsigned long long solve_launch_id_ = 0;   // tag = launch id << 40 | generation: never matches a stale slot
    bool fused_solve_ok_ = true;
    // every lb entry is lb_u_ and every ub entry ub_u_ (both set with nlopt_set_*_bounds1): the default dual kernels take
    // the bounds as two scalars instead of reading the lb / ub arrays, which stay filled for the other kernels
    bool scalar_bounds_ = false;
    double lb_u_ = 0.0, ub_u_ = 0.0;
    // sigma index: sidx_[j] indexes palette_ (sigma_palette.hpp) and sigma_[j] == palette value, bit for bit, while
    // sidx_valid_.  Valid from sigma_init_from() with scalar bounds and a uniform initial step; lost for the rest of the
    // run when sigma is uploaded, the palette would pass its cap, or end_outer_kernel finds a mismatch.  sigma_ stays
    // the source of truth for every kernel that does not read the index.
    bool sidx_valid_ = false;
    unsigned short *sidx_ = nullptr, *next_ = nullptr;      // device: [ld] indices (padding lanes 0), [cap][3] transitions
    double *pal_ = nullptr;                                 // device: [cap] values
    double *pal_pinned_ = nullptr;                          // pinned staging of pal_ / next_
    unsigned short *next_pinned_ = nullptr;
    SigmaPalette palette_;
    size_t pal_uploaded_ = 0, rows_uploaded_ = 0;           // palette entries / transition rows already on the device
    double sidx_sigma_min_ = 0.0;
    int kernel_cfg_ = -1;        // -1: measured default for (variant, m)          // index into the launch-geometry table of device_backend.cu

    // device state
    double *pool_ = nullptr;
    size_t pool_bytes_ = 0;
    double *x_ = nullptr, *xcur_ = nullptr, *xprev_ = nullptr, *xprevprev_ = nullptr, *lb_ = nullptr, *ub_ = nullptr,
           *sigma_ = nullptr, *g_ = nullptr, *gcur_ = nullptr, *G_ = nullptr, *Gcur_ = nullptr;
    double *w_dev_ = nullptr, *xtol_abs_dev_ = nullptr;
    bool cand_in_x_ = true;       // the latest candidate's values live in x_ (start point / just accepted)

    // reduction workspace + result mailbox
    double *partials_ = nullptr, *vsums_ = nullptr, *out_dev_ = nullptr;
    unsigned *tickets_ = nullptr;
    double *out_host_ = nullptr;                     // mapped pinned
    unsigned long long *flag_host_ = nullptr;        // mapped pinned
    unsigned long long seq_ = 0;
    int nvp_ = 24;

    // staging for host callbacks
    double *h_x_ = nullptr;
    double *h_x_view_ = nullptr;                     // what the callbacks read: h_x_, or the node-shared segment
    double *h_grad_[2] = {nullptr, nullptr};
    size_t h_grad_cap_ = 0;
    int h_grad_next_ = 0;
    cudaEvent_t h_grad_done_[2] = {nullptr, nullptr};
    double *h_xs_ = nullptr, *h_gs_[2] = {nullptr, nullptr};     // sharded host callbacks: pinned shard of x, gradient staging
    cudaEvent_t h_gs_done_[2] = {nullptr, nullptr};
    int h_gs_next_ = 0, h_xs_slot_ = -1;
    unsigned long long h_xs_epoch_ = 0;
    double *xfull_dev_ = nullptr;                    // multi-rank host callbacks: gathered x
    double *pen_rows_ = nullptr;                     // augmented-Lagrangian objective: gradient rows of the folded constraints
    unsigned pen_total_ = 0;                         // their number (scalar constraints)
    double *scalar_dev_ = nullptr;                   // multi-rank device callbacks: value all-reduce
    std::vector<double> pend_val_;                   // shard-local values waiting for finish_evals()
    std::vector<char> pend_set_;
    bool pend_any_ = false;
    size_t scalar_cap_ = 0;
    // asynchronous device callbacks (nlopt_b200_dfunc2): [1+m][8] virtual-shard sums, device + pinned mirror
    double *vs2_dev_ = nullptr, *vs2_host_ = nullptr;
    size_t vs2_cap_ = 0;
    std::vector<const FuncSpec *> pend2_;
    bool pend2_any_ = false;
    // terms callbacks (nlopt_b200_dtfunc): [terms_rows_][ld] terms, shared by every terms callback of a point (stream
    // order), and their [terms_rows_][groups_local] group sums
    unsigned terms_rows_ = 0;                        // max m over the terms callbacks, 0: none
    double *terms_ = nullptr, *terms_part_ = nullptr;
    nlopt_b200_shard shard_{};
    double *halo_edges_ = nullptr;
    const double *halo_ptr_ = nullptr;
    unsigned long long halo_epoch_ = 0;
    size_t shard_cap_ = 0;                           // largest padded shard length over all ranks
    unsigned long long x_epoch_ = 1, h_x_epoch_ = 0; // which (slot, epoch) h_x_ currently mirrors
    int h_x_slot_ = -1;

    cudaStream_t stream_ = nullptr, copy_stream_ = nullptr;

    // optional per-launch timing of the dual kernel
    bool time_kernels_ = false;
    std::vector<cudaEvent_t> ev_pool_;
    size_t ev_used_ = 0;
    void drain_events();

    std::string err_;
    double cb_seconds_ = 0;
    nlopt_b200_stats local_stats_{};
    nlopt_b200_stats *stats_ = &local_stats_;
    unsigned max_cdim_ = 1;
};

void release_cached_blocks();

}  // namespace nb200
