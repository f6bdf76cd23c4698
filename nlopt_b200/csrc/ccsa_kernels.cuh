// ccsa_kernels.cuh -- the CUDA kernels of the MMA/CCSAQ hot path (sm_90a).
//
//   dual_eval_kernel      : one dual evaluation  y -> x*(y), val, g0, w, g_1..g_m over this rank's shard, m <= 16
//                           (reference: static dual_func, src/algs/mma/mma.c:59-137 and
//                            src/algs/mma/ccsa_quadratic.c:79-148); dual_eval_tma_kernel: same, operands staged by TMA
//   dual_eval_wide_kernel : the same for ANY number of constraints (m > 16): rows of the gradient block streamed in
//                           blocks of 8, the five n-vectors read once (the reference has no cap on m, mma.c:173)
//   dual_solve_kernel     : a whole dual solve (mma.c:275-288) in one persistent cooperative launch -- the default path
//   sigma_init_kernel     : mma.c:202-210
//   end_outer_kernel      : nlopt_stop_x norms (src/util/stop.c:98-108) + sigma update (mma.c:431-442,
//                           ccsa_quadratic.c:577-590) + xprev/xprevprev rotation (mma.c:264-265), one pass
//   penalty_axpy_kernel   : gradient of the augmented-Lagrangian objective (src/algs/auglag/auglag.c:47-48, :59-60)
//   negate_kernel         : sign flip of a maximised device / sharded objective's gradient (optimize.c:969-989)
//
// Arithmetic contract: every per-variable expression is evaluated with the reference's operation
// order using __dmul_rn/__dadd_rn/__dsub_rn/__ddiv_rn/__dsqrt_rn, which nvcc never contracts into
// FMAs -- the reference is built with -ffp-contract=off (CMakeLists.txt:281-284).  x*(y) is
// therefore bit-identical to the reference; only the ORDER of the n-term sums differs (fixed
// tree, see below), which is the documented parity tolerance.
//
// Reduction contract (deterministic and independent of the grid and of the number of GPUs): the global
// index space is cut into S = 8*P groups whose boundaries depend on n only (geometry.hpp).  A group is
// reduced with a fixed lane->element map and a fixed shuffle / shared-memory tree into one record of m+3
// sums, which its sweeper drops into a TAGGED 16-byte slot {value, tag} with one 128-bit store -- no fence,
// no atomic, no ticket.  The P records of a "virtual shard" (8 shards; each rank owns 8/world) are folded in a
// canonical order by a dedicated folder CTA that polls the tags (fold_generation), the rank's shard sums in
// index order, and the 8 shard sums of all ranks in index order.  Every kernel here uses the same folder code,
// so every path gives the same bits.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "dual_mma.hpp"
#include "pair_math.cuh"

namespace nb200 {

constexpr int kBlock = 256;              // threads per CTA of every kernel here
constexpr int kWarps = kBlock / 32;
constexpr int kVirtualShards = 8;        // V: fixed, so 1/2/4/8 ranks give bit-identical sums
constexpr int kMaxParamM = 16;           // multipliers that travel as kernel parameters (register-row kernels); m > 16: wide kernel
constexpr int kMaxNV = 3 + kMaxParamM;   // accumulators one CTA of the register-row kernels carries: val, g0, w, <=16 g_i
constexpr int kWideMaxM = 2048;          // the wide kernel keeps 96 bytes of shared memory per row: 4 per-row scalars and the
                                         // 8 warps' row sums; 192 KiB of dynamic shared memory at m = 2048

// ---- exact-rounding arithmetic (never fused) ---------------------------------------------
__device__ __forceinline__ double mulx(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double addx(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double subx(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double divx(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ unsigned long long nb_globaltimer()     // nanoseconds, one clock for all SMs and all GPUs of a node
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// streaming loads: read-once data must not displace anything in L1.  The L2 behaviour is chosen per ARRAY through a
// cache-policy operand: arrays the caller asks to keep (DualArgs::l2_keep, a bit per operand array) are loaded
// evict_last so that they survive in the 50 MB L2 from one dual evaluation to the next -- the persistent solve
// kernel re-reads the same (5+m) arrays every generation, and once a rank's shard is small enough (8 GPUs at
// n = 1e7: 10 MB per array) some of them fit; everything else is loaded evict_first so that it does not push them out.
__device__ __forceinline__ double2 ld_stream(const double2 *p)
{
    double2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ double2 ld_stream_pol(const double2 *p, unsigned long long pol)
{
    double2 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(v.x), "=d"(v.y) : "l"(p), "l"(pol));
    return v;
}

struct L2Policies {
    unsigned long long keep, stream;
    unsigned mask;                      // bit k set: operand array k (0 x, 1 lb, 2 ub, 3 sigma, 4 grad f, 5+i row i) is kept
    __device__ __forceinline__ void init(unsigned m)
    {
        mask = m;
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep));
        asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(stream));
    }
    __device__ __forceinline__ double2 ld(const double2 *p, int k) const
    {
        if (mask == 0u) return ld_stream(p);          // nothing to protect: the plain streaming load (no policy operand)
        return ld_stream_pol(p, ((mask >> k) & 1u) ? keep : stream);
    }
};
__device__ __forceinline__ void st_stream(double2 *p, double2 v)
{
    asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(v.x), "d"(v.y) : "memory");
}

// ---- tagged 128-bit mailbox slots (cross-rank exchange) ---------------------------------------------------
__device__ __forceinline__ void box_put(double *slot, double value, unsigned long long tag)
{
    asm volatile("st.volatile.global.v2.b64 [%0], {%1, %2};" ::"l"(slot), "l"(__double_as_longlong(value)), "l"(tag) : "memory");
}
__device__ __forceinline__ bool box_get(const double *slot, unsigned long long tag, double *value)
{
    long long v;
    unsigned long long t;
    asm volatile("ld.volatile.global.v2.b64 {%0, %1}, [%2];" : "=l"(v), "=l"(t) : "l"(slot) : "memory");
    *value = __longlong_as_double(v);
    return t == tag;
}
constexpr int kBoxStride = 24;           // slots per virtual shard record (comm.hpp): <= 19 sums + 1 flag slot
constexpr int kBoxFlagSlot = kMaxNV;     // slot 19: "this rank's time limit has expired" (see box_exchange)

// The same slots inside one GPU (group records and published multipliers of the persistent solve kernel):
// gpu-scope relaxed accesses are served by the L2.  (The .volatile = system-scope forms above, needed across
// NVLink, are slower per lane request when 32 lanes hit 32 different lines.)
__device__ __forceinline__ void slot_put(double *slot, double value, unsigned long long tag)
{
    asm volatile("st.relaxed.gpu.global.v2.b64 [%0], {%1, %2};" ::"l"(slot), "l"(__double_as_longlong(value)), "l"(tag) : "memory");
}
// Polling many slots per thread: strong (volatile / relaxed) loads of one thread complete one after the other
// (measured: the folder's tail grew with the number of strong loads per thread), weak loads pipeline.  ld.global.cg always reads the L2 -- where the producers' stores land -- and the
// tag travels in the same 16 bytes as the value, so a slot whose tag matches is complete.
__device__ __forceinline__ bool slot_peek(const double *slot, unsigned long long tag, double *value)
{
    long long v;
    unsigned long long t;
    asm volatile("ld.global.cg.v2.b64 {%0, %1}, [%2];" : "=l"(v), "=l"(t) : "l"(slot) : "memory");
    *value = __longlong_as_double(v);
    return t == tag;
}
__device__ __forceinline__ int ld_gpu_s32(const int *p)
{
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ bool slot_get(const double *slot, unsigned long long tag, double *value)
{
    long long v;
    unsigned long long t;
    asm volatile("ld.relaxed.gpu.global.v2.b64 {%0, %1}, [%2];" : "=l"(v), "=l"(t) : "l"(slot) : "memory");
    *value = __longlong_as_double(v);
    return t == tag;
}

// Lane k < nv: write this rank's shard records into every peer's mailbox, then gather all 8 records of
// sum k from the own mailbox and fold them in index order.  Lane kBoxFlagSlot carries one extra value per rank the
// same way (`flag`, 0 or 1: the rank's time limit has expired); its total comes back in *any_flag (warp-uniform), so
// that every rank takes the SAME decision -- a rank-local clock test would let one rank stop while its peers wait
// for its next record.  Returns the total in lanes < nv; *timed_out (a peer died) is warp-uniform.
// vsums: the shard sums written by this CTA (shared memory): plain loads.
// Polling: the 8 x (nv + 1) awaited slots are dealt out over the 32 lanes (slot s = 8 k + v to lane s % 32, register
// s / 32), so a poll round costs a lane ceil(8 (nv + 1) / 32) strong loads -- 2 for m = 4 -- instead of the 8 it cost when
// lane k fetched all 8 records of its own sum: strong (system-scope) loads of one thread complete one after the other,
// and this round trip is on the serial path of every generation on several GPUs.
// The records then travel to the lane that owns their sum by shuffles and are added in the same index order as before.
constexpr int kBoxPollRegs = (8 * (kMaxNV + 1) + 31) / 32;      // 5
__device__ __forceinline__ double box_exchange(double *const *box, int rank, int world, unsigned long long seq,
                                               const double *vsums, int nvp, unsigned local_vshards, unsigned v0,
                                               int nv, int lane, double flag, int *any_flag, int *timed_out)
{
    const int buf = (int) (seq & 1ull);
    if (lane < nv || lane == kBoxFlagSlot) {
        for (unsigned v = 0; v < local_vshards; ++v) {
            const double val = lane < nv ? vsums[(unsigned long long) v * nvp + lane] : flag;
            for (int r = 0; r < world; ++r)
                box_put(box[r] + 2ull * (((unsigned long long) buf * 8 + v0 + v) * kBoxStride + lane), val, seq);
        }
    }
    const int nslots = 8 * (nv + 1);
    const int nreg = (nslots + 31) >> 5;
    const double *mine = box[rank] + 2ull * ((unsigned long long) buf * 8 * kBoxStride);
    const double *slot[kBoxPollRegs];
#pragma unroll
    for (int j = 0; j < kBoxPollRegs; ++j) {
        const int sidx = lane + 32 * j;
        const int k = sidx >> 3, v = sidx & 7;
        slot[j] = mine + 2ull * ((unsigned long long) v * kBoxStride + (k < nv ? k : kBoxFlagSlot));
    }
    double x[kBoxPollRegs];
#pragma unroll
    for (int j = 0; j < kBoxPollRegs; ++j) x[j] = 0.0;
    const unsigned long long t0 = nb_globaltimer();
    int to = 0;
    for (;;) {
        bool all = true;
#pragma unroll
        for (int j = 0; j < kBoxPollRegs; ++j)
            if (j < nreg && lane + 32 * j < nslots) all = box_get(slot[j], seq, &x[j]) && all;
        if (__all_sync(0xffffffffu, all)) break;
        if (__any_sync(0xffffffffu, nb_globaltimer() - t0 > 10000000000ull)) { to = 1; break; }      // 10 s: a peer died
    }
    // lane kd's sum: records (kd, v), v = 0..7, in index order
    const int kd = lane < nv ? lane : (lane == kBoxFlagSlot ? nv : -1);
    double total = 0.0;
#pragma unroll
    for (int v = 0; v < kVirtualShards; ++v) {
        const int sidx = kd >= 0 ? 8 * kd + v : 0;
        double pick = 0.0;
#pragma unroll
        for (int j = 0; j < kBoxPollRegs; ++j)
            if (j < nreg) {
                const double t = __shfl_sync(0xffffffffu, x[j], sidx & 31);
                if ((sidx >> 5) == j) pick = t;
            }
        total = v == 0 ? pick : addx(total, pick);
    }
    if (kd < 0) total = 0.0;
    *timed_out = to;
    *any_flag = __shfl_sync(0xffffffffu, total, kBoxFlagSlot) > 0.0 ? 1 : 0;
    return total;
}

// ---- arguments of one dual evaluation -------------------------------------------------------
constexpr int kGroupWarps = 8;           // warps that sweep one group together (fixed: part of the reduction order)
constexpr int kChunkPairs = 32 * kGroupWarps;   // 256 double2 pairs = 512 variables = 4 KB per array per sweep step

struct DualArgs {
    // shard-local arrays (16-byte aligned, padded with sigma = 0 lanes)
    const double *x, *lb, *ub, *sigma, *g;
    const double *G;              // m rows of ld doubles
    double *xcur;                 // written iff STORE
    unsigned long long ld;        // row stride of G in doubles
    // group geometry (global, depends on n only): group s covers chunks [s*nchunks/S, (s+1)*nchunks/S)
    unsigned long long nchunks;   // ceil(ceil(n/2) / 256) over ALL ranks
    unsigned long long chunk0;    // first global chunk of this rank
    unsigned nseg_total;          // S = 8 * P
    unsigned seg0;                // first global group of this rank
    unsigned segs_per_vshard;     // P
    unsigned local_vshards;       // 8 / world
    // reduction workspace
    double *grouptags;            // [nvp][local groups] tagged slots {value, tag}: the group records
    unsigned long long tag;       // tag of this evaluation's records (unique per launch)
    double *out_dev;              // [8][nvp] all-rank exchange buffer (this rank's slots filled)   (NCCL path)
    volatile double *out_host;    // mapped pinned [nvp]; written when publish_host or the mailbox exchange is used
    volatile unsigned long long *flag_host;
    unsigned long long seq;
    int publish_host;             // 1: single rank, results + flag go straight to the host
    int nvp;                      // stride of one record (>= 3 + m)
    // fused cross-rank exchange over NVLink peer memory (null box[0]: NCCL path instead)
    double *box[8];               // box[r]: rank r's mailbox as mapped into this process (CUDA IPC)
    int rank, world;
    // the multipliers and penalties
    int m;                        // total number of constraints (rows of G)
    unsigned active;              // bit i clear: constraint i switched off (MMA, NaN value)            (m <= 16)
    unsigned l2_keep;             // operand arrays to hold in L2 across evaluations (L2Policies::mask)
    double rho, half_rho, u_ccsaq;    // u_ccsaq = rho + sum_i rhoc_i y_i (ccsa_quadratic.c:116-120)
    double y[kMaxParamM], rhoc[kMaxParamM], half_rhoc[kMaxParamM];       // (m <= 16)
    const double *wide;           // m > 16: device block  y[m] | rhoc[m] | half_rhoc[m] | active[m] (1.0 / 0.0)
    double lb_u, ub_u;            // the value of every lb / ub entry when both are uniform (read by the SB instantiations)
    // sigma index (DeviceBackend: valid with uniform bounds and a uniform initial step): sigma[j] == pal[sidx[j]] bit for
    // bit, read by the kSigmaIndex instantiations of dual_solve_tma_kernel instead of sigma
    const unsigned short *sidx;
    const double *pal;
    __device__ __forceinline__ double u() const { return u_ccsaq; }
};

// pair range [p_lo, p_hi) of global group `seg`, relative to the start of this rank's shard
__device__ __forceinline__ void group_pairs(unsigned long long nchunks, unsigned nseg_total, unsigned long long chunk0,
                                            unsigned seg, unsigned long long *p_lo, unsigned long long *p_hi)
{
    *p_lo = ((unsigned long long) seg * nchunks / nseg_total - chunk0) * kChunkPairs;
    *p_hi = ((unsigned long long) (seg + 1) * nchunks / nseg_total - chunk0) * kChunkPairs;
}

// ---- block-level reduction with a fixed tree (end_outer_kernel) ----------------------------------
template <int NV, int BLOCK = kBlock>
__device__ __forceinline__ void block_reduce_to(double (&acc)[NV], double *smem /* [(BLOCK/32)*NV] */, double *out)
{
    constexpr int kWarpsB = BLOCK / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        double v = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v = addx(v, __shfl_xor_sync(0xffffffffu, v, off));
        if (lane == 0) smem[warp * NV + k] = v;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double s = smem[threadIdx.x];
#pragma unroll
        for (int w = 1; w < kWarpsB; ++w) s = addx(s, smem[w * NV + threadIdx.x]);
        out[threadIdx.x] = s;
    }
    __syncthreads();
}

// true in exactly one CTA: the one whose ticket completes `total`   (end_outer_kernel: once per outer iteration)
__device__ __forceinline__ bool is_last_arrival(unsigned *ticket, unsigned total, int *s_flag)
{
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) *s_flag = (atomicAdd(ticket, 1u) == total - 1u);
    __syncthreads();
    return *s_flag != 0;
}

// ---- per-variable closed forms ------------------------------------------------------------------
// MAXM rows of grad_c are kept in registers (m <= MAXM); FULL means m == MAXM with every constraint active, which
// strips the per-row predicates from the unrolled loops (the common case m in {1,2,4,8,16}).
// MMA: mma.c:96-129.
template <int MAXM, bool FULL, class MU>
__device__ __forceinline__ double mma_point(const MU &a, double x, double lb, double ub, double s, double g,
                                            const double (&Gr)[MAXM > 0 ? MAXM : 1], double (&acc)[3 + (MAXM > 0 ? MAXM : 1)])
{
    if (s == 0) return x;                                    // fixed variable, mma.c:96-99
    const double ag_s = mulx(fabs(g), s);
    double u = g;
    double v = addx(ag_s, a.half_rho);
#pragma unroll
    for (int i = 0; i < MAXM; ++i)
        if (FULL || (i < a.m && ((a.active >> i) & 1u))) {
            u = addx(u, mulx(Gr[i], a.y[i]));
            v = addx(v, mulx(addx(mulx(fabs(Gr[i]), s), a.half_rhoc[i]), a.y[i]));
        }
    const double s2 = mulx(s, s);
    u = mulx(u, s2);
    const double r = divx(u, mulx(v, s));
    double dx = divx(divx(u, v), subx(-1.0, __dsqrt_rn(fabs(subx(1.0, mulx(r, r))))));   // mma.c:108
    double xc = addx(x, dx);
    if (xc > ub) xc = ub; else if (xc < lb) xc = lb;        // mma.c:110-111
    const double lim = mulx(0.9, s), hi = addx(x, lim), lo = subx(x, lim);
    if (xc > hi) xc = hi; else if (xc < lo) xc = lo;        // mma.c:112-113
    dx = subx(xc, x);
    const double dx2 = mulx(dx, dx);
    const double dinv = divx(1.0, subx(s2, dx2));
    acc[0] = addx(acc[0], mulx(addx(mulx(u, dx), mulx(v, dx2)), dinv));                  // mma.c:119
    const double c = mulx(s2, dx);
    acc[1] = addx(acc[1], mulx(addx(mulx(g, c), mulx(addx(ag_s, a.half_rho), dx2)), dinv));   // mma.c:123
    acc[2] = addx(acc[2], mulx(mulx(0.5, dx2), dinv));                                  // mma.c:125
#pragma unroll
    for (int k = 0; k < MAXM; ++k)
        if (FULL || (k < a.m && ((a.active >> k) & 1u)))
            acc[3 + k] = addx(acc[3 + k],
                              mulx(addx(mulx(Gr[k], c), mulx(addx(mulx(fabs(Gr[k]), s), a.half_rhoc[k]), dx2)), dinv));   // mma.c:127
    return xc;
}

// CCSAQ: ccsa_quadratic.c:111-140
template <int MAXM, bool FULL, class MU>
__device__ __forceinline__ double ccsaq_point(const MU &a, double x, double lb, double ub, double s, double g,
                                              const double (&Gr)[MAXM > 0 ? MAXM : 1], double (&acc)[3 + (MAXM > 0 ? MAXM : 1)])
{
    if (s == 0) return x;                                    // ccsa_quadratic.c:111-114
    double v = g;
#pragma unroll
    for (int i = 0; i < MAXM; ++i)
        if (FULL || i < a.m) v = addx(v, mulx(Gr[i], a.y[i]));
    const double u = a.u();
    const double s2 = mulx(s, s);
    double dx = divx(mulx(-s2, v), u);                       // ccsa_quadratic.c:122
    if (fabs(dx) > s) dx = copysign(s, dx);                  // ccsa_quadratic.c:126
    double xc = addx(x, dx);
    if (xc > ub) xc = ub; else if (xc < lb) xc = lb;
    dx = subx(xc, x);
    const double dx2 = mulx(dx, dx);
    acc[0] = addx(acc[0], addx(mulx(v, dx), divx(mulx(mulx(0.5, u), dx2), s2)));         // ccsa_quadratic.c:134
    const double q = divx(mulx(0.5, dx2), s2);
    acc[1] = addx(acc[1], addx(mulx(g, dx), mulx(a.rho, q)));                            // :137
    acc[2] = addx(acc[2], q);                                                            // :138
#pragma unroll
    for (int k = 0; k < MAXM; ++k)
        if (FULL || k < a.m) acc[3 + k] = addx(acc[3 + k], addx(mulx(Gr[k], dx), mulx(a.rhoc[k], q)));       // :139-140
    return xc;
}

// Where the pair form of MMA is used: with 4 or more gradient rows the two interleaved variables of MMA no longer fit
// the 80-register budget of 3 CTAs/SM (they spill) -- there the sequential form stays.
#ifndef NB200_PAIR_MMA_MAXM
#define NB200_PAIR_MMA_MAXM 2
#endif
template <int MAXM>
constexpr bool kPairMMA = MAXM <= NB200_PAIR_MMA_MAXM;

// ---- the same closed forms for the two variables of one 128-bit load, as straight-line code (pair_math.cuh) -------
// Every value is produced by the same operation on the same operands as in mma_point / ccsaq_point; only the divisions,
// the square root and the reciprocal come from the written-out fast paths, with the builtins as the fallback.
template <int MAXM, bool FULL, class MU>
__device__ __forceinline__ double2 mma_pair(const MU &a, const double2 x, const double2 lb, const double2 ub, const double2 s,
                                            const double2 g, const double (&Ga)[MAXM > 0 ? MAXM : 1],
                                            const double (&Gb)[MAXM > 0 ? MAXM : 1], double (&acc)[3 + (MAXM > 0 ? MAXM : 1)])
{
    double2 xc;
    if (s.x == 0 || s.y == 0) {                              // a fixed variable or a padding lane in the pair (mma.c:96-99)
        xc.x = mma_point<MAXM, FULL>(a, x.x, lb.x, ub.x, s.x, g.x, Ga, acc);
        xc.y = mma_point<MAXM, FULL>(a, x.y, lb.y, ub.y, s.y, g.y, Gb, acc);
        return xc;
    }
    // u, v (mma.c:101-106)
    const double v0A = addx(mulx(fabs(g.x), s.x), a.half_rho), v0B = addx(mulx(fabs(g.y), s.y), a.half_rho);
    double uA = g.x, uB = g.y, vA = v0A, vB = v0B;
#pragma unroll
    for (int i = 0; i < MAXM; ++i)
        if (FULL || (i < a.m && ((a.active >> i) & 1u))) {
            const double yi = a.y[i], hi = a.half_rhoc[i];
            uA = addx(uA, mulx(Ga[i], yi));
            uB = addx(uB, mulx(Gb[i], yi));
            vA = addx(vA, mulx(addx(mulx(fabs(Ga[i]), s.x), hi), yi));
            vB = addx(vB, mulx(addx(mulx(fabs(Gb[i]), s.y), hi), yi));
        }
    const double s2A = mulx(s.x, s.x), s2B = mulx(s.y, s.y);
    uA = mulx(uA, s2A);
    uB = mulx(uB, s2B);
    // dx (mma.c:108): four independent divisions, two square roots, two more divisions
    unsigned bad = 0u;
    const double rA = div_fast(uA, mulx(vA, s.x), bad), rB = div_fast(uB, mulx(vB, s.y), bad);
    const double qA = div_fast(uA, vA, bad), qB = div_fast(uB, vB, bad);
    const double sqA = sqrt_fast(fabs(subx(1.0, mulx(rA, rA))), bad), sqB = sqrt_fast(fabs(subx(1.0, mulx(rB, rB))), bad);
    double dxA = div_fast(qA, subx(-1.0, sqA), bad), dxB = div_fast(qB, subx(-1.0, sqB), bad);
    if (bad) {                                               // some operand outside the fast paths' range: the builtins
        const double r1 = divx(uA, mulx(vA, s.x)), r2 = divx(uB, mulx(vB, s.y));
        dxA = divx(divx(uA, vA), subx(-1.0, __dsqrt_rn(fabs(subx(1.0, mulx(r1, r1))))));
        dxB = divx(divx(uB, vB), subx(-1.0, __dsqrt_rn(fabs(subx(1.0, mulx(r2, r2))))));
    }
    // clamps (mma.c:109-114)
    double xA = addx(x.x, dxA), xB = addx(x.y, dxB);
    if (xA > ub.x) xA = ub.x; else if (xA < lb.x) xA = lb.x;
    if (xB > ub.y) xB = ub.y; else if (xB < lb.y) xB = lb.y;
    const double limA = mulx(0.9, s.x), limB = mulx(0.9, s.y);
    const double hiA = addx(x.x, limA), loA = subx(x.x, limA), hiB = addx(x.y, limB), loB = subx(x.y, limB);
    if (xA > hiA) xA = hiA; else if (xA < loA) xA = loA;
    if (xB > hiB) xB = hiB; else if (xB < loB) xB = loB;
    dxA = subx(xA, x.x);
    dxB = subx(xB, x.y);
    const double dx2A = mulx(dxA, dxA), dx2B = mulx(dxB, dxB);
    const double dA = subx(s2A, dx2A), dB = subx(s2B, dx2B);
    unsigned bad2 = 0u;
    double dinvA = rcp_fast(dA, bad2), dinvB = rcp_fast(dB, bad2);
    if (bad2) {
        dinvA = divx(1.0, dA);
        dinvB = divx(1.0, dB);
    }
    // the sums (mma.c:119-129): first variable, then second, as the sequential form adds them
    const double cA = mulx(s2A, dxA), cB = mulx(s2B, dxB);
    acc[0] = addx(acc[0], mulx(addx(mulx(uA, dxA), mulx(vA, dx2A)), dinvA));
    acc[0] = addx(acc[0], mulx(addx(mulx(uB, dxB), mulx(vB, dx2B)), dinvB));
    acc[1] = addx(acc[1], mulx(addx(mulx(g.x, cA), mulx(v0A, dx2A)), dinvA));
    acc[1] = addx(acc[1], mulx(addx(mulx(g.y, cB), mulx(v0B, dx2B)), dinvB));
    acc[2] = addx(acc[2], mulx(mulx(0.5, dx2A), dinvA));
    acc[2] = addx(acc[2], mulx(mulx(0.5, dx2B), dinvB));
#pragma unroll
    for (int k = 0; k < MAXM; ++k)
        if (FULL || (k < a.m && ((a.active >> k) & 1u))) {
            const double hk = a.half_rhoc[k];
            acc[3 + k] = addx(acc[3 + k], mulx(addx(mulx(Ga[k], cA), mulx(addx(mulx(fabs(Ga[k]), s.x), hk), dx2A)), dinvA));
            acc[3 + k] = addx(acc[3 + k], mulx(addx(mulx(Gb[k], cB), mulx(addx(mulx(fabs(Gb[k]), s.y), hk), dx2B)), dinvB));
        }
    xc.x = xA;
    xc.y = xB;
    return xc;
}

// CCSAQ: the divisor of the first division is u = rho + sum rhoc_i y_i, the same for every variable
// (ccsa_quadratic.c:116-122): its reciprocal is prepared once per group (`U`); the other two divisions of a variable
// share the divisor sigma^2 (:134-138) and one prepared reciprocal.
template <int MAXM, bool FULL, class MU>
__device__ __forceinline__ double2 ccsaq_pair(const MU &a, const DivBy &U, const double2 x, const double2 lb, const double2 ub,
                                              const double2 s, const double2 g, const double (&Ga)[MAXM > 0 ? MAXM : 1],
                                              const double (&Gb)[MAXM > 0 ? MAXM : 1], double (&acc)[3 + (MAXM > 0 ? MAXM : 1)])
{
    double2 xc;
    if (s.x == 0 || s.y == 0) {                              // ccsa_quadratic.c:111-114
        xc.x = ccsaq_point<MAXM, FULL>(a, x.x, lb.x, ub.x, s.x, g.x, Ga, acc);
        xc.y = ccsaq_point<MAXM, FULL>(a, x.y, lb.y, ub.y, s.y, g.y, Gb, acc);
        return xc;
    }
    double vA = g.x, vB = g.y;
#pragma unroll
    for (int i = 0; i < MAXM; ++i)
        if (FULL || i < a.m) {
            const double yi = a.y[i];
            vA = addx(vA, mulx(Ga[i], yi));
            vB = addx(vB, mulx(Gb[i], yi));
        }
    const double u = U.b;
    const double s2A = mulx(s.x, s.x), s2B = mulx(s.y, s.y);
    const double nA = mulx(-s2A, vA), nB = mulx(-s2B, vB);
    unsigned bad = 0u;
    double dxA = div_by(nA, U, bad), dxB = div_by(nB, U, bad);        // ccsa_quadratic.c:122
    if (bad) {
        dxA = divx(nA, u);
        dxB = divx(nB, u);
    }
    if (fabs(dxA) > s.x) dxA = copysign(s.x, dxA);          // :126
    if (fabs(dxB) > s.y) dxB = copysign(s.y, dxB);
    double xA = addx(x.x, dxA), xB = addx(x.y, dxB);
    if (xA > ub.x) xA = ub.x; else if (xA < lb.x) xA = lb.x;
    if (xB > ub.y) xB = ub.y; else if (xB < lb.y) xB = lb.y;
    dxA = subx(xA, x.x);
    dxB = subx(xB, x.y);
    const double dx2A = mulx(dxA, dxA), dx2B = mulx(dxB, dxB);
    const double hu = mulx(0.5, u);
    const double n0A = mulx(hu, dx2A), n0B = mulx(hu, dx2B), n1A = mulx(0.5, dx2A), n1B = mulx(0.5, dx2B);
    const DivBy SA = prep_div(s2A), SB = prep_div(s2B);
    unsigned bad2 = 0u;
    double t0A = div_by(n0A, SA, bad2), t0B = div_by(n0B, SB, bad2);
    double qA = div_by(n1A, SA, bad2), qB = div_by(n1B, SB, bad2);
    if (bad2) {
        t0A = divx(n0A, s2A); t0B = divx(n0B, s2B);
        qA = divx(n1A, s2A); qB = divx(n1B, s2B);
    }
    acc[0] = addx(acc[0], addx(mulx(vA, dxA), t0A));        // :134
    acc[0] = addx(acc[0], addx(mulx(vB, dxB), t0B));
    acc[1] = addx(acc[1], addx(mulx(g.x, dxA), mulx(a.rho, qA)));   // :137
    acc[1] = addx(acc[1], addx(mulx(g.y, dxB), mulx(a.rho, qB)));
    acc[2] = addx(acc[2], qA);                               // :138
    acc[2] = addx(acc[2], qB);
#pragma unroll
    for (int k = 0; k < MAXM; ++k)
        if (FULL || k < a.m) {
            const double rk = a.rhoc[k];
            acc[3 + k] = addx(acc[3 + k], addx(mulx(Ga[k], dxA), mulx(rk, qA)));     // :139-140
            acc[3 + k] = addx(acc[3 + k], addx(mulx(Gb[k], dxB), mulx(rk, qB)));
        }
    xc.x = xA;
    xc.y = xB;
    return xc;
}

template <int NV>
__device__ __forceinline__ void warp_fold(double (&acc)[NV])
{
#pragma unroll
    for (int k = 0; k < NV; ++k) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc[k] = addx(acc[k], __shfl_xor_sync(0xffffffffu, acc[k], off));
    }
}

// ---- folding the tagged group records of one evaluation (one "generation") --------------------------------------
// Slot (group gl, sum k) lives at grouptags[2 * (k * ngroups + gl)]: the 32 lanes of a poll read 512 contiguous bytes.
// fold_generation<NV>: called by ALL 256 threads of the folder CTA.  Polls the records tagged `tag` of the local
// virtual shards for the sums [k0, k0 + nk), nk <= NV, and leaves the shard sums in s_vs[v * NV + k] (valid after
// the call for warp 0, which is the only reader).
// Canonical order of one shard's P records: chain t in [0, 256) adds records t, t+256, ... in index order; the 32
// chains of "fold warp" w = t / 32 meet in an xor butterfly; the 8 fold-warp results are added in warp order.  Work
// item (v, w) = fold warp w of local shard v; items are dealt round-robin to the 8 physical warps in (v, w) order --
// shards complete roughly in index order, and when P <= 32 (small n, or one shard per rank with 8 GPUs) all shards
// are polled side by side.  Empty fold warps contribute the +0.0 parked in s_w by fold_init.
// Warp-uniform control flow: a warp polls until all of its lanes have their record (measured: a warp whose lanes
// left the poll loop at different times was several times slower per shard).
// barrier of the 8 folder warps (a named barrier with an explicit count: the TMA kernel's CTAs carry a ninth warp)
__device__ __forceinline__ void fold_barrier() { asm volatile("bar.sync 1, %0;" ::"r"(32 * kGroupWarps) : "memory"); }

template <int NV>
__device__ __forceinline__ void fold_init(double *s_w)
{
    for (int i = threadIdx.x; i < kVirtualShards * kGroupWarps * NV; i += 32 * kGroupWarps) s_w[i] = 0.0;
    fold_barrier();
}

template <int NV>
__device__ __forceinline__ void fold_generation(const double *grouptags, unsigned ngroups, unsigned P, unsigned local_vshards,
                                                unsigned long long tag, int k0, int nk, double *s_w, double *s_vs,
                                                bool reverse = false)
{
    const int lane = threadIdx.x & 31;
    const int sub = threadIdx.x >> 5;
    const unsigned fw_all = (P + 31u) / 32u;
    const unsigned fw_per = fw_all < (unsigned) kGroupWarps ? fw_all : (unsigned) kGroupWarps;      // non-empty fold warps per shard
    const unsigned nitems = local_vshards * fw_per;
    // (Polling two items per round trip was tried and measured slower.)
    // reverse: the items are polled last shard first, for generations whose groups were claimed in descending order.
    // Each item writes its own slot of s_w, so the order in which they are polled does not change a bit.
    for (unsigned i = sub; i < nitems; i += kGroupWarps) {
        const unsigned item = reverse ? nitems - 1 - i : i;
        const unsigned v = item / fw_per, w = item % fw_per;
        double acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[k] = 0.0;
        const double *base = grouptags + 2ull * ((unsigned long long) k0 * ngroups + (unsigned long long) v * P);
        for (unsigned r0 = 32u * w; r0 < P; r0 += 32 * kGroupWarps) {
            const unsigned r = r0 + lane;
            const bool has = r < P;
            const double *rec = base + 2ull * (has ? r : 0u);
            double val[NV];
            for (;;) {                // the sums of a record are fetched together: one round trip per poll
                bool all = true;
#pragma unroll
                for (int k = 0; k < NV; ++k) {
                    val[k] = 0.0;
                    if (k < nk) all = slot_peek(rec + 2ull * k * ngroups, tag, &val[k]) && all;
                }
                if (__all_sync(0xffffffffu, all || !has)) break;
                __nanosleep(20);
            }
            if (has) {
#pragma unroll
                for (int k = 0; k < NV; ++k) acc[k] = addx(acc[k], val[k]);
            }
        }
        warp_fold<NV>(acc);
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < NV; ++k) s_w[(v * kGroupWarps + w) * NV + k] = acc[k];
        }
    }
    fold_barrier();
    // the 8 fold-warp results of every (shard, sum) pair in warp order: one thread per pair (a single lane walking all
    // shards cost 64 dependent shared-memory adds on every generation's serial tail)
    if (threadIdx.x < local_vshards * NV) {
        const unsigned v = threadIdx.x / NV, k = threadIdx.x % NV;
        double t = s_w[(v * kGroupWarps) * NV + k];
#pragma unroll
        for (int w = 1; w < kGroupWarps; ++w) t = addx(t, s_w[(v * kGroupWarps + w) * NV + k]);
        s_vs[v * NV + k] = t;
    }
    fold_barrier();
}

// The folder CTA of the one-evaluation kernels (the last CTA of the grid; sweepers never wait for it, so it may start
// late when the grid exceeds the machine).  Sums [0, nv_total) in tiles of NV.
//   single rank          : totals -> mapped pinned out_host, then the flag
//   mailbox exchange     : shard sums -> every peer's mailbox -> totals -> out_host, flag      (nv_total <= kMaxNV)
//   NCCL exchange        : shard sums -> out_dev (ncclAllGather + publish_kernel follow on the stream)
template <int NV>
__device__ __noinline__ void eval_folder(const DualArgs &a, int nv_total)
{
    __shared__ double s_vs[kVirtualShards * NV];
    __shared__ double s_w[kVirtualShards * kGroupWarps * NV];
    const int lane = threadIdx.x & 31, sub = threadIdx.x >> 5;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;
    fold_init<NV>(s_w);
    for (int k0 = 0; k0 < nv_total; k0 += NV) {
        const int nk = nv_total - k0 < NV ? nv_total - k0 : NV;
        fold_generation<NV>(a.grouptags, ngroups, a.segs_per_vshard, a.local_vshards, a.tag, k0, nk, s_w, s_vs);
        if (sub == 0) {
            if (a.publish_host) {
                if (lane < nk) {
                    double s = s_vs[lane];
                    for (unsigned v = 1; v < a.local_vshards; ++v) s = addx(s, s_vs[v * NV + lane]);
                    a.out_host[k0 + lane] = s;
                }
            } else if (a.box[0] == nullptr) {
                const unsigned v0 = a.seg0 / a.segs_per_vshard;
                if (lane < nk)
                    for (unsigned v = 0; v < a.local_vshards; ++v)
                        a.out_dev[(unsigned long long) (v0 + v) * a.nvp + k0 + lane] = s_vs[v * NV + lane];
            } else {
                int timed_out = 0, any_flag = 0;
                const double total = box_exchange(a.box, a.rank, a.world, a.seq, s_vs, NV, a.local_vshards,
                                                  a.seg0 / a.segs_per_vshard, nk, lane, 0.0, &any_flag, &timed_out);
                if (lane < nk) a.out_host[k0 + lane] = timed_out ? __longlong_as_double(0x7ff8000000000000ll) : total;
            }
        }
        fold_barrier();
    }
    if (sub == 0 && (a.publish_host || a.box[0] != nullptr)) {
        __threadfence_system();
        __syncwarp();
        if (lane == 0) {
            *a.flag_host = a.seq;
            __threadfence_system();
        }
    }
}

// ---- the dual evaluation kernel ---------------------------------------------------------------------
// Persistent sweeper CTAs (grid sized to the machine) + one folder CTA.  A *group* is a contiguous run of
// 512-variable chunks; the 8 warps of a group slot sweep it together -- sweep step t reads one 4 KB-contiguous chunk
// per array, warp w taking lanes [32w, 32w+32) of it -- but every warp keeps its OWN m+3 accumulators over the group
// and folds them with a fixed xor-butterfly into a warp record.  The streaming loop has no barrier; one
// slot barrier per group hands the 8 warp records to warp 0 through shared memory.
// Fold tree (all in fixed order, all un-fused adds):
//   warp record -> group record (8 warp records in warp order, by warp 0 of the slot)
//               -> virtual-shard sum (P group records, canonical order, by the folder CTA)
//               -> rank sum / exchange (8/world shard sums in index order).
// A record depends only on n (the cuts) -- never on the grid size, on which CTA swept the group or on the
// number of ranks -- so the m+3 sums are bit-identical for every launch geometry and every world size.
//
// Sweep one group: this warp's lanes of every chunk of group `gl`, m+3 lane accumulators.
// SB ("scalar bounds"): every lb entry equals a.lb_u and every ub entry a.ub_u (box bounds set with
// nlopt_set_*_bounds1).  The two arrays are not read: 3 + m operand arrays per evaluation instead of 5 + m.  The
// closed forms receive the same values as from the arrays, so the results are the same bits.
template <int VARIANT, int MAXM, bool FULL, int UNROLL, bool SB, class MU>
__device__ __forceinline__ void sweep_group(const DualArgs &a, const MU &mu, bool store, unsigned gl, int sub, int lane,
                                            double (&acc)[3 + (MAXM > 0 ? MAXM : 1)])
{
    constexpr int MR = MAXM > 0 ? MAXM : 1;
    const double2 *x2 = reinterpret_cast<const double2 *>(a.x);
    const double2 *lb2 = reinterpret_cast<const double2 *>(a.lb);
    const double2 *ub2 = reinterpret_cast<const double2 *>(a.ub);
    const double2 *s2v = reinterpret_cast<const double2 *>(a.sigma);
    const double2 *g2 = reinterpret_cast<const double2 *>(a.g);
    unsigned long long p_lo, p_hi;
    group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + gl, &p_lo, &p_hi);
    DivBy U;
    if (VARIANT != 0) U = prep_div(mu.u());                  // CCSAQ: every variable divides by the same u

    for (unsigned long long p0 = p_lo + sub * 32 + lane; p0 < p_hi; p0 += (unsigned long long) kChunkPairs * UNROLL) {
        double2 vx[UNROLL], vlb[UNROLL], vub[UNROLL], vs[UNROLL], vg[UNROLL];
        double Ga[UNROLL][MR], Gb[UNROLL][MR];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const unsigned long long p = p0 + (unsigned long long) kChunkPairs * u;
            const bool live = u == 0 || p < p_hi;
            vs[u] = make_double2(0.0, 0.0);      // sigma = 0 lanes are skipped by both formulas
            vx[u] = vlb[u] = vub[u] = vg[u] = make_double2(0.0, 0.0);
            if (SB) {
                vlb[u] = make_double2(a.lb_u, a.lb_u);
                vub[u] = make_double2(a.ub_u, a.ub_u);
            }
            if (live) {
                vx[u] = ld_stream(x2 + p);
                if (!SB) { vlb[u] = ld_stream(lb2 + p); vub[u] = ld_stream(ub2 + p); }
                vs[u] = ld_stream(s2v + p); vg[u] = ld_stream(g2 + p);
            }
#pragma unroll
            for (int i = 0; i < MR; ++i) {
                Ga[u][i] = 0.0;
                Gb[u][i] = 0.0;
                if (MAXM > 0 && (FULL || i < mu.m) && live) {
                    const double2 *gp = reinterpret_cast<const double2 *>(a.G + (unsigned long long) i * a.ld) + p;
                    const double2 t = ld_stream(gp);
                    Ga[u][i] = t.x;
                    Gb[u][i] = t.y;
                }
            }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const unsigned long long p = p0 + (unsigned long long) kChunkPairs * u;
            const bool live = u == 0 || p < p_hi;
            double2 xc;
            if (VARIANT == 0 && kPairMMA<MAXM>) xc = mma_pair<MAXM, FULL>(mu, vx[u], vlb[u], vub[u], vs[u], vg[u], Ga[u], Gb[u], acc);
            else if (VARIANT != 0) xc = ccsaq_pair<MAXM, FULL>(mu, U, vx[u], vlb[u], vub[u], vs[u], vg[u], Ga[u], Gb[u], acc);
            else {
                xc.x = mma_point<MAXM, FULL>(mu, vx[u].x, vlb[u].x, vub[u].x, vs[u].x, vg[u].x, Ga[u], acc);
                xc.y = mma_point<MAXM, FULL>(mu, vx[u].y, vlb[u].y, vub[u].y, vs[u].y, vg[u].y, Gb[u], acc);
            }
            if (store && live) st_stream(reinterpret_cast<double2 *>(a.xcur) + p, xc);
        }
    }
}

// ---- the same sweep in two halves: the operand loads of a chunk, and the arithmetic on them --------------------------
// The persistent solve kernel issues the loads of the FIRST chunk of a group before it looks for the multipliers of the
// generation (the operands do not depend on y): while warp 0 polls the published slots and the CTA meets at its barrier
// the 5+m loads of every thread are already in flight, so one load latency (from HBM or the L2) leaves
// the critical path of every generation.  Same lanes, same order of operations as sweep_group: the same bits.
template <int MAXM>
struct ChunkOperands {
    double2 x, lb, ub, s, g;
    double Ga[MAXM > 0 ? MAXM : 1], Gb[MAXM > 0 ? MAXM : 1];
};

template <int MAXM, bool FULL, bool POL, bool SB>
__device__ __forceinline__ void load_chunk(const DualArgs &a, int m, const L2Policies &pol, unsigned long long p, bool live,
                                           ChunkOperands<MAXM> &r)
{
    constexpr int MR = MAXM > 0 ? MAXM : 1;
    r.s = make_double2(0.0, 0.0);                 // sigma = 0 lanes are skipped by both formulas
    r.x = r.lb = r.ub = r.g = make_double2(0.0, 0.0);
    if (SB) {                                     // uniform bounds (see sweep_group): no lb / ub loads
        r.lb = make_double2(a.lb_u, a.lb_u);
        r.ub = make_double2(a.ub_u, a.ub_u);
    }
    if (live) {
        const double2 *x2 = reinterpret_cast<const double2 *>(a.x) + p;
        const double2 *lb2 = reinterpret_cast<const double2 *>(a.lb) + p;
        const double2 *ub2 = reinterpret_cast<const double2 *>(a.ub) + p;
        const double2 *s2v = reinterpret_cast<const double2 *>(a.sigma) + p;
        const double2 *g2 = reinterpret_cast<const double2 *>(a.g) + p;
        if (POL) {
            r.x = pol.ld(x2, 0);
            if (!SB) { r.lb = pol.ld(lb2, 1); r.ub = pol.ld(ub2, 2); }
            r.s = pol.ld(s2v, 3); r.g = pol.ld(g2, 4);
        } else {
            r.x = ld_stream(x2);
            if (!SB) { r.lb = ld_stream(lb2); r.ub = ld_stream(ub2); }
            r.s = ld_stream(s2v); r.g = ld_stream(g2);
        }
    }
#pragma unroll
    for (int i = 0; i < MR; ++i) {
        r.Ga[i] = 0.0;
        r.Gb[i] = 0.0;
        if (MAXM > 0 && (FULL || i < m) && live) {
            const double2 *gp = reinterpret_cast<const double2 *>(a.G + (unsigned long long) i * a.ld) + p;
            const double2 t = POL ? pol.ld(gp, 5 + i) : ld_stream(gp);
            r.Ga[i] = t.x;
            r.Gb[i] = t.y;
        }
    }
}

// PAIR_MMA: the MMA pair form (callers with a 128-register budget set it for any row count)
template <int VARIANT, int MAXM, bool FULL, bool PAIR_MMA, class MU>
__device__ __forceinline__ double2 compute_chunk(const MU &mu, const DivBy &U, const ChunkOperands<MAXM> &r,
                                                 double (&acc)[3 + (MAXM > 0 ? MAXM : 1)])
{
    double2 xc;
    if (VARIANT == 0 && PAIR_MMA) xc = mma_pair<MAXM, FULL>(mu, r.x, r.lb, r.ub, r.s, r.g, r.Ga, r.Gb, acc);
    else if (VARIANT != 0) xc = ccsaq_pair<MAXM, FULL>(mu, U, r.x, r.lb, r.ub, r.s, r.g, r.Ga, r.Gb, acc);
    else {
        xc.x = mma_point<MAXM, FULL>(mu, r.x.x, r.lb.x, r.ub.x, r.s.x, r.g.x, r.Ga, acc);
        xc.y = mma_point<MAXM, FULL>(mu, r.x.y, r.lb.y, r.ub.y, r.s.y, r.g.y, r.Gb, acc);
    }
    return xc;
}

// the rest of a group whose first chunk (pair index p_first of this lane, `first`) is already on its way
template <int VARIANT, int MAXM, bool FULL, bool POL, bool PAIR_MMA, bool SB, class MU>
__device__ __forceinline__ void sweep_group_preloaded(const DualArgs &a, const MU &mu, const L2Policies &pol, bool store,
                                                      unsigned long long p_first, unsigned long long p_hi, ChunkOperands<MAXM> &r,
                                                      double (&acc)[3 + (MAXM > 0 ? MAXM : 1)])
{
    DivBy U;
    U.b = 1.0; U.r = 1.0; U.hb = 0x3ff00000; U.zero_ok = 1u;
    if (VARIANT != 0) U = prep_div(mu.u());                  // CCSAQ: every variable divides by the same u
    unsigned long long p = p_first;
    bool live = p < p_hi;
    while (live) {
        const double2 xc = compute_chunk<VARIANT, MAXM, FULL, PAIR_MMA>(mu, U, r, acc);
        if (store) st_stream(reinterpret_cast<double2 *>(a.xcur) + p, xc);
        p += kChunkPairs;
        live = p < p_hi;
        if (live) load_chunk<MAXM, FULL, POL, SB>(a, mu.m, pol, p, true, r);
    }
}

// group record = the 8 warp records added in warp order, dropped into the group's tagged slots
template <int NV>
__device__ __forceinline__ void put_group_record(const double *srec, double *grouptags, unsigned ngroups, unsigned gl,
                                                 unsigned long long tag, int lane)
{
    if (lane < NV) {
        double s = srec[lane];
#pragma unroll
        for (int w = 1; w < kGroupWarps; ++w) s = addx(s, srec[w * NV + lane]);
        slot_put(grouptags + 2ull * ((unsigned long long) lane * ngroups + gl), s, tag);
    }
}

template <int VARIANT, int MAXM, bool FULL, bool STORE, int BLOCK, int UNROLL, int MINB, bool SB>
__global__ void __launch_bounds__(BLOCK, MINB) dual_eval_kernel(const __grid_constant__ DualArgs a)
{
    constexpr int MR = MAXM > 0 ? MAXM : 1;
    constexpr int NV = 3 + MR;
    static_assert(BLOCK == 32 * kGroupWarps, "one group slot per CTA");
    if (blockIdx.x == gridDim.x - 1) {
        eval_folder<NV>(a, NV);
        return;
    }
    const int lane = threadIdx.x & 31;
    const int sub = threadIdx.x >> 5;
    const unsigned nslots = gridDim.x - 1;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;
    __shared__ double s_rec[2][kGroupWarps * NV];
    int parity = 0;
    for (unsigned gl = blockIdx.x; gl < ngroups; gl += nslots) {
        double acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[k] = 0.0;
        sweep_group<VARIANT, MAXM, FULL, UNROLL, SB>(a, a, STORE, gl, sub, lane, acc);   // multipliers = the parameter block itself

        // warp record -> shared memory; one CTA barrier per group; the record buffer is double-buffered across
        // iterations so the next group's writers can never overtake this group's reader.
        warp_fold<NV>(acc);
        double *srec = s_rec[parity];
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < NV; ++k) srec[sub * NV + k] = acc[k];
        }
        __syncthreads();
        parity ^= 1;
        if (sub == 0) put_group_record<NV>(srec, a.grouptags, ngroups, gl, a.tag, lane);
    }
}

// ---- the dual evaluation kernel, TMA-staged form -------------------------------------------------------------
// Same groups, same per-warp accumulators, same fold tree (=> same bits) as dual_eval_kernel; what changes is
// how the operands arrive.  A producer warp issues 1-D TMA bulk copies (cp.async.bulk + mbarrier
// complete_tx): one 4 KB chunk of each of the 5+m arrays per stage, STAGES stages deep, running ahead
// across group boundaries so the pipeline never drains.  The 8 consumer warps wait on the stage's "full"
// barrier, read their double2 lanes from shared memory, and release the stage on its "empty" barrier.
// No load ever occupies a consumer register before it is needed, so many more bytes are in flight per SM
// than the register form can hold at the same occupancy.
__device__ __forceinline__ unsigned smem_addr(const void *p) { return (unsigned) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
    unsigned ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void tma_bulk_load(void *smem_dst, const void *gmem_src, unsigned bytes, unsigned long long *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}

constexpr int kTmaBlock = 32 * (kGroupWarps + 1);        // 8 consumer warps + 1 producer warp
constexpr unsigned kChunkBytes = kChunkPairs * 16;       // 4 KB per array per stage
template <int VARIANT, int MAXM, bool STORE, int STAGES, int MINB>
__global__ void __launch_bounds__(kTmaBlock, MINB) dual_eval_tma_kernel(const __grid_constant__ DualArgs a)
{
    constexpr int MR = MAXM > 0 ? MAXM : 1;
    constexpr int NV = 3 + MR;
    constexpr int NARR = 5 + MAXM;                            // x lb ub sigma g + MAXM gradient rows
    extern __shared__ __align__(128) unsigned char s_raw[];
    double2 *s_tile = reinterpret_cast<double2 *>(s_raw);     // [STAGES][NARR][kChunkPairs]
    __shared__ unsigned long long s_full[STAGES], s_empty[STAGES];
    __shared__ double s_rec[2][kGroupWarps * NV];

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;
    const unsigned nslots = gridDim.x - 1;

    if (blockIdx.x == gridDim.x - 1) {                        // the folder CTA: its 8 first warps
        if (warp < kGroupWarps) eval_folder<NV>(a, NV);
        return;
    }

    if (threadIdx.x == 0) {
        for (int st = 0; st < STAGES; ++st) {
            mbar_init(&s_full[st], 1);                        // one arrive.expect_tx by the producer
            mbar_init(&s_empty[st], kGroupWarps);             // one arrive per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kGroupWarps) {
        // ---------------- producer ----------------
        if (lane == 0) {
            const double *src[NARR];
            src[0] = a.x; src[1] = a.lb; src[2] = a.ub; src[3] = a.sigma; src[4] = a.g;
#pragma unroll
            for (int i = 0; i < MAXM; ++i) src[5 + i] = a.G + (unsigned long long) i * a.ld;
            int st = 0;
            unsigned phase = 0;
            for (unsigned gl = blockIdx.x; gl < ngroups; gl += nslots) {
                unsigned long long p_lo, p_hi;
                group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + gl, &p_lo, &p_hi);
                for (unsigned long long p = p_lo; p < p_hi; p += kChunkPairs) {
                    mbar_wait(&s_empty[st], phase ^ 1u);      // passes at once on a fresh barrier
                    mbar_expect_tx(&s_full[st], NARR * kChunkBytes);
#pragma unroll
                    for (int k = 0; k < NARR; ++k)
                        tma_bulk_load(s_tile + ((size_t) st * NARR + k) * kChunkPairs, src[k] + 2 * p, kChunkBytes, &s_full[st]);
                    if (++st == STAGES) { st = 0; phase ^= 1u; }
                }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const int sub = warp;
    int st = 0;
    unsigned phase = 0;
    int parity = 0;
    for (unsigned gl = blockIdx.x; gl < ngroups; gl += nslots) {
        unsigned long long p_lo, p_hi;
        group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + gl, &p_lo, &p_hi);
        double acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[k] = 0.0;
        for (unsigned long long p = p_lo; p < p_hi; p += kChunkPairs) {
            mbar_wait(&s_full[st], phase);
            const double2 *t = s_tile + (size_t) st * NARR * kChunkPairs + sub * 32 + lane;
            const double2 vx = t[0], vlb = t[kChunkPairs], vub = t[2 * kChunkPairs], vs = t[3 * kChunkPairs],
                          vg = t[4 * kChunkPairs];
            double Ga[MR], Gb[MR];
#pragma unroll
            for (int i = 0; i < MR; ++i) {
                Ga[i] = 0.0; Gb[i] = 0.0;
                if (MAXM > 0) { const double2 g2 = t[(5 + i) * kChunkPairs]; Ga[i] = g2.x; Gb[i] = g2.y; }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&s_empty[st]);         // operands are in registers: release the stage
            if (++st == STAGES) { st = 0; phase ^= 1u; }
            double2 xc;
            if (VARIANT == 0) {
                xc.x = mma_point<MAXM, true>(a, vx.x, vlb.x, vub.x, vs.x, vg.x, Ga, acc);
                xc.y = mma_point<MAXM, true>(a, vx.y, vlb.y, vub.y, vs.y, vg.y, Gb, acc);
            } else {
                xc.x = ccsaq_point<MAXM, true>(a, vx.x, vlb.x, vub.x, vs.x, vg.x, Ga, acc);
                xc.y = ccsaq_point<MAXM, true>(a, vx.y, vlb.y, vub.y, vs.y, vg.y, Gb, acc);
            }
            if (STORE) st_stream(reinterpret_cast<double2 *>(a.xcur) + p + sub * 32 + lane, xc);
        }

        warp_fold<NV>(acc);
        double *srec = s_rec[parity];
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < NV; ++k) srec[sub * NV + k] = acc[k];
        }
        asm volatile("bar.sync 1, %0;" ::"r"(32 * kGroupWarps) : "memory");      // the 8 consumer warps only
        parity ^= 1;
        if (sub == 0) put_group_record<NV>(srec, a.grouptags, ngroups, gl, a.tag, lane);
    }
}

// ---- the dual evaluation kernel for any number of constraints (m > 16) ----------------------------------------
// The reference has no cap on m (mma.c:173; loops :101-129).  With more rows than registers can hold, one sweep step
// (one 512-variable chunk, two variables per thread) makes two passes over the m rows of the gradient block:
//   pass A  rows in blocks of 8 (eight 128-bit loads in flight per thread): u, v of mma.c:101-106 (v of
//           ccsa_quadratic.c:116-121) accumulated in row order, exactly the reference's chain;
//   then    the closed-form minimiser, clamps, and the three row-independent sums, as in the register-row kernels;
//   pass B  the same rows again -- they were read microseconds ago by this CTA, so they come from L1/L2, not from
//           HBM: HBM traffic stays (5 + m) * 8 bytes per variable -- for the g_i terms (mma.c:126-129,
//           ccsa_quadratic.c:139-140).
// Reduction of the g_i terms (m accumulators do not fit in registers either): per row and chunk, a lane adds its two
// terms, the warp reduces eight rows at a time with an exchange-and-halve butterfly (9 shuffles for 8 rows instead of
// 40), and lane 4r of the warp adds the row's chunk total to the warp's running row sum in shared memory -- chunks in
// index order.  Group record = the 8 warps' row sums in warp order; from there on the canonical fold tree.  The
// multipliers, penalties and the "constraint switched off" flags (MMA, NaN value) come from a device block (a.wide)
// staged in shared memory.  Deterministic, independent of the grid and of the number of ranks like every other path.
constexpr int kWideRows = 8;              // rows per block

// lane values t[0..8) of eight rows -> row r's warp total in lanes 4r .. 4r+3 (returned)
__device__ __forceinline__ double reduce8_rows(double (&t)[kWideRows], int lane)
{
    const bool b4 = (lane & 16) != 0, b3 = (lane & 8) != 0, b2 = (lane & 4) != 0;
    double q[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {         // xor 16: lanes with bit 4 clear keep rows 0-3, the others rows 4-7
        const double send = b4 ? t[j] : t[j + 4];
        const double keep = b4 ? t[j + 4] : t[j];
        q[j] = addx(keep, __shfl_xor_sync(0xffffffffu, send, 16));
    }
    double h[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {         // xor 8: of its four rows a lane keeps the lower (bit 3 clear) or upper pair
        const double send = b3 ? q[j] : q[j + 2];
        const double keep = b3 ? q[j + 2] : q[j];
        h[j] = addx(keep, __shfl_xor_sync(0xffffffffu, send, 8));
    }
    const double send = b2 ? h[0] : h[1]; // xor 4: one row left
    const double keep = b2 ? h[1] : h[0];
    double s = addx(keep, __shfl_xor_sync(0xffffffffu, send, 4));
    s = addx(s, __shfl_xor_sync(0xffffffffu, s, 2));
    s = addx(s, __shfl_xor_sync(0xffffffffu, s, 1));
    return s;                             // row 4*b4 + 2*b3 + b2 = lane / 4
}

template <int VARIANT, bool STORE>
__global__ void __launch_bounds__(kBlock, 2) dual_eval_wide_kernel(const __grid_constant__ DualArgs a)
{
    extern __shared__ __align__(16) double s_dyn[];           // y[m] | rhoc[m] | half_rhoc[m] | act[m] | wrow[8][mp]
    const int m = a.m;
    const int mp = (m + kWideRows - 1) / kWideRows * kWideRows;   // rows padded to whole blocks (padding rows: act = 0)
    double *s_y = s_dyn, *s_rhoc = s_dyn + mp, *s_hrhoc = s_dyn + 2 * mp, *s_act = s_dyn + 3 * mp, *s_wrow = s_dyn + 4 * mp;
    __shared__ double s_rec[kGroupWarps * 3];
    const int lane = threadIdx.x & 31;
    const int sub = threadIdx.x >> 5;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;
    if (blockIdx.x == gridDim.x - 1) {
        eval_folder<16>(a, 3 + m);
        return;
    }
    for (int i = threadIdx.x; i < mp; i += kBlock) {
        const bool in = i < m;
        s_y[i] = in ? a.wide[i] : 0.0;
        s_rhoc[i] = in ? a.wide[m + i] : 0.0;
        s_hrhoc[i] = in ? a.wide[2 * m + i] : 0.0;
        s_act[i] = in ? a.wide[3 * m + i] : 0.0;
    }
    __syncthreads();
    const unsigned nslots = gridDim.x - 1;
    const double2 *x2 = reinterpret_cast<const double2 *>(a.x);
    const double2 *lb2 = reinterpret_cast<const double2 *>(a.lb);
    const double2 *ub2 = reinterpret_cast<const double2 *>(a.ub);
    const double2 *s2v = reinterpret_cast<const double2 *>(a.sigma);
    const double2 *g2 = reinterpret_cast<const double2 *>(a.g);
    double *wrow = s_wrow + (size_t) sub * mp;                // this warp's running row sums over the group

    for (unsigned gl = blockIdx.x; gl < ngroups; gl += nslots) {
        for (int i = lane; i < mp; i += 32) wrow[i] = 0.0;
        __syncwarp();
        unsigned long long p_lo, p_hi;
        group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + gl, &p_lo, &p_hi);
        double acc[3] = {0.0, 0.0, 0.0};
        for (unsigned long long p = p_lo + sub * 32 + lane; p < p_hi; p += kChunkPairs) {
            const double2 vx = ld_stream(x2 + p), vlb = ld_stream(lb2 + p), vub = ld_stream(ub2 + p), vs = ld_stream(s2v + p),
                          vg = ld_stream(g2 + p);
            const double2 *Gp = reinterpret_cast<const double2 *>(a.G) + p;
            const unsigned long long ldp = a.ld / 2;          // row stride in double2
            // ---- pass A: u, v ----
            double ua = vg.x, ub_ = vg.y, va = 0.0, vb = 0.0;
            double agsa = 0.0, agsb = 0.0;
            if (VARIANT == 0) {
                agsa = mulx(fabs(vg.x), vs.x); agsb = mulx(fabs(vg.y), vs.y);
                va = addx(agsa, a.half_rho); vb = addx(agsb, a.half_rho);
            }
            for (int i0 = 0; i0 < mp; i0 += kWideRows) {
                double2 Gi[kWideRows];
#pragma unroll
                for (int r = 0; r < kWideRows; ++r) Gi[r] = i0 + r < m ? __ldg(Gp + (unsigned long long) (i0 + r) * ldp) : make_double2(0.0, 0.0);
#pragma unroll
                for (int r = 0; r < kWideRows; ++r) {
                    const int i = i0 + r;
                    if (VARIANT == 0) {
                        if (s_act[i] != 0.0) {
                            const double yi = s_y[i], hr = s_hrhoc[i];
                            ua = addx(ua, mulx(Gi[r].x, yi));
                            ub_ = addx(ub_, mulx(Gi[r].y, yi));
                            va = addx(va, mulx(addx(mulx(fabs(Gi[r].x), vs.x), hr), yi));
                            vb = addx(vb, mulx(addx(mulx(fabs(Gi[r].y), vs.y), hr), yi));
                        }
                    } else if (i < m) {
                        const double yi = s_y[i];
                        ua = addx(ua, mulx(Gi[r].x, yi));
                        ub_ = addx(ub_, mulx(Gi[r].y, yi));
                    }
                }
            }
            // ---- the minimiser and the row-independent sums (same expressions as mma_point / ccsaq_point) ----
            double2 xc = vx;
            double dxa = 0.0, dxb = 0.0;          // x*(y) - x
            double fa = 0.0, fb = 0.0;            // MMA: s2 * dx ("c"), CCSAQ: dx^2 / (2 s2) ("q")
            double da = 0.0, db = 0.0;            // MMA: dx^2 / (s2 - dx^2) numerator helper: dx2;  unused for CCSAQ
            double ia = 0.0, ib = 0.0;            // MMA: 1 / (s2 - dx^2)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const double x = h ? vx.y : vx.x, lb = h ? vlb.y : vlb.x, ub = h ? vub.y : vub.x, s = h ? vs.y : vs.x,
                             g = h ? vg.y : vg.x;
                if (s == 0) continue;                         // fixed variable: no contribution anywhere
                double xcj, dx;
                if (VARIANT == 0) {
                    double u = h ? ub_ : ua;
                    const double v = h ? vb : va, ag_s = h ? agsb : agsa;
                    const double s2 = mulx(s, s);
                    u = mulx(u, s2);
                    const double r = divx(u, mulx(v, s));
                    dx = divx(divx(u, v), subx(-1.0, __dsqrt_rn(fabs(subx(1.0, mulx(r, r))))));
                    xcj = addx(x, dx);
                    if (xcj > ub) xcj = ub; else if (xcj < lb) xcj = lb;
                    const double lim = mulx(0.9, s), hi = addx(x, lim), lo = subx(x, lim);
                    if (xcj > hi) xcj = hi; else if (xcj < lo) xcj = lo;
                    dx = subx(xcj, x);
                    const double dx2 = mulx(dx, dx);
                    const double dinv = divx(1.0, subx(s2, dx2));
                    acc[0] = addx(acc[0], mulx(addx(mulx(u, dx), mulx(v, dx2)), dinv));
                    const double c = mulx(s2, dx);
                    acc[1] = addx(acc[1], mulx(addx(mulx(g, c), mulx(addx(ag_s, a.half_rho), dx2)), dinv));
                    acc[2] = addx(acc[2], mulx(mulx(0.5, dx2), dinv));
                    if (h) { fb = c; db = dx2; ib = dinv; } else { fa = c; da = dx2; ia = dinv; }
                } else {
                    const double v = h ? ub_ : ua;
                    const double u = a.u_ccsaq;
                    const double s2 = mulx(s, s);
                    dx = divx(mulx(-s2, v), u);
                    if (fabs(dx) > s) dx = copysign(s, dx);
                    xcj = addx(x, dx);
                    if (xcj > ub) xcj = ub; else if (xcj < lb) xcj = lb;
                    dx = subx(xcj, x);
                    const double dx2 = mulx(dx, dx);
                    acc[0] = addx(acc[0], addx(mulx(v, dx), divx(mulx(mulx(0.5, u), dx2), s2)));
                    const double q = divx(mulx(0.5, dx2), s2);
                    acc[1] = addx(acc[1], addx(mulx(g, dx), mulx(a.rho, q)));
                    acc[2] = addx(acc[2], q);
                    if (h) fb = q; else fa = q;
                }
                if (h) { xc.y = xcj; dxb = dx; } else { xc.x = xcj; dxa = dx; }
            }
            if (STORE) st_stream(reinterpret_cast<double2 *>(a.xcur) + p, xc);
            const bool on_a = vs.x != 0, on_b = vs.y != 0;
            // ---- pass B: the g_i terms ----
            for (int i0 = 0; i0 < mp; i0 += kWideRows) {
                double2 Gi[kWideRows];
#pragma unroll
                for (int r = 0; r < kWideRows; ++r) Gi[r] = i0 + r < m ? __ldg(Gp + (unsigned long long) (i0 + r) * ldp) : make_double2(0.0, 0.0);
                double t[kWideRows];
#pragma unroll
                for (int r = 0; r < kWideRows; ++r) {
                    const int i = i0 + r;
                    double ta = 0.0, tb = 0.0;
                    if (VARIANT == 0) {
                        if (s_act[i] != 0.0) {
                            const double hr = s_hrhoc[i];
                            if (on_a) ta = mulx(addx(mulx(Gi[r].x, fa), mulx(addx(mulx(fabs(Gi[r].x), vs.x), hr), da)), ia);
                            if (on_b) tb = mulx(addx(mulx(Gi[r].y, fb), mulx(addx(mulx(fabs(Gi[r].y), vs.y), hr), db)), ib);
                        }
                    } else if (i < m) {
                        const double rc = s_rhoc[i];
                        if (on_a) ta = addx(mulx(Gi[r].x, dxa), mulx(rc, fa));
                        if (on_b) tb = addx(mulx(Gi[r].y, dxb), mulx(rc, fb));
                    }
                    t[r] = addx(ta, tb);
                }
                const double s = reduce8_rows(t, lane);
                if ((lane & 3) == 0) {
                    const int i = i0 + (lane >> 2);
                    wrow[i] = addx(wrow[i], s);
                }
            }
        }
        // ---- group record: sums 0..2 like the register-row kernels, sums 3.. from the warps' row sums ----
        warp_fold<3>(acc);
        if (lane == 0) { s_rec[sub * 3] = acc[0]; s_rec[sub * 3 + 1] = acc[1]; s_rec[sub * 3 + 2] = acc[2]; }
        __syncthreads();
        const unsigned long long tag = a.tag;
        for (int k = threadIdx.x; k < 3 + m; k += kBlock) {
            double s;
            if (k < 3) {
                s = s_rec[k];
                for (int w = 1; w < kGroupWarps; ++w) s = addx(s, s_rec[w * 3 + k]);
            } else {
                s = s_wrow[k - 3];
                for (int w = 1; w < kGroupWarps; ++w) s = addx(s, s_wrow[(size_t) w * mp + k - 3]);
            }
            slot_put(a.grouptags + 2ull * ((unsigned long long) k * ngroups + gl), s, tag);
        }
        __syncthreads();                          // the row sums are re-zeroed at the top of the next group
    }
}

// ---- the persistent dual-SOLVE kernel: one launch per dual solve ------------------------------------------
// (SURVEY.md 8(f)-1.)  The m-dimensional dual optimiser moves into the kernel: all CTAs stay resident
// (cooperative launch) and walk *generations*.  Generation g = one dual evaluation at the trial multipliers y_g.
//
//   sweeper CTAs (all but the last): claim groups from a monotonic counter (claim c -> generation
//     c / ngroups + 1, group c % ngroups), sweep them exactly like dual_eval_kernel (same warp records,
//     same group records => same bits) and drop each group record into its tagged slots.  A sweeper that runs
//     out of work in generation g claims a group of generation g + 1 and ISSUES ITS FIRST OPERAND LOADS before it
//     starts to poll for y_{g+1} (the loads do not depend on y): the serial part of a generation -- last record,
//     fold, exchange, optimiser step, publication -- overlaps with (5+m) x 4 KB x #CTAs of HBM traffic.
//   the folder CTA (the last one): fold_generation, then warp 0 exchanges the shard sums over the NVLink mailbox
//     when there are several ranks, feeds F and grad F to the WarpDualMachine held in ITS registers (lane i owns
//     multiplier i), and publishes y_{g+1} as tagged slots the sweepers poll (again no fence: a slot is valid iff
//     its tag is the awaited generation).
// Versus one launch per evaluation this removes launch latency, the PCIe result hop and the host turn-
// around from every evaluation; the host sees one launch and one result per dual solve.
//
// Timeline instrumentation (tools/trace_solve.py builds a separate library with -DNB200_TRACE; the product build
// contains none of it).  Per generation g, 16 counters at trace[16 g]: 0 published | 1 ~min / 2 max "CTA saw it" |
// 3 ~min / 4 max "group record stored" | 5 all shard sums in | 6 totals ready | 7 optimiser done | 8 sum / 9 count
// of per-group sweep times | TMA-staged form only: 10 ~min / 11 max "a CTA stored its last group record of g",
// 12 max / 13 ~min "a producer found its ring full of g's chunks while its consumers wait for g's multipliers".
// Row 0 holds the CTA start times.  All in %globaltimer nanoseconds.
#ifdef NB200_TRACE
constexpr int kTraceGens = 512;
#define NB_TR(...) __VA_ARGS__
#else
#define NB_TR(...)
#endif

// The dual optimiser of dual_mma.hpp (DualMachine: mma.c:145-452 with m' = 0 constraints, and its level-3 step
// mma.c:59-137), restated for one warp: lane i < m owns y_i, g_i, sigma_i, ...; the scalars are replicated in every
// lane and every lane executes the same scalar control flow.  Sums over i are taken in index order through shuffles,
// so every operation and its order are those of the host machine: the two produce the same bits
// (tests/test_dual_machine_gpu.py replays the reference's dual trajectories into both; test_gpu_parity.py::
// test_fused_solve_stop_rules_equal_host_driven compares whole runs).
// MAXM bounds m at compile time: the index-order sums over the multipliers are unrolled to MAXM trips with a predicate
// i < m, so that their shuffles are issued back to back instead of one per loop trip (they sit on the serial path of
// every generation).
template <int MAXM>
struct WarpDualMachine {
    double y, g, sigma, ycur, yprev, yprevprev, lo, hi;          // lane i: element i (lanes >= m: sigma = 0)
    double rho, fbase, fmin, fcur, fprev, gval, wval;
    unsigned k;
    long nevals;
    int awaiting_first, ret, m;
    DualStop st;

    __device__ __forceinline__ int start(int m_, double y0, double lo_, double hi_, const DualStop &stop, int lane)
    {
        m = m_;
        st = stop;
        nevals = 0;
        k = 0;
        const bool in = lane < m;
        y = in ? y0 : 0.0; lo = in ? lo_ : 0.0; hi = in ? hi_ : 0.0;
        const bool bad = in && (lo > hi || y < lo || y > hi);                        // optimize.c:547-551
        ret = __any_sync(0xffffffffu, bad) ? kRetInvalid : kRetSuccess;
        sigma = !in ? 0.0 : ((nl_isinf(hi) || nl_isinf(lo)) ? 1.0 : mulx(0.5, subx(hi, lo)));   // mma.c:202-210
        g = ycur = yprev = yprevprev = 0.0;
        rho = 1.0;
        fbase = fmin = fcur = fprev = gval = wval = 0.0;
        awaiting_first = 1;
        return ret;
    }

    __device__ __forceinline__ double trial() const { return awaiting_first ? y : ycur; }

    __device__ __forceinline__ bool limits_hit(bool time_up)
    {
        if (st.maxeval > 0 && nevals >= st.maxeval) ret = kRetMaxeval;
        else if (time_up) ret = kRetMaxtime;
        return ret != kRetSuccess;
    }
    __device__ __forceinline__ bool outer_top(bool time_up)          // mma.c:255-265
    {
        fprev = fcur;
        if (limits_hit(time_up)) return true;
        if (++k > 1) yprevprev = yprev;
        yprev = ycur;
        return false;
    }
    __device__ __forceinline__ bool x_converged(int lane) const     // stop.c:98-108, unit weights, uniform xtol_abs
    {
        const double d = fabs(subx(ycur, yprev)), a = fabs(ycur);
        double dn = 0.0, xn = 0.0;
#pragma unroll
        for (int i = 0; i < MAXM; ++i) {
            const double di = __shfl_sync(0xffffffffu, d, i), ai = __shfl_sync(0xffffffffu, a, i);
            if (i < m) { dn = addx(dn, di); xn = addx(xn, ai); }
        }
        if (dn < mulx(st.xtol_rel, xn)) return true;
        return !__any_sync(0xffffffffu, lane < m && d >= st.xtol_abs);
    }
    __device__ __forceinline__ bool outer_end(int lane)              // mma.c:418-446
    {
        if (rel_stop(fprev, fcur, st.ftol_rel, st.ftol_abs)) ret = kRetFtol;
        if (x_converged(lane)) ret = kRetXtol;
        if (ret != kRetSuccess) return true;
        rho = mulx(0.1, rho) > 1e-5 ? mulx(0.1, rho) : 1e-5;
        if (k > 1 && lane < m) {
            const double osc = mulx(subx(ycur, yprev), subx(yprev, yprevprev));
            double s = mulx(sigma, osc < 0 ? 0.7 : (osc > 0 ? 1.2 : 1.0));
            if (!nl_isinf(hi) && !nl_isinf(lo)) {
                const double top = mulx(10.0, subx(hi, lo)), bot = mulx(0.01, subx(hi, lo));
                s = s < top ? s : top;
                s = s > bot ? s : bot;
            }
            sigma = s > 0.0 ? s : 0.0;                    // sigma_min = 0
        }
        return false;
    }

    // Feed F(trial()) and this lane's gradient component; `time_up`: the (rank-agreed) time limit has expired.
    // Returns true when finished (code in ret, multipliers in y).
    __device__ __forceinline__ bool feed_pre(double F, double grad, bool time_up, int lane)
    {
        if (awaiting_first) {                            // mma.c:218
            awaiting_first = 0;
            g = grad; ycur = y;
            fbase = fmin = fcur = F;
            nevals = 1;
            return outer_top(time_up);
        }
        fcur = F;                                        // mma.c:297
        ++nevals;
        const bool inner_done = gval >= fcur;            // mma.c:304
        if (fcur < fmin) {                               // mma.c:334 with m' = 0: always "feasible"
            fbase = fmin = fcur;
            y = ycur; g = grad;
        }
        if (limits_hit(time_up)) return true;
        if (inner_done) {
            if (outer_end(lane)) return true;
            if (outer_top(time_up)) return true;
        } else if (fcur > gval) {                        // mma.c:403-404
            const double a = mulx(10.0, rho), b = mulx(1.1, addx(rho, divx(subx(fcur, gval), wval)));
            rho = a < b ? a : b;
        }
        return false;
    }

    // The MMA dual evaluation with zero constraints on the m dual variables (mma.c:59-137, m = 0): the next trial
    // point ycur and the approximant's gval / wval.
    __device__ __forceinline__ void step(int lane)
    {
        const double s = sigma;
        const bool has = lane < m && s != 0;
        double gt = 0.0, wt = 0.0;
        if (lane < m && s == 0) ycur = y;
        if (has) {
            double u = g;
            const double v = addx(mulx(fabs(g), s), mulx(0.5, rho));
            const double s2 = mulx(s, s);
            u = mulx(u, s2);
            const double r = divx(u, mulx(v, s));
            double dy = divx(divx(u, v), subx(-1.0, __dsqrt_rn(fabs(subx(1.0, mulx(r, r))))));
            double yc = addx(y, dy);
            if (yc > hi) yc = hi;
            else if (yc < lo) yc = lo;
            if (yc > addx(y, mulx(0.9, s))) yc = addx(y, mulx(0.9, s));
            else if (yc < subx(y, mulx(0.9, s))) yc = subx(y, mulx(0.9, s));
            ycur = yc;
            dy = subx(yc, y);
            const double dy2 = mulx(dy, dy), dinv = divx(1.0, subx(s2, dy2)), c = mulx(s2, dy);
            gt = mulx(addx(mulx(g, c), mulx(addx(mulx(fabs(g), s), mulx(0.5, rho)), dy2)), dinv);
            wt = mulx(mulx(0.5, dy2), dinv);
        }
        double gs = fbase, ws = 0.0;                      // mma.c:123-125: the terms added in index order
#pragma unroll
        for (int i = 0; i < MAXM; ++i) {
            const double gi = __shfl_sync(0xffffffffu, gt, i), wi = __shfl_sync(0xffffffffu, wt, i);
            const int hi_ = __shfl_sync(0xffffffffu, (int) has, i);
            if (i < m) if (hi_) { gs = addx(gs, gi); ws = addx(ws, wi); }
        }
        gval = gs;
        wval = ws;
    }
};

constexpr int kPubSlots = kMaxParamM + 2;     // y_i | u_ccsaq | flags
struct SolveState {                       // device global; the head is zeroed by the host before every launch
    unsigned long long claim;             // monotonic group-claim counter
    int done;                             // 1: leave
    int pad;
    double pub[2 * kPubSlots];            // tagged slots {value, tag}: trial multipliers of the generation in flight,
                                          // u = rho + sum rhoc_i y_i, and (as an integer) bit 0 = also store x*(y)
};

struct SolveArgs {
    DualArgs d;                           // arrays, geometry, workspace, exchange boxes (d.y: the warm start)
    SolveState *st;
    unsigned long long tag0;              // launch id << 40; generation g carries tag0 | g
    double fval;                          // objective value at x
    double cval[kMaxParamM];              // constraint values with switched-off ones zeroed (mma.c:78)
    double lo[kMaxParamM], hi[kMaxParamM];    // box of the multipliers
    DualStop stop;
    volatile double *res_host;            // mapped pinned: raw sums [24] | y [32] | nevals | ret | generations
    NB_TR(unsigned long long *trace;)
};
constexpr int kResY = 24, kResCounts = 24 + 32;

struct SharedMultipliers {                // what the point functions read in the solve kernel
    const double *y, *rhoc, *half_rhoc;   // y in shared memory; penalties from the parameter block
    double rho, half_rho, u_ccsaq;
    unsigned active;
    int m;
    __device__ __forceinline__ double u() const { return u_ccsaq; }
};

// The folder CTA's loop (kept out of line so that its registers do not weigh on the sweep loop).
// s_vs [8 x NV] (the shard sums of the generation in flight) and s_w [8 x 8 x NV] (per shard: the 8 fold-warp results)
// are provided by the caller: the TMA-staged kernel's folder CTA lends its (otherwise unused) stage ring.
// serp: the sweepers claim the groups of even generations in descending order (dual_solve_tma_kernel); the folder
// polls the shards of those generations in the same order.
template <int NV>
__device__ __noinline__ void solve_folder(const SolveArgs &sa, double *s_vs, double *s_w, void *mach_storage, bool serp = false)
{
    const DualArgs &a = sa.d;
    SolveState *st = sa.st;
    const int lane = threadIdx.x & 31;
    const int sub = threadIdx.x >> 5;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;
    __shared__ int s_exit;
    constexpr int MAXM = NV - 3;
    // The dual optimiser's state belongs to warp 0 and is needed for one short turn per generation.  It rests in shared memory
    // and is brought into registers only for that turn, so that it does not weigh on the poll-and-fold loop that all
    // eight warps run in between (at the 80-register budget of the 3-CTAs/SM kernels it used to be spilled there:
    // ~400 bytes of local-memory traffic on the serial path of every generation).
    WarpDualMachine<MAXM> *const s_mach = static_cast<WarpDualMachine<MAXM> *>(mach_storage);      // [32], shared memory of the caller
    __shared__ int s_final_pass;
    const unsigned long long t_start = nb_globaltimer();
    if (threadIdx.x == 0) { s_exit = 0; s_final_pass = 0; }
    if (sub == 0) {
        WarpDualMachine<MAXM> mach;
        const double y0 = lane < a.m ? a.y[lane] : 0.0, lo = lane < a.m ? sa.lo[lane] : 0.0, hi = lane < a.m ? sa.hi[lane] : 0.0;
        const int rc = mach.start(a.m, y0, lo, hi, sa.stop, lane);       // d.y carries the warm start
        if (rc != kRetSuccess) {          // start point outside the box: report, publish nothing
            if (lane == 0) {              // the whole count record: no evaluation, no generation
                sa.res_host[kResCounts] = 0.0;
                sa.res_host[kResCounts + 1] = (double) rc;
                sa.res_host[kResCounts + 2] = 0.0;
                __threadfence_system();
                *a.flag_host = a.seq;
                __threadfence_system();
                *reinterpret_cast<volatile int *>(&st->done) = 1;
                s_exit = 1;
            }
        } else {
            double u = a.rho;
#pragma unroll
            for (int i = 0; i < MAXM; ++i) {
                const double yi = __shfl_sync(0xffffffffu, mach.y, i);
                if (i < a.m) u = addx(u, mulx(a.rhoc[i], yi));
            }
            NB_TR(if (lane == 0) sa.trace[16] = nb_globaltimer();)
            if (lane < a.m) slot_put(st->pub + 2 * lane, mach.y, sa.tag0 | 1ull);
            if (lane == 0) {
                slot_put(st->pub + 2 * kMaxParamM, u, sa.tag0 | 1ull);
                slot_put(st->pub + 2 * (kMaxParamM + 1), __longlong_as_double(0ll), sa.tag0 | 1ull);
            }
        }
        s_mach[lane] = mach;
    }
    fold_init<NV>(s_w);
    if (s_exit) return;
    for (unsigned long long gen = 1;; ++gen) {
        const unsigned long long tag = sa.tag0 | gen;
        fold_generation<NV>(a.grouptags, ngroups, a.segs_per_vshard, a.local_vshards, tag, 0, NV, s_w, s_vs, serp && !(gen & 1));
        // ---- warp 0: totals (exchange if sharded), the dual optimiser's turn, publication ----
        if (sub == 0) {
            NB_TR(if (lane == 0 && gen < kTraceGens) sa.trace[16 * gen + 5] = nb_globaltimer();)
            WarpDualMachine<MAXM> mach = s_mach[lane];
            const int final_pass = s_final_pass;
            double total = 0.0;               // lane k < NV holds sum k
            int timed_out = 0;
            // the time limit: a rank-local clock test, made collective by the exchange (see box_exchange)
            int time_up = sa.stop.maxtime > 0 && (double) (nb_globaltimer() - t_start) * 1e-9 >= sa.stop.maxtime;
            if (a.box[0] == nullptr) {
                if (lane < NV) {
                    total = s_vs[lane];
                    for (unsigned v = 1; v < a.local_vshards; ++v) total = addx(total, s_vs[v * NV + lane]);
                }
            } else {
                total = box_exchange(a.box, a.rank, a.world, a.seq + gen, s_vs, NV, a.local_vshards,
                                     a.seg0 / a.segs_per_vshard, NV, lane, time_up ? 1.0 : 0.0, &time_up, &timed_out);     // one tag per generation
            }
            NB_TR(if (lane == 0 && gen < kTraceGens) sa.trace[16 * gen + 6] = nb_globaltimer();)
            // F and grad F from the sums, constants added in the reference's order (mma.c:75-78, :135)
            int finished = 0, next_final = 0;
            if (!final_pass) {
                const double yt = mach.trial();
                const double cv = lane < a.m ? sa.cval[lane] : 0.0;
                const double gsum = __shfl_sync(0xffffffffu, total, (lane + 3) & 31);      // lane i < m: sum 3 + i
                const double grad = lane < a.m ? -addx(cv, gsum) : 0.0;                     // -g_i(y)
                double val = sa.fval;
#pragma unroll
                for (int i = 0; i < MAXM; ++i) {
                    const double yi = __shfl_sync(0xffffffffu, yt, i), ci = __shfl_sync(0xffffffffu, cv, i);
                    if (i < a.m) val = addx(val, mulx(yi, ci));
                }
                val = addx(val, __shfl_sync(0xffffffffu, total, 0));
                finished = timed_out ? 1 : (mach.feed_pre(-val, grad, time_up != 0, lane) ? 1 : 0);
                if (timed_out) mach.ret = kRetFailure;
                if (!finished) mach.step(lane);
                if (finished && !timed_out) next_final = 1;          // one more pass at the solution, storing x*(y)
            }
            NB_TR(if (lane == 0 && gen < kTraceGens) sa.trace[16 * gen + 7] = nb_globaltimer();)
            if (final_pass || timed_out) {
                // publish the result of the solve: raw sums of the final pass, multipliers, counts
                if (lane < NV) sa.res_host[lane] = total;
                if (lane < a.m) sa.res_host[kResY + lane] = mach.y;
                if (lane == 0) {
                    sa.res_host[kResCounts] = (double) mach.nevals;
                    sa.res_host[kResCounts + 1] = (double) mach.ret;
                    sa.res_host[kResCounts + 2] = (double) gen;
                }
                __threadfence_system();
                __syncwarp();
                if (lane == 0) {
                    *a.flag_host = a.seq;
                    __threadfence_system();
                    *reinterpret_cast<volatile int *>(&st->done) = 1;
                    s_exit = 1;
                }
            } else {
                // publish generation gen + 1
                const double trial = next_final ? mach.y : mach.ycur;
                const unsigned long long ntag = sa.tag0 | (gen + 1);
                double u = a.rho;
#pragma unroll
                for (int i = 0; i < MAXM; ++i) {
                    const double ti = __shfl_sync(0xffffffffu, trial, i);
                    if (i < a.m) u = addx(u, mulx(a.rhoc[i], ti));
                }
                NB_TR(if (lane == 0 && gen + 1 < kTraceGens) sa.trace[16 * (gen + 1)] = nb_globaltimer();)
                if (lane < a.m) slot_put(st->pub + 2 * lane, trial, ntag);
                if (lane == 0) {
                    slot_put(st->pub + 2 * kMaxParamM, u, ntag);
                    slot_put(st->pub + 2 * (kMaxParamM + 1), __longlong_as_double((long long) next_final), ntag);
                }
                if (lane == 0) s_final_pass = next_final;
                s_mach[lane] = mach;
            }
        }
        fold_barrier();
        if (s_exit) return;
    }
}

template <int VARIANT, int MAXM, bool FULL, bool POL, int BLOCK, int MINB, bool SB>
__global__ void __launch_bounds__(BLOCK, MINB) dual_solve_kernel(const __grid_constant__ SolveArgs sa)
{
    constexpr int MR = MAXM > 0 ? MAXM : 1;
    constexpr int NV = 3 + MR;
    static_assert(BLOCK == 32 * kGroupWarps, "one group slot per CTA");
    static_assert(kGroupWarps == kVirtualShards, "the folder CTA gives one warp to each virtual shard");
    if (blockIdx.x == gridDim.x - 1) {
        __shared__ double s_vs[kVirtualShards * NV];
        __shared__ double s_w[kVirtualShards * kGroupWarps * NV];
        __shared__ __align__(16) unsigned char s_mach[32 * sizeof(WarpDualMachine<NV - 3>)];
        solve_folder<NV>(sa, s_vs, s_w, s_mach);
        return;
    }
    const DualArgs &a = sa.d;
    SolveState *st = sa.st;
    const int lane = threadIdx.x & 31;
    const int sub = threadIdx.x >> 5;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;
    __shared__ double s_rec[2][kGroupWarps * NV];
    __shared__ double s_y[kMaxParamM];
    __shared__ double s_u;
    __shared__ int s_store, s_exit;
    __shared__ unsigned long long s_claim[2];

    // ================================ sweeper CTAs ================================
    unsigned long long next_c = 0;
    if (threadIdx.x == 0) { s_exit = 0; s_store = 0; s_claim[0] = atomicAdd(&st->claim, 1ull); }
    NB_TR(if (threadIdx.x == 0) { const unsigned long long t = nb_globaltimer(); atomicMax(&sa.trace[1], ~t); atomicMax(&sa.trace[2], t); })
    __syncthreads();

    L2Policies pol;
    pol.init(a.l2_keep);

    int parity = 0;
    unsigned long long my_gen = 0;        // generation whose multipliers are in s_y
    for (int it = 0;; ++it) {
        const unsigned long long c = s_claim[it & 1];
        const unsigned long long want = c / ngroups + 1;
        const unsigned gl = (unsigned) (c % ngroups);
        // the first chunk's operands are requested before anything else: they do not depend on the multipliers
        unsigned long long p_lo, p_hi;
        group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + gl, &p_lo, &p_hi);
        const unsigned long long p_first = p_lo + sub * 32 + lane;
        ChunkOperands<MAXM> first;
        load_chunk<MAXM, FULL, POL, SB>(a, a.m, pol, p_first, p_first < p_hi, first);
        // wait until generation `want` is published (or the solve has finished); refresh the multipliers
        if (want != my_gen) {
            if (sub == 0) {                   // warp 0 polls, warp-uniformly: lane i < m: y_i, lane m: u, the others: flags
                const int slot = lane < a.m ? lane : (lane == a.m ? kMaxParamM : kMaxParamM + 1);
                const unsigned long long tag = sa.tag0 | want;
                double v;
                int ex = 0;
                unsigned spins = 0;
                for (;;) {
                    if (__all_sync(0xffffffffu, slot_get(st->pub + 2 * slot, tag, &v))) break;
                    if ((++spins & 7u) == 0u && __any_sync(0xffffffffu, ld_gpu_s32(&st->done))) {
                        ex = !__all_sync(0xffffffffu, slot_get(st->pub + 2 * slot, tag, &v));     // published before done was raised?
                        break;
                    }
                    __nanosleep(20);
                }
                if (ex) s_exit = 1;
                else if (lane < a.m) s_y[lane] = v;
                else if (lane == a.m) s_u = v;
                else if (lane == a.m + 1) s_store = (int) (__double_as_longlong(v) & 1ll);
            }
            __syncthreads();
            if (s_exit) return;
            NB_TR(if (threadIdx.x == 0 && want < kTraceGens) { const unsigned long long t = nb_globaltimer();
                      atomicMax(&sa.trace[16 * want + 1], ~t); atomicMax(&sa.trace[16 * want + 2], t); })
            my_gen = want;
        }
        // claim the next group now; the result is parked in a register until the sweep is over
        if (threadIdx.x == 0) next_c = atomicAdd(&st->claim, 1ull);

        SharedMultipliers mu;
        mu.y = s_y; mu.rhoc = a.rhoc; mu.half_rhoc = a.half_rhoc; mu.u_ccsaq = s_u;
        mu.rho = a.rho; mu.half_rho = a.half_rho;
        mu.active = a.active; mu.m = a.m;
        double acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[k] = 0.0;
        NB_TR(const unsigned long long tr_s0 = nb_globaltimer();)
        // (the 128-register instantiations, MINB <= 2, have room for the MMA pair form with 4 rows)
        sweep_group_preloaded<VARIANT, MAXM, FULL, POL, kPairMMA<MAXM> || (MINB <= 2 && MAXM <= 4), SB>(a, mu, pol, s_store != 0, p_first, p_hi, first, acc);

        warp_fold<NV>(acc);
        double *srec = s_rec[parity];
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < NV; ++k) srec[sub * NV + k] = acc[k];
        }
        if (threadIdx.x == 0) s_claim[(it + 1) & 1] = next_c;
        __syncthreads();
        parity ^= 1;
        if (sub == 0) put_group_record<NV>(srec, a.grouptags, ngroups, gl, sa.tag0 | my_gen, lane);
        NB_TR(if (sub == 0 && lane == 0 && my_gen < kTraceGens) { const unsigned long long t = nb_globaltimer(); unsigned long long *r = sa.trace + 16 * my_gen;
                  atomicMax(r + 3, ~t); atomicMax(r + 4, t); atomicAdd(r + 8, t - tr_s0); atomicAdd(r + 9, 1ull); })
    }
}

// ---- the persistent dual-solve kernel with a per-thread asynchronous operand pipeline ---------------------------------
// The register form above walks a group one chunk at a time: request (5+m) x 16 bytes per thread, wait for them, compute,
// next chunk.  All resident warps of an SM do this in step, so the load latency and the arithmetic of a chunk add up
// instead of overlapping (at the 8-GPU shard of n = 1e7 a generation is ~5 such steps per CTA: latency-bound, not
// HBM-bound).  Here every thread copies ITS OWN 16 bytes of each operand array of the chunks
// ahead with cp.async (LDGSTS: global -> shared without passing through registers) into its private column of a ring
// of STAGES shared-memory stages, and reads the stage back (LDS.128) when it gets there.  A thread only ever reads what
// it copied itself, so the ring needs no barrier, no mbarrier and no producer warp (the TMA-staged form below has all
// three and measured slower than the register form); the only synchronisation is cp.async.wait_group on the thread's
// own copies.  The prefetch cursor runs ahead of the arithmetic across chunk, GROUP and GENERATION boundaries: the
// operands do not depend on the multipliers, so while the folder CTA folds, exchanges, steps the dual optimiser and
// publishes y_{g+1}, the first STAGES chunks of every sweeper's next group are already on their way.
// Same lanes, same per-warp accumulators, same fold tree as every other kernel here: the same bits.
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int VARIANT, int MAXM, bool FULL, int STAGES, int MINB>
__global__ void __launch_bounds__(kBlock, MINB) dual_solve_async_kernel(const __grid_constant__ SolveArgs sa)
{
    constexpr int MR = MAXM > 0 ? MAXM : 1;
    constexpr int NV = 3 + MR;
    constexpr int NARR = 5 + MAXM;
    static_assert(MAXM >= 1 && STAGES >= 2 && STAGES <= 4, "ring of 2..4 stages");
    extern __shared__ __align__(16) unsigned char s_ring[];    // [STAGES][NARR][kBlock] double2: thread t owns column t
    if (blockIdx.x == gridDim.x - 1) {                          // the folder CTA: its ring holds the fold scratch
        double *scratch = reinterpret_cast<double *>(s_ring);
        constexpr size_t kFoldDoubles = (size_t) kVirtualShards * NV + (size_t) kVirtualShards * kGroupWarps * NV;
        static_assert((size_t) STAGES * NARR * kChunkBytes >= kFoldDoubles * sizeof(double) + 32 * sizeof(WarpDualMachine<NV - 3>) + 16, "fold scratch fits the ring");
        solve_folder<NV>(sa, scratch, scratch + kVirtualShards * NV, scratch + ((kFoldDoubles + 1) & ~(size_t) 1));
        return;
    }
    const DualArgs &a = sa.d;
    SolveState *st = sa.st;
    const int lane = threadIdx.x & 31;
    const int sub = threadIdx.x >> 5;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;
    __shared__ double s_rec[2][kGroupWarps * NV];
    __shared__ double s_y[kMaxParamM];
    __shared__ double s_u;
    __shared__ int s_store, s_exit;
    __shared__ volatile unsigned long long s_clm[4];            // claim of the CTA's group number `it` at [it & 3] ...
    __shared__ volatile int s_clm_it[4];                        // ... valid iff this says `it`
    double2 *const col = reinterpret_cast<double2 *>(s_ring) + threadIdx.x;      // element (stage s, array k): col[(s * NARR + k) * kBlock]

    const double *src[NARR];
    src[0] = a.x; src[1] = a.lb; src[2] = a.ub; src[3] = a.sigma; src[4] = a.g;
#pragma unroll
    for (int i = 0; i < MAXM; ++i) src[5 + i] = a.G + (unsigned long long) i * a.ld;

    unsigned long long next_c = 0;
    if (threadIdx.x < 4) s_clm_it[threadIdx.x] = -1;
    __syncthreads();
    if (threadIdx.x == 0) { s_exit = 0; s_store = 0; s_clm[0] = atomicAdd(&st->claim, 1ull); s_clm_it[0] = 0; }
    NB_TR(if (threadIdx.x == 0) { const unsigned long long t = nb_globaltimer(); atomicMax(&sa.trace[1], ~t); atomicMax(&sa.trace[2], t); })
    __syncthreads();

    // the prefetch cursor: the next chunk to request is pair pf_p (this lane's) of the CTA's group number pf_it
    unsigned issued = 0, consumed = 0;
    int pf_it = -1;
    unsigned long long pf_p = 0, pf_hi = 0;
    auto pump = [&]() {
        while (issued - consumed < (unsigned) STAGES) {
            if (pf_p >= pf_hi) {                                // this group is fully requested: move on to the next claim, if known
                const int nit = pf_it + 1;
                if (s_clm_it[nit & 3] != nit) break;
                const unsigned long long c = s_clm[nit & 3];
                unsigned long long lo, hi;
                group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + (unsigned) (c % ngroups), &lo, &hi);
                pf_it = nit;
                pf_p = lo + sub * 32 + lane;
                pf_hi = hi;
                continue;
            }
            double2 *dst = col + (size_t) (issued % STAGES) * NARR * kBlock;
#pragma unroll
            for (int k = 0; k < NARR; ++k)
                if (k < 5 || FULL || k - 5 < a.m) cp_async16(dst + (size_t) k * kBlock, reinterpret_cast<const double2 *>(src[k]) + pf_p);
            cp_async_commit();
            ++issued;
            pf_p += kChunkPairs;
        }
    };

    int parity = 0;
    unsigned long long my_gen = 0;        // generation whose multipliers are in s_y
    for (int it = 0;; ++it) {
        const unsigned long long c = s_clm[it & 3];
        const unsigned long long want = c / ngroups + 1;
        const unsigned gl = (unsigned) (c % ngroups);
        unsigned long long p_lo, p_hi;
        group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + gl, &p_lo, &p_hi);
        pump();                               // the head of this group is requested before we look for the multipliers
        if (want != my_gen) {
            if (sub == 0) {                   // warp 0 polls, warp-uniformly: lane i < m: y_i, lane m: u, the others: flags
                const int slot = lane < a.m ? lane : (lane == a.m ? kMaxParamM : kMaxParamM + 1);
                const unsigned long long tag = sa.tag0 | want;
                double v;
                int ex = 0;
                unsigned spins = 0;
                for (;;) {
                    if (__all_sync(0xffffffffu, slot_get(st->pub + 2 * slot, tag, &v))) break;
                    if ((++spins & 7u) == 0u && __any_sync(0xffffffffu, ld_gpu_s32(&st->done))) {
                        ex = !__all_sync(0xffffffffu, slot_get(st->pub + 2 * slot, tag, &v));     // published before done was raised?
                        break;
                    }
                    __nanosleep(20);
                }
                if (ex) s_exit = 1;
                else if (lane < a.m) s_y[lane] = v;
                else if (lane == a.m) s_u = v;
                else if (lane == a.m + 1) s_store = (int) (__double_as_longlong(v) & 1ll);
            }
            __syncthreads();
            if (s_exit) {
                cp_async_wait<0>();           // a CTA must not retire with copies into its shared memory in flight
                return;
            }
            NB_TR(if (threadIdx.x == 0 && want < kTraceGens) { const unsigned long long t = nb_globaltimer();
                      atomicMax(&sa.trace[16 * want + 1], ~t); atomicMax(&sa.trace[16 * want + 2], t); })
            my_gen = want;
        }
        // claim the next group now; thread 0 publishes it to the CTA after its first chunk (the atomic's latency hides
        // behind that chunk's arithmetic), so that the cursors can cross into the next group while this one is computed
        if (threadIdx.x == 0) next_c = atomicAdd(&st->claim, 1ull);
        bool claim_pending = threadIdx.x == 0;

        SharedMultipliers mu;
        mu.y = s_y; mu.rhoc = a.rhoc; mu.half_rhoc = a.half_rhoc; mu.u_ccsaq = s_u;
        mu.rho = a.rho; mu.half_rho = a.half_rho;
        mu.active = a.active; mu.m = a.m;
        DivBy U;
        U.b = 1.0; U.r = 1.0; U.hb = 0x3ff00000; U.zero_ok = 1u;
        if (VARIANT != 0) U = prep_div(mu.u());
        const bool store = s_store != 0;
        double acc[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) acc[k] = 0.0;
        NB_TR(const unsigned long long tr_s0 = nb_globaltimer();)
        for (unsigned long long p = p_lo + sub * 32 + lane; p < p_hi; p += kChunkPairs) {
            // this chunk is the oldest outstanding copy group of the thread: wait until at most the newer ones are pending
            const unsigned newer = issued - consumed - 1u;
            if (newer == 0u) cp_async_wait<0>();
            else if (newer == 1u) cp_async_wait<1>();
            else if (newer == 2u) cp_async_wait<2>();
            else cp_async_wait<3>();
            const double2 *t = col + (size_t) (consumed % STAGES) * NARR * kBlock;
            ChunkOperands<MAXM> r;
            r.x = t[0]; r.lb = t[kBlock]; r.ub = t[2 * kBlock]; r.s = t[3 * kBlock]; r.g = t[4 * kBlock];
#pragma unroll
            for (int i = 0; i < MR; ++i) {
                r.Ga[i] = 0.0; r.Gb[i] = 0.0;
                if (FULL || i < a.m) { const double2 g2 = t[(5 + i) * kBlock]; r.Ga[i] = g2.x; r.Gb[i] = g2.y; }
            }
            const double2 xc = compute_chunk<VARIANT, MAXM, FULL, (MINB <= 2 && MAXM <= 4) || kPairMMA<MAXM>>(mu, U, r, acc);
            if (store) st_stream(reinterpret_cast<double2 *>(a.xcur) + p, xc);
            ++consumed;
            if (claim_pending) {
                s_clm[(it + 1) & 3] = next_c;
                __threadfence_block();
                s_clm_it[(it + 1) & 3] = it + 1;
                claim_pending = false;
            }
            pump();
        }

        warp_fold<NV>(acc);
        double *srec = s_rec[parity];
        if (lane == 0) {
#pragma unroll
            for (int k = 0; k < NV; ++k) srec[sub * NV + k] = acc[k];
        }
        if (claim_pending) {                  // an empty group
            s_clm[(it + 1) & 3] = next_c;
            __threadfence_block();
            s_clm_it[(it + 1) & 3] = it + 1;
        }
        __syncthreads();
        parity ^= 1;
        if (sub == 0) put_group_record<NV>(srec, a.grouptags, ngroups, gl, sa.tag0 | my_gen, lane);
        NB_TR(if (sub == 0 && lane == 0 && my_gen < kTraceGens) { const unsigned long long t = nb_globaltimer(); unsigned long long *r = sa.trace + 16 * my_gen;
                  atomicMax(r + 3, ~t); atomicMax(r + 4, t); atomicAdd(r + 8, t - tr_s0); atomicAdd(r + 9, 1ull); })
    }
}

// ---- the persistent dual-solve kernel, TMA-staged form --------------------------------------------------------
// For small shards (several GPUs, or mid-size n) a generation is LATENCY-bound in the register form: a sweeper CTA walks
// its few chunks one after the other, each step a dependent load -> compute, and nothing is in flight while it waits
// for the next multipliers.  Here a producer warp feeds a ring of STAGES shared-memory stages with 1-D TMA bulk copies
// (one 4 KB chunk of each of the 5+m operand arrays per stage).  The operands do not depend on the multipliers, so the
// producer simply runs ahead: across chunk, group AND generation boundaries.  While the folder CTA folds, exchanges,
// steps the dual optimiser and publishes y_{g+1}, every sweeper's ring fills with the first chunks of generation g + 1;
// when y arrives the consumers start from shared memory and the producer keeps STAGES chunks in flight behind them.
//   producer (warp 8, one thread): claims groups from the same monotonic counter as the register form (claim c ->
//     generation c / ngroups + 1, group c % ngroups, counted down on even generations), and for every chunk waits for a free stage, writes the stage's
//     metadata {generation, group, first/last chunk, pair offset}, arms the "full" barrier and issues the bulk loads.
//   consumers (warps 0-7): follow the stage metadata -- first chunk of a group in a new generation: wait for that
//     generation's multipliers (warp 0 polls the tagged slots, as in the register form); every chunk: operands from
//     shared memory to registers, release the stage, evaluate; last chunk of a group: warp records -> group record ->
//     tagged slots.  Same lanes, same per-warp accumulators, same fold tree: the same bits as every other kernel here.
//   leaving: when the solve is over the consumers stop the producer and wait for the copies it has already issued
//     (a CTA must not retire with bulk copies into its shared memory in flight).
// BM, which operands a stage holds:
//   kBoundArrays:  5 + m arrays {x, lb, ub, sigma, g, G_0..}
//   kScalarBounds (uniform bounds, as SB in sweep_group): 3 + m arrays {x, sigma, g, G_0..}; no lb / ub copies are issued
//     and the consumers hand make_double2(lb_u, lb_u) / make_double2(ub_u, ub_u) to the unchanged closed forms
//   kSigmaIndex (uniform bounds and the sigma index is valid, sigma_palette.hpp): 2 + m arrays {x, g, G_0..} and the
//     chunk's 512 16-bit sigma indices (1 KB); the consumers look sigma up in the palette and hand the closed forms the
//     same double2 as the fp64 array would have given.
enum : int { kBoundArrays = 0, kScalarBounds = 1, kSigmaIndex = 2 };
constexpr unsigned kIdxChunkBytes = 2 * 2 * kChunkPairs;
struct StageMeta {
    unsigned long long gen;       // generation the chunk belongs to
    unsigned long long p;         // pair offset of the chunk
    unsigned gl;                  // local group
    unsigned flags;               // 1: first chunk of its group, 2: last chunk, 4: empty group (no data in the stage)
};

__device__ __forceinline__ bool mbar_test(unsigned long long *bar, unsigned parity)
{
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
    return ok != 0;
}

template <int VARIANT, int MAXM, int STAGES, int MINB, int BM>
__global__ void __launch_bounds__(kTmaBlock, MINB) dual_solve_tma_kernel(const __grid_constant__ SolveArgs sa)
{
    constexpr int MR = MAXM > 0 ? MAXM : 1;
    constexpr int NV = 3 + MR;
    constexpr int NB = BM == kBoundArrays ? 2 : 0;           // bound arrays in a stage
    constexpr bool SIDX = BM == kSigmaIndex;
    constexpr int KG = SIDX ? 1 + NB : 2 + NB;                // tile of grad f; sigma (fp64) is tile 1 + NB
    constexpr int NARR = KG + 1 + MAXM;                       // fp64 tiles in a stage
    static_assert(MAXM >= 1, "the solve kernels need at least one constraint");
    extern __shared__ __align__(128) unsigned char s_raw[];
    double2 *s_tile = reinterpret_cast<double2 *>(s_raw);     // [STAGES][NARR][kChunkPairs]
    const unsigned *s_idx = reinterpret_cast<const unsigned *>(s_raw + (size_t) STAGES * NARR * kChunkBytes);   // [STAGES][kChunkPairs] (SIDX)
    __shared__ unsigned long long s_full[STAGES], s_empty[STAGES];
    __shared__ StageMeta s_meta[STAGES];
    __shared__ double s_rec[2][kGroupWarps * NV];
    __shared__ double s_y[kMaxParamM];
    __shared__ double s_u;
    __shared__ int s_store, s_exit;
    __shared__ volatile int s_stop, s_prod_done;
    __shared__ volatile unsigned long long s_issued;
    NB_TR(__shared__ volatile unsigned long long s_park_gen;)   // generation whose multipliers warp 0 is polling for, else 0

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    if (blockIdx.x == gridDim.x - 1) {                        // the folder CTA: its 8 first warps; its stage ring holds the fold scratch
        double *scratch = reinterpret_cast<double *>(s_raw);
        static_assert((size_t) STAGES * NARR * kChunkBytes >= (size_t) (kVirtualShards * NV + kVirtualShards * kGroupWarps * NV) * sizeof(double), "fold scratch fits the ring");
        constexpr size_t kFoldDoubles = (size_t) kVirtualShards * NV + (size_t) kVirtualShards * kGroupWarps * NV;
        static_assert((size_t) STAGES * NARR * kChunkBytes >= kFoldDoubles * sizeof(double) + 32 * sizeof(WarpDualMachine<NV - 3>) + 16, "fold scratch + optimiser state fit the ring");
        if (warp < kGroupWarps) solve_folder<NV>(sa, scratch, scratch + kVirtualShards * NV, scratch + ((kFoldDoubles + 1) & ~(size_t) 1), true);
        return;
    }
    const DualArgs &a = sa.d;
    SolveState *st_g = sa.st;
    const unsigned ngroups = a.segs_per_vshard * a.local_vshards;

    if (threadIdx.x == 0) {
        for (int st = 0; st < STAGES; ++st) {
            mbar_init(&s_full[st], 1);
            mbar_init(&s_empty[st], kGroupWarps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        s_exit = 0; s_store = 0; s_stop = 0; s_prod_done = 0; s_issued = 0ull; NB_TR(s_park_gen = 0ull;)
    }
    __syncthreads();

    if (warp == kGroupWarps) {
        // ---------------- producer ----------------
        if (lane == 0) {
            const double *src[NARR];
            src[0] = a.x;
            if (NB) { src[1] = a.lb; src[2] = a.ub; }
            if (!SIDX) src[1 + NB] = a.sigma;
            src[KG] = a.g;
#pragma unroll
            for (int i = 0; i < MAXM; ++i) src[KG + 1 + i] = a.G + (unsigned long long) i * a.ld;
            int st = 0;
            unsigned phase = 0;
            unsigned long long issued = 0;
            bool stop = false;
            while (!stop) {
                const unsigned long long c = atomicAdd(&st_g->claim, 1ull);
                const unsigned long long gen = c / ngroups + 1;
                // serpentine: even generations take the groups in descending order, so that a generation starts on the
                // groups the previous one read last, which are still in the L2 (the group records, and so the sums, do
                // not depend on the order in which the groups are swept)
                const unsigned gl = (gen & 1) ? (unsigned) (c % ngroups) : ngroups - 1u - (unsigned) (c % ngroups);
                unsigned long long p_lo, p_hi;
                group_pairs(a.nchunks, a.nseg_total, a.chunk0, a.seg0 + gl, &p_lo, &p_hi);
                const bool empty = p_lo == p_hi;
                for (unsigned long long p = p_lo; p < p_hi || (empty && p == p_lo); p += kChunkPairs) {
                    NB_TR(bool tr_parked = false;)
                    while (!mbar_test(&s_empty[st], phase ^ 1u)) {        // a fresh barrier passes at once
                        if (s_stop) { stop = true; break; }
                        NB_TR(if (!tr_parked && s_park_gen == gen && gen < kTraceGens) {
                                  tr_parked = true; const unsigned long long t = nb_globaltimer();
                                  atomicMax(&sa.trace[16 * gen + 12], t); atomicMax(&sa.trace[16 * gen + 13], ~t); })
                    }
                    if (stop) break;
                    StageMeta mt;
                    mt.gen = gen; mt.p = p; mt.gl = gl;
                    mt.flags = (p == p_lo ? 1u : 0u) | ((empty || p + kChunkPairs >= p_hi) ? 2u : 0u) | (empty ? 4u : 0u);
                    s_meta[st] = mt;
                    if (empty) {
                        mbar_arrive(&s_full[st]);                         // no bytes: the phase completes on this arrival
                    } else {
                        mbar_expect_tx(&s_full[st], NARR * kChunkBytes + (SIDX ? kIdxChunkBytes : 0u));
#pragma unroll
                        for (int k = 0; k < NARR; ++k)
                            tma_bulk_load(s_tile + ((size_t) st * NARR + k) * kChunkPairs, src[k] + 2 * p, kChunkBytes, &s_full[st]);
                        if (SIDX)
                            tma_bulk_load((void *) (s_idx + (size_t) st * kChunkPairs), a.sidx + 2 * p, kIdxChunkBytes, &s_full[st]);
                    }
                    s_issued = ++issued;
                    if (++st == STAGES) { st = 0; phase ^= 1u; }
                    if (empty) break;
                }
            }
            __threadfence_block();
            s_prod_done = 1;
        }
        return;
    }

    // ---------------- consumers ----------------
    const int sub = warp;
    int st = 0;
    unsigned phase = 0;
    int parity = 0;
    unsigned long long my_gen = 0, consumed = 0;
    SharedMultipliers mu;
    mu.y = s_y; mu.rhoc = a.rhoc; mu.half_rhoc = a.half_rhoc; mu.u_ccsaq = 0.0;
    mu.rho = a.rho; mu.half_rho = a.half_rho;
    mu.active = a.active; mu.m = a.m;
    double acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = 0.0;
    bool store = false;
    NB_TR(unsigned long long tr_s0 = 0, tr_last = 0;)       // warp 0: start of the group in flight, time of the last record
    for (;;) {
        mbar_wait(&s_full[st], phase);                        // the stage's bytes and its metadata are visible
        const StageMeta mt = s_meta[st];
        if (mt.flags & 1u) {
            if (mt.gen != my_gen) {
                // wait until generation mt.gen is published (or the solve has finished); refresh the multipliers
                if (sub == 0) {
                    const int slot = lane < a.m ? lane : (lane == a.m ? kMaxParamM : kMaxParamM + 1);
                    const unsigned long long tag = sa.tag0 | mt.gen;
                    double v;
                    int ex = 0;
                    unsigned spins = 0;
                    NB_TR(if (lane == 0) s_park_gen = mt.gen;)
                    for (;;) {
                        if (__all_sync(0xffffffffu, slot_get(st_g->pub + 2 * slot, tag, &v))) break;
                        if ((++spins & 7u) == 0u && __any_sync(0xffffffffu, ld_gpu_s32(&st_g->done))) {
                            ex = !__all_sync(0xffffffffu, slot_get(st_g->pub + 2 * slot, tag, &v));
                            break;
                        }
                        __nanosleep(20);
                    }
                    NB_TR(if (lane == 0) s_park_gen = 0ull;)
                    if (ex) s_exit = 1;
                    else if (lane < a.m) s_y[lane] = v;
                    else if (lane == a.m) s_u = v;
                    else if (lane == a.m + 1) s_store = (int) (__double_as_longlong(v) & 1ll);
                }
                asm volatile("bar.sync 1, %0;" ::"r"(32 * kGroupWarps) : "memory");
                NB_TR(if (threadIdx.x == 0) {
                          const unsigned long long t = nb_globaltimer();
                          if (my_gen && my_gen < kTraceGens) { atomicMax(&sa.trace[16 * my_gen + 10], ~tr_last); atomicMax(&sa.trace[16 * my_gen + 11], tr_last); }
                          if (!s_exit && mt.gen < kTraceGens) { atomicMax(&sa.trace[16 * mt.gen + 1], ~t); atomicMax(&sa.trace[16 * mt.gen + 2], t); } })
                if (s_exit) break;
                my_gen = mt.gen;
                mu.u_ccsaq = s_u;
                store = s_store != 0;
            }
            NB_TR(tr_s0 = nb_globaltimer();)
#pragma unroll
            for (int k = 0; k < NV; ++k) acc[k] = 0.0;
        }
        double2 vx = make_double2(0.0, 0.0), vlb = vx, vub = vx, vs = vx, vg = vx;
        double Ga[MR], Gb[MR];
#pragma unroll
        for (int i = 0; i < MR; ++i) { Ga[i] = 0.0; Gb[i] = 0.0; }
        const bool has = !(mt.flags & 4u);
        unsigned iw = 0;                                      // SIDX: the two 16-bit sigma indices of this lane's pair
        if (has) {
            const double2 *t = s_tile + (size_t) st * NARR * kChunkPairs + sub * 32 + lane;
            vx = t[0];
            if (NB) {
                vlb = t[kChunkPairs];
                vub = t[2 * kChunkPairs];
            } else {
                vlb = make_double2(a.lb_u, a.lb_u);
                vub = make_double2(a.ub_u, a.ub_u);
            }
            if (SIDX) iw = s_idx[(size_t) st * kChunkPairs + sub * 32 + lane];
            else vs = t[(1 + NB) * kChunkPairs];
            vg = t[KG * kChunkPairs];
#pragma unroll
            for (int i = 0; i < MAXM; ++i) { const double2 g2 = t[(KG + 1 + i) * kChunkPairs]; Ga[i] = g2.x; Gb[i] = g2.y; }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&s_empty[st]);             // operands are in registers: release the stage
        if (++st == STAGES) { st = 0; phase ^= 1u; }
        ++consumed;
        if (SIDX && has) vs = make_double2(__ldg(a.pal + (iw & 0xffffu)), __ldg(a.pal + (iw >> 16)));
        if (has) {
            double2 xc;
            if (VARIANT == 0) {
                xc.x = mma_point<MAXM, true>(mu, vx.x, vlb.x, vub.x, vs.x, vg.x, Ga, acc);
                xc.y = mma_point<MAXM, true>(mu, vx.y, vlb.y, vub.y, vs.y, vg.y, Gb, acc);
            } else {
                xc.x = ccsaq_point<MAXM, true>(mu, vx.x, vlb.x, vub.x, vs.x, vg.x, Ga, acc);
                xc.y = ccsaq_point<MAXM, true>(mu, vx.y, vlb.y, vub.y, vs.y, vg.y, Gb, acc);
            }
            if (store) st_stream(reinterpret_cast<double2 *>(a.xcur) + mt.p + sub * 32 + lane, xc);
        }
        if (mt.flags & 2u) {
            warp_fold<NV>(acc);
            double *srec = s_rec[parity];
            if (lane == 0) {
#pragma unroll
                for (int k = 0; k < NV; ++k) srec[sub * NV + k] = acc[k];
            }
            asm volatile("bar.sync 1, %0;" ::"r"(32 * kGroupWarps) : "memory");
            parity ^= 1;
            if (sub == 0) put_group_record<NV>(srec, a.grouptags, ngroups, mt.gl, sa.tag0 | my_gen, lane);
            NB_TR(if (sub == 0 && lane == 0 && my_gen < kTraceGens) { const unsigned long long t = nb_globaltimer(); unsigned long long *r = sa.trace + 16 * my_gen;
                      atomicMax(r + 3, ~t); atomicMax(r + 4, t); atomicAdd(r + 8, t - tr_s0); atomicAdd(r + 9, 1ull); tr_last = t; })
        }
    }
    // ---- leaving: stop the producer, then wait for every copy it has issued (the stage we hold is complete) ----
    if (threadIdx.x == 0) {
        s_stop = 1;
        while (!s_prod_done) __nanosleep(20);
        __threadfence_block();
        const unsigned long long issued = s_issued;
        unsigned long long done = consumed + 1;               // stages whose full barrier we have already passed
        if (++st == STAGES) { st = 0; phase ^= 1u; }
        for (; done < issued; ++done) {
            mbar_wait(&s_full[st], phase);
            if (++st == STAGES) { st = 0; phase ^= 1u; }
        }
    }
    asm volatile("bar.sync 1, %0;" ::"r"(32 * kGroupWarps) : "memory");
}

// Gradient of the augmented-Lagrangian objective (auglag.c:47-48, :59-60): g_j += coef_k * row_k[j] for the
// K penalty rows in index order, separate multiply and add like the reference's loop (=> bit-identical gradient).
// Rows with coef == 0 flagged by `skip` are left out entirely (an inactive inequality adds nothing, auglag.c:57).
constexpr int kPenaltyRowsPerLaunch = 16;
struct PenaltyCoefs {
    double c[kPenaltyRowsPerLaunch];
    int row[kPenaltyRowsPerLaunch];       // index of the row in the scratch block
    int count;
};
__global__ void __launch_bounds__(kBlock) penalty_axpy_kernel(double *__restrict__ g, const double *__restrict__ rows,
                                                               unsigned long long ld, unsigned long long n_local,
                                                               const __grid_constant__ PenaltyCoefs pc)
{
    const unsigned long long stride = (unsigned long long) gridDim.x * blockDim.x;
    for (unsigned long long j = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; j < n_local; j += stride) {
        double v = g[j];
        for (int k = 0; k < pc.count; ++k) v = addx(v, mulx(pc.c[k], rows[(unsigned long long) pc.row[k] * ld + j]));
        g[j] = v;
    }
}

// Maximisation with a device or sharded objective (nlopt_b200_set_max_objective_*): the library minimises -f, so the
// gradient the callback wrote is negated in place.  Flipping the sign bit is IEEE negation and gives the bits of
// g[j] = -g[j] on the host for every input: +-0, subnormals, infinities and NaN payloads only change sign.  Two
// variables per 128-bit load and store (a row starts 16-byte aligned); an odd n_local leaves one tail element.  Exactly
// n_local entries are touched: the padding lanes stay +0.0.
__global__ void __launch_bounds__(kBlock) negate_kernel(double *__restrict__ g, unsigned long long n_local)
{
    constexpr unsigned long long kSign = 0x8000000000000000ull;
    const unsigned long long pairs = n_local >> 1, stride = (unsigned long long) gridDim.x * blockDim.x;
    const unsigned long long t = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x;
    ulonglong2 *g2 = reinterpret_cast<ulonglong2 *>(g);
    for (unsigned long long p = t; p < pairs; p += stride) {
        ulonglong2 v = g2[p];
        v.x ^= kSign;
        v.y ^= kSign;
        g2[p] = v;
    }
    if ((n_local & 1) && t == 0) {
        unsigned long long *tail = reinterpret_cast<unsigned long long *>(g) + (n_local - 1);
        *tail ^= kSign;
    }
}

// After the all-gather (several ranks): fold the 8 shard sums in index order and publish.
__global__ void publish_kernel(const double *all_vsums /* [8][nvp] */, int nv, int nvp, volatile double *out_host,
                               volatile unsigned long long *flag_host, unsigned long long seq)
{
    for (int k = threadIdx.x; k < nv; k += blockDim.x) {      // one CTA
        double s = all_vsums[k];
        for (int v = 1; v < kVirtualShards; ++v) s = addx(s, all_vsums[v * nvp + k]);
        out_host[k] = s;
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        *flag_host = seq;
        __threadfence_system();
    }
}

// ---- one-element halo of the shard for stencil device callbacks (include/nlopt_b200.h: nlopt_b200_dfunc2, halo = 1) ----
// Mailbox form: lane 0 hands this rank's first element to the left neighbour (its right halo cell), lane 1 the last
// element to the right neighbour (its left halo cell), as tagged 128-bit peer stores into slots 20 / 21 of virtual-shard
// record 0 (slots 0..19 carry the dual sums and the time flag); then each lane polls the cell it is owed.
constexpr int kBoxHaloLeft = 20, kBoxHaloRight = 21;
struct HaloArgs {
    double *x;                    // shard start; cells x[-1] and x[n_pad] are the halo
    unsigned long long n_local;   // > 0
    unsigned long long right_cell;    // index of the right halo cell (n_local when the shard fills its padded length)
    double *box[8];
    int rank, world;
    unsigned long long seq;
};
__global__ void halo_exchange_kernel(const __grid_constant__ HaloArgs a)
{
    const int lane = threadIdx.x;
    const int buf = (int) (a.seq & 1ull);
    const bool left = a.rank > 0, right = a.rank + 1 < a.world;
    if (lane == 0 && left)
        box_put(a.box[a.rank - 1] + 2ull * ((unsigned long long) buf * 8 * kBoxStride + kBoxHaloRight), a.x[0], a.seq);
    if (lane == 1 && right)
        box_put(a.box[a.rank + 1] + 2ull * ((unsigned long long) buf * 8 * kBoxStride + kBoxHaloLeft), a.x[a.n_local - 1], a.seq);
    if ((lane == 0 && left) || (lane == 1 && right)) {
        const double *mine = a.box[a.rank] + 2ull * ((unsigned long long) buf * 8 * kBoxStride + (lane == 0 ? kBoxHaloLeft : kBoxHaloRight));
        const unsigned long long t0 = nb_globaltimer();
        double v;
        bool ok;
        while (!(ok = box_get(mine, a.seq, &v)))
            if (nb_globaltimer() - t0 > 10000000000ull) break;              // 10 s: a peer died
        if (!ok) v = __longlong_as_double(0x7ff8000000000000ll);
        if (lane == 0) a.x[-1] = v; else a.x[a.right_cell] = v;
    }
}
// NCCL form: edges[r] = {first, last} of every rank (all-gathered); pick the neighbours' values
__global__ void halo_apply_kernel(double *x, unsigned long long right_cell, const double *edges, int rank, int world)
{
    if (threadIdx.x == 0 && rank > 0) x[-1] = edges[2 * (rank - 1) + 1];
    if (threadIdx.x == 1 && rank + 1 < world) x[right_cell] = edges[2 * (rank + 1)];
}
__global__ void halo_pack_kernel(const double *x, unsigned long long n_local, double *edges, int rank)
{
    if (threadIdx.x == 0) { edges[2 * rank] = x[0]; edges[2 * rank + 1] = x[n_local - 1]; }
}

__global__ void fill_kernel(double *dst, double value, unsigned long long n_local)
{
    for (unsigned long long j = blockIdx.x * (unsigned long long) blockDim.x + threadIdx.x; j < n_local;
         j += (unsigned long long) gridDim.x * blockDim.x)
        dst[j] = value;
}

// ---- sigma initialisation, mma.c:202-210 ---------------------------------------------------------
__device__ __forceinline__ bool dev_isinf(double v) { return fabs(v) >= HUGE_VAL * 0.99 || isinf(v); }

// sidx (or null): the sigma index, whose palette entry 1 is the one value this kernel writes (sigma_palette.hpp)
__global__ void sigma_init_kernel(double *sigma, const double *lb, const double *ub, const double *sigma_init,
                                  double sigma_min, unsigned long long n_local, unsigned short *sidx)
{
    for (unsigned long long j = blockIdx.x * (unsigned long long) blockDim.x + threadIdx.x; j < n_local;
         j += (unsigned long long) gridDim.x * blockDim.x) {
        double s;
        if (sigma_init && sigma_init[j] > 0) s = sigma_init[j];
        else if (dev_isinf(ub[j]) || dev_isinf(lb[j])) s = 1.0;
        else s = mulx(0.5, subx(ub[j], lb[j]));
        sigma[j] = s > sigma_min ? s : sigma_min;
        if (sidx) sidx[j] = 1;
    }
}

// ---- fused end-of-outer-iteration pass -------------------------------------------------------------
// Also the stop test + "keep the point" of the NLOPT_AUGLAG* outer loop (DeviceBackend::stop_x_keep): update_sigma = 0
// and a null xprevprev, so xprev (the best point) <- xcur and nothing else is written.
struct EndOuterArgs {
    const double *xcur;
    double *xprev, *xprevprev, *sigma;
    const double *lb, *ub;
    const double *w;          // x weights or null (stop.c:37-79)
    const double *xtol_abs;   // or null
    unsigned long long n_local, nchunks, chunk0;
    unsigned nseg_total, seg0, segs_per_vshard, local_vshards;
    double *partials, *vsums;
    unsigned *tickets;
    double *out_dev;
    volatile double *out_host;
    volatile unsigned long long *flag_host;
    unsigned long long seq;
    int publish_host, nvp;
    int update_sigma;         // k > 1
    double kappa;             // 0.01 (mma.c:439) or 1e-8 (ccsa_quadratic.c:587)
    double sigma_min;
    // sigma index (or null sidx): sidx[j] <- next[3 sidx[j] + branch]; every variable whose new sigma differs from
    // pal[sidx[j]] is counted into the 4th sum, and the host stops using the index
    unsigned short *sidx;
    const unsigned short *next;
    const double *pal;
};

__global__ void __launch_bounds__(kBlock) end_outer_kernel(const __grid_constant__ EndOuterArgs a)
{
    constexpr int NV = 4;     // sum w|dx|, sum w|x|, count of |dx| >= xtol_abs, count of sigma index mismatches
    __shared__ double s_red[kWarps * NV];
    __shared__ int s_flag;
    const unsigned seg = a.seg0 + blockIdx.x;
    unsigned long long p_lo, p_hi;
    group_pairs(a.nchunks, a.nseg_total, a.chunk0, seg, &p_lo, &p_hi);
    double acc[NV] = {0.0, 0.0, 0.0, 0.0};
    for (unsigned long long p = p_lo + threadIdx.x; p < p_hi; p += kBlock) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const unsigned long long j = 2 * p + h;
            if (j >= a.n_local) break;
            const double xc = a.xcur[j], xp = a.xprev[j];
            const double d = fabs(subx(xc, xp));
            if (a.w) {
                acc[0] = addx(acc[0], mulx(a.w[j], d));
                acc[1] = addx(acc[1], mulx(a.w[j], fabs(xc)));
            } else {
                acc[0] = addx(acc[0], d);
                acc[1] = addx(acc[1], fabs(xc));
            }
            if (a.xtol_abs && d >= a.xtol_abs[j]) acc[2] = addx(acc[2], 1.0);
            if (a.update_sigma) {
                const double xpp = a.xprevprev[j];
                const double osc = mulx(subx(xc, xp), subx(xp, xpp));
                const int br = osc < 0 ? 0 : (osc > 0 ? 1 : 2);
                const double s0 = a.sigma[j];
                double s = mulx(s0, br == 0 ? 0.7 : (br == 1 ? 1.2 : 1.0));
                const double lo = a.lb[j], hi = a.ub[j];
                if (!dev_isinf(hi) && !dev_isinf(lo)) {
                    const double range = subx(hi, lo);
                    const double top = mulx(10.0, range), bot = mulx(a.kappa, range);
                    s = s < top ? s : top;
                    s = s > bot ? s : bot;
                }
                s = s > a.sigma_min ? s : a.sigma_min;
                a.sigma[j] = s;
                if (a.sidx) {     // the index before the update (sigma_0 included) and after it must both match
                    const unsigned short i0 = a.sidx[j], t = a.next[3u * i0 + br];
                    a.sidx[j] = t;
                    if (__double_as_longlong(__ldg(a.pal + i0)) != __double_as_longlong(s0) ||
                        __double_as_longlong(__ldg(a.pal + t)) != __double_as_longlong(s))
                        acc[3] = addx(acc[3], 1.0);
                }
            }
            if (a.xprevprev) a.xprevprev[j] = xp;
            a.xprev[j] = xc;
        }
    }
    block_reduce_to<NV>(acc, s_red, a.partials + (unsigned long long) blockIdx.x * a.nvp);
    const unsigned vs_local = blockIdx.x / a.segs_per_vshard;
    if (!is_last_arrival(a.tickets + vs_local, a.segs_per_vshard, &s_flag)) return;
    acc[0] = acc[1] = acc[2] = acc[3] = 0.0;
    {
        const double *base = a.partials + (unsigned long long) vs_local * a.segs_per_vshard * a.nvp;
        for (unsigned sgi = threadIdx.x; sgi < a.segs_per_vshard; sgi += kBlock)
#pragma unroll
            for (int k = 0; k < NV; ++k) acc[k] = addx(acc[k], __ldcg(base + (unsigned long long) sgi * a.nvp + k));
    }
    block_reduce_to<NV>(acc, s_red, a.vsums + (unsigned long long) vs_local * a.nvp);
    if (!is_last_arrival(a.tickets + a.local_vshards, a.local_vshards, &s_flag)) return;
    if (threadIdx.x < NV) {
        if (a.publish_host) {
            double s = __ldcg(a.vsums + threadIdx.x);
            for (unsigned v = 1; v < a.local_vshards; ++v) s = addx(s, __ldcg(a.vsums + (unsigned long long) v * a.nvp + threadIdx.x));
            a.out_host[threadIdx.x] = s;
            __threadfence_system();
        } else {
            const unsigned v0 = a.seg0 / a.segs_per_vshard;
            for (unsigned v = 0; v < a.local_vshards; ++v)
                a.out_dev[(unsigned long long) (v0 + v) * a.nvp + threadIdx.x] = __ldcg(a.vsums + (unsigned long long) v * a.nvp + threadIdx.x);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (unsigned v = 0; v <= a.local_vshards; ++v) a.tickets[v] = 0;
        if (a.publish_host) {
            *a.flag_host = a.seq;
            __threadfence_system();
        }
    }
}

}  // namespace nb200
