// stream_probe.cu -- how fast can this card stream the dual kernels' operand set from HBM, with no arithmetic at all?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build/stream_probe tools/probes/stream_probe.cu && build/stream_probe [n] [m]
// Reads (3 + m) separate arrays of n doubles (the operand set of one dual evaluation with uniform bounds: x, sigma, g and
// the m gradient rows; n = 1e7, m = 4 by default: 560 MB) with the kernels' 128-bit ld.global.nc.L1::no_allocate loads,
// grid-stride over 16-byte pairs, all (3 + m) loads of a step issued before they are combined.  Swept over CTAs per SM
// and pairs per thread and step (UNROLL); each point is the median and the best of 30 timed launches (CUDA events) after
// 5 warm-up launches.  The best point is the ceiling the sweep of the dual kernels can be compared against.
//   build/stream_probe serpentine [n] [m]
// Serpentine mode: the operand set of the sigma-index solve kernel (2 + m arrays of n doubles and n 16-bit indices: 500 MB
// at n = 1e7, m = 4) streamed pass after pass in three orders, alternated in rounds so that clock and neighbours affect
// all three alike: forward every pass; forward and backward on alternate passes (each pass starts on the lines the
// previous one read last, which may still be in the L2); the same with the loads of the part of each pass that the next
// one does not reuse (all but the last L2-size worth) marked L2::evict_first.  Reports the median per-pass time.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ double2 ld_stream(const double2 *p)
{
    double2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
    return v;
}

template <int NARR, int UNROLL>
__global__ void __launch_bounds__(256) stream(const double2 *base, size_t ld2, size_t npairs, unsigned long long *sink)
{
    unsigned long long acc = 0;
    const size_t stride = (size_t) gridDim.x * blockDim.x * UNROLL;
    for (size_t p = (size_t) blockIdx.x * blockDim.x * UNROLL + threadIdx.x; p < npairs; p += stride) {
        double2 v[UNROLL][NARR];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
#pragma unroll
            for (int k = 0; k < NARR; ++k)
                v[u][k] = p + u * blockDim.x < npairs ? ld_stream(base + k * ld2 + p + u * blockDim.x) : make_double2(0.0, 0.0);
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
#pragma unroll
            for (int k = 0; k < NARR; ++k) acc ^= __double_as_longlong(v[u][k].x) ^ __double_as_longlong(v[u][k].y);
    }
    if (acc == 0x5EED5EED5EED5EEDull) *sink = acc;       // keeps the loads; never true: equal values cancel in pairs
}

__device__ __forceinline__ double2 ld_first(const double2 *p, unsigned long long pol)
{
    double2 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(v.x), "=d"(v.y) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ unsigned ld_idx(const unsigned *p, bool first, unsigned long long pol)
{
    unsigned v;
    if (first) asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    else asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// one pass over NARR double arrays and one array of pair indices (32 bits per pair); rev: from the last pair down;
// pairs of the pass order below `hint_end` are loaded evict_first
template <int NARR>
__global__ void __launch_bounds__(256) stream_dir(const double2 *base, const unsigned *idx, size_t ld2, size_t npairs, int rev,
                                                  size_t hint_end, unsigned long long *sink)
{
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    unsigned long long acc = 0;
    const size_t stride = (size_t) gridDim.x * blockDim.x;
    for (size_t q = (size_t) blockIdx.x * blockDim.x + threadIdx.x; q < npairs; q += stride) {
        const size_t p = rev ? npairs - 1 - q : q;
        const bool first = q < hint_end;
        double2 v[NARR];
#pragma unroll
        for (int k = 0; k < NARR; ++k) v[k] = first ? ld_first(base + k * ld2 + p, pol) : ld_stream(base + k * ld2 + p);
        acc ^= ld_idx(idx + p, first, pol);
#pragma unroll
        for (int k = 0; k < NARR; ++k) acc ^= __double_as_longlong(v[k].x) ^ __double_as_longlong(v[k].y);
    }
    if (acc == 0x5EED5EED5EED5EEDull) *sink = acc;
}

template <int NARR>
int serpentine(size_t n, int sms, size_t l2_bytes)
{
    const size_t ld = (n + 511) / 512 * 512, npairs = ld / 2;
    const double bytes = (16.0 * NARR + 4.0) * npairs;
    double2 *base;
    unsigned *idx;
    unsigned long long *sink;
    CK(cudaMalloc(&base, 8 * ld * NARR));
    CK(cudaMalloc(&idx, 2 * ld));
    CK(cudaMalloc(&sink, 8));
    CK(cudaMemset(base, 0x5a, 8 * ld * NARR));
    CK(cudaMemset(idx, 0x01, 2 * ld));
    const size_t reuse_pairs = (size_t) (l2_bytes / (16.0 * NARR + 4.0));
    const size_t hint_end = npairs > reuse_pairs ? npairs - reuse_pairs : 0;
    const int grid = sms * 4;
    printf("serpentine: %d double arrays + 16-bit indices, %.1f MB per pass, L2 %.0f MB, grid %d x 256\n", NARR, bytes / 1e6,
           l2_bytes / 1e6, grid);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const char *names[3] = {"forward only", "forward / backward", "forward / backward + evict_first"};
    std::vector<float> per[3];
    const int passes = 20;
    for (int round = 0; round < 6; ++round)
        for (int mode = 0; mode < 3; ++mode) {
            for (int w = 0; w < 3; ++w) stream_dir<NARR><<<grid, 256>>>(base, idx, ld / 2, npairs, 0, 0, sink);
            for (int k = 0; k < passes; ++k) {
                const int rev = mode == 0 ? 0 : (k & 1);
                float t = 0;
                CK(cudaEventRecord(e0));
                stream_dir<NARR><<<grid, 256>>>(base, idx, ld / 2, npairs, rev, mode == 2 ? hint_end : 0, sink);
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
                CK(cudaEventElapsedTime(&t, e0, e1));
                if (k > 0) per[mode].push_back(t);       // the first pass of a run has no predecessor in its order
            }
        }
    CK(cudaGetLastError());
    double med[3];
    for (int mode = 0; mode < 3; ++mode) {
        std::sort(per[mode].begin(), per[mode].end());
        const float m = per[mode][per[mode].size() / 2];
        med[mode] = m;
        printf("%-34s median %7.1f us  %6.0f GB/s   quartiles %7.1f .. %7.1f us  (%zu passes)\n", names[mode], m * 1e3,
               bytes / (m * 1e-3) * 1e-9, per[mode][per[mode].size() / 4] * 1e3, per[mode][3 * per[mode].size() / 4] * 1e3,
               per[mode].size());
    }
    printf("gain per pass against forward only: %+.1f %% (forward / backward), %+.1f %% (+ evict_first)\n",
           100.0 * (med[0] / med[1] - 1.0), 100.0 * (med[0] / med[2] - 1.0));
    CK(cudaFree(base));
    CK(cudaFree(idx));
    CK(cudaFree(sink));
    return 0;
}

template <int NARR, int UNROLL>
int sweep(const double2 *base, size_t ld2, size_t npairs, int sms, unsigned long long *sink, double *best_gbs)
{
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const double bytes = 16.0 * (double) npairs * NARR;
    for (int per_sm : {2, 3, 4, 6, 8}) {
        const int grid = sms * per_sm;
        for (int w = 0; w < 5; ++w) stream<NARR, UNROLL><<<grid, 256>>>(base, ld2, npairs, sink);
        CK(cudaGetLastError());
        std::vector<float> ms;
        for (int r = 0; r < 30; ++r) {
            float t = 0;
            CK(cudaEventRecord(e0));
            stream<NARR, UNROLL><<<grid, 256>>>(base, ld2, npairs, sink);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaEventElapsedTime(&t, e0, e1));
            ms.push_back(t);
        }
        std::sort(ms.begin(), ms.end());
        const double med = bytes / (ms[ms.size() / 2] * 1e-3) * 1e-9, best = bytes / (ms[0] * 1e-3) * 1e-9;
        *best_gbs = std::max(*best_gbs, best);
        printf("arrays %d  unroll %d  CTAs/SM %d (grid %5d x 256): median %7.1f us  %6.0f GB/s   best %6.0f GB/s\n", NARR, UNROLL,
               per_sm, grid, ms[ms.size() / 2] * 1e3, med, best);
    }
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    return 0;
}

int main(int argc, char **argv)
{
    const bool serp = argc > 1 && std::string(argv[1]) == "serpentine";
    if (serp) { --argc; ++argv; }
    const size_t n = argc > 1 ? (size_t) atof(argv[1]) : 10000000;
    const int m = argc > 2 ? atoi(argv[2]) : 4;
    if (serp) {
        if (m != 4) { printf("serpentine: m must be 4\n"); return 1; }
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, 0));
        printf("%s, %d SMs\n", prop.name, prop.multiProcessorCount);
        return serpentine<6>(n, prop.multiProcessorCount, (size_t) prop.l2CacheSize);
    }
    if (m != 1 && m != 4) { printf("m must be 1 or 4\n"); return 1; }
    const int narr = 3 + m;
    const size_t ld = (n + 511) / 512 * 512;            // the library's padded shard length
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("%s, %d SMs, L2 %d MB; n = %zu, m = %d: %d arrays, %.1f MB per pass\n", prop.name, prop.multiProcessorCount,
           prop.l2CacheSize >> 20, n, m, narr, 8.0 * ld * narr / 1e6);
    double2 *base;
    unsigned long long *sink;
    CK(cudaMalloc(&base, 8 * ld * narr));
    CK(cudaMemset(base, 0x5a, 8 * ld * narr));      // not zeros: nothing for the memory system to treat specially
    CK(cudaMalloc(&sink, 8));
    double best = 0;
    const int sms = prop.multiProcessorCount;
    int rc = 0;
    if (m == 4) {
        rc |= sweep<7, 1>(base, ld / 2, ld / 2, sms, sink, &best);
        rc |= sweep<7, 2>(base, ld / 2, ld / 2, sms, sink, &best);
    } else {
        rc |= sweep<4, 1>(base, ld / 2, ld / 2, sms, sink, &best);
        rc |= sweep<4, 2>(base, ld / 2, ld / 2, sms, sink, &best);
    }
    printf("ceiling: %.0f GB/s (best launch of the sweep)\n", best);
    CK(cudaFree(base));
    CK(cudaFree(sink));
    return rc;
}
