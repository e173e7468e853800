// DRY, "don't repeat yourself" (DESIGN.md section 24): penalise every token that would extend a repeat of an earlier
// span of the request's history, by an amount that grows exponentially with the repeat's length.
//
// One cluster of C CTAs per row (C from the history capacity, at most 8); the CTAs split the row's history ends.  Each
// CTA stages the row's breakers and the last TL_DRY_MAX_MATCH ids of the history (h_{n-1} = the step's input token)
// in shared memory, then
//   1. for each of its ends e computes the match length l(e) against the suffix and, when it reaches the allowed
//      length, the candidate x_t - P[l(e) - a] from the unpenalised row, kept in the row's scratch slot e;
//   2. after a cluster barrier (no entry of the row has been written before it), lowers x_t to each of its candidates
//      with an atomic minimum.  Every candidate of t was computed from the same x_t, so the row keeps the one of the
//      longest match whatever the order of the atomics: the result is deterministic.
// Work follows the window, not the vocabulary; nothing is zeroed per step.  Rank 0 appends the input token to the
// history at index n - 1 (idempotent: a replay writes the same id).
#include <cooperative_groups.h>

#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

namespace tl {

namespace {

constexpr int DRY_THREADS = 256;
constexpr int DRY_ENDS_MIN = 4096;  // history ends per CTA before the cluster grows
constexpr int DRY_MAX_CLUSTER = 8;

__device__ __forceinline__ bool is_breaker(const int32_t *b, int nb, int32_t t) {
    int lo = 0, hi = nb;  // sorted ascending
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (b[mid] < t) lo = mid + 1;
        else hi = mid;
    }
    return lo < nb && b[lo] == t;
}

// x = min(x, v) for non-NaN fp32 values: non-negative floats order as signed ints, negative ones in reverse as unsigned.
__device__ __forceinline__ void atomic_min_f32(float *x, float v) {
    if (v >= 0.f) atomicMin(reinterpret_cast<int *>(x), __float_as_int(v));
    else atomicMax(reinterpret_cast<unsigned int *>(x), __float_as_uint(v));
}

__global__ void __launch_bounds__(DRY_THREADS) dry_kernel(float *__restrict__ x, const tl_dry_row *__restrict__ dry,
                                                          const int32_t *__restrict__ positions, const int32_t *__restrict__ tokens,
                                                          int32_t *__restrict__ history, float *__restrict__ scratch, int vocab, int capacity) {
    __shared__ int32_t s_brk[TL_DRY_MAX_BREAKERS];
    __shared__ int32_t s_suffix[TL_DRY_MAX_MATCH];  // s_suffix[i] = h_{n-1-i}
    __shared__ float s_pen[TL_DRY_MAX_MATCH];
    __shared__ int s_free;  // the suffix's breaker-free length (capped)
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = static_cast<int>(cluster.block_rank());
    const int C = static_cast<int>(cluster.num_blocks());
    const int row = blockIdx.y;

    griddep_wait();  // the rows are the previous launch's output
    const tl_dry_row *d = dry + row;
    const int n = positions[row];
    if (!(d->flags & TL_DRY_ON) || n < 1 || n > capacity) return;  // uniform over the cluster: no barrier is skipped
    const int a = d->allowed_length, N = d->last_n;
    const int nb = min(max(d->num_breakers, 0), TL_DRY_MAX_BREAKERS);
    const int lo = N > 0 ? max(0, n - N) : 0;
    int32_t *h = history + static_cast<size_t>(row) * capacity;
    const int32_t last = tokens[row];
    if (threadIdx.x < TL_DRY_MAX_BREAKERS) s_brk[threadIdx.x] = threadIdx.x < nb ? d->breakers[threadIdx.x] : 0;
    if (threadIdx.x < TL_DRY_MAX_MATCH) {
        const int j = n - 1 - static_cast<int>(threadIdx.x);
        s_suffix[threadIdx.x] = j == n - 1 ? last : j >= 0 ? h[j] : -1;
        s_pen[threadIdx.x] = d->penalty[threadIdx.x];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int f = 0;
        while (f < TL_DRY_MAX_MATCH && f < n && !is_breaker(s_brk, nb, s_suffix[f])) ++f;
        s_free = f;
    }
    __syncthreads();
    const int free_len = s_free;
    float *xr = x + static_cast<size_t>(row) * vocab;
    float *sc = scratch + static_cast<size_t>(row) * capacity;
    const int first = lo + rank * DRY_THREADS + static_cast<int>(threadIdx.x), stride = C * DRY_THREADS;
    if (free_len >= a) {  // else no end can match a ids (h_{n-1} a breaker: free_len 0): nothing is penalised
        for (int e = first; e <= n - 2; e += stride) {
            const int32_t t = e + 1 == n - 1 ? last : h[e + 1];
            float v = NAN;
            if (t >= 0 && t < vocab && !is_breaker(s_brk, nb, t)) {
                const int lim = min(free_len, e - lo + 1);
                int l = 0;
                while (l < lim && __ldg(h + e - l) == s_suffix[l]) ++l;
                if (l >= a) {
                    const float p = s_pen[l - a];
                    v = isinf(p) ? -INFINITY : __fsub_rn(xr[t], p);
                }
            }
            sc[e] = v;
        }
    }
    cluster.sync();  // every candidate of the row was read from the unpenalised row
    if (free_len >= a) {
        for (int e = first; e <= n - 2; e += stride) {
            const float v = sc[e];
            if (v == v) atomic_min_f32(xr + (e + 1 == n - 1 ? last : h[e + 1]), v);
        }
    }
    if (rank == 0 && threadIdx.x == 0) h[n - 1] = last;
}

}  // namespace

int launch_dry_penalty(float *x, const tl_dry_row *dry, const int32_t *positions, const int32_t *tokens, int32_t *history, float *scratch,
                       int rows, int vocab, int capacity, cudaStream_t st) {
    if (rows == 0) return TL_OK;
    const int cluster = min(DRY_MAX_CLUSTER, max(1, ceil_div(capacity, DRY_ENDS_MIN)));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cluster, rows);
    cfg.blockDim = dim3(DRY_THREADS);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 2 : 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, dry_kernel, x, dry, positions, tokens, history, scratch, vocab, capacity);
    if (e != cudaSuccess) return fail(TL_ECUDA, "dry_penalty: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("dry_penalty");
    return TL_OK;
}

}  // namespace tl
