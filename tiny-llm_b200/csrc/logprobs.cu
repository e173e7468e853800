// Log-probabilities, ranks and top-N alternatives of logits rows (DESIGN.md section 8a).
//
// Each row is read by a cluster of C CTAs (C = ceil(V / 4096), at most 8, sample_plan's rule), exactly as tl_sample
// reads it: CTA r stages the r-th slice in shared memory once, as fp32, and everything the CTAs exchange is an integer
// or a first-maximum-wins candidate, merged over distributed shared memory.  So every launch gives the same bits for a
// row, whatever the row count, the row's index or graph capture.
//
//   1. stage the slice; the first-maximum-wins argmax gives the row maximum m; the target's value x_t is read from the
//      CTA that holds it.
//   2. S = sum over non-NaN i of round(expf(fl(x_i - m)) * 2^40), 64-bit integers (exact in any order), and the rank
//      count #{i : x_i > x_t}.  lp(x) = fl(fl(x - m) - logf(fl(S) * 2^-40)), lse = fl(m + logf(...)).
//   3. (rows with top_n > 0) radix select of the N-th largest order key on count histograms, 2 levels for bf16 and 4
//      for fp16 / fp32; when the equal keys at the N-th place are more than the list has room for, 3 more levels
//      select the lowest ids among them (keys ~id, 24 bits).  The N chosen entries are gathered by CTA 0 and ordered
//      by (value descending, id ascending).
#include <cooperative_groups.h>

#include <climits>

#include "common.cuh"
#include "kernels.h"
#include "row_cluster.cuh"

namespace cg = cooperative_groups;

namespace tl {

namespace {

constexpr int ID_LEVELS = 3;                             // ids < 2^24: three 8-bit levels of ~id
constexpr float MASS_UNSCALE = 9.094947017729282e-13f;  // 2^-40

// The one expression every reported log-probability comes from.
__device__ __forceinline__ float log_prob(float x, float m, float log_s) { return __fsub_rn(__fsub_rn(x, m), log_s); }

template <typename T, int LEVELS>
__global__ void __launch_bounds__(SAMPLE_THREADS)
    logprobs_kernel(const T *__restrict__ logits, const int32_t *__restrict__ targets, const int32_t *__restrict__ top_n,
                    const int32_t *__restrict__ out_index, float *__restrict__ lse_out, float *__restrict__ lp_out, int32_t *__restrict__ rank_out,
                    int32_t *__restrict__ top_ids, float *__restrict__ top_lp, int vocab, int slice, int vec, int max_n, int out_capacity) {
    extern __shared__ float4 smem_dyn[];
    float *xs = reinterpret_cast<float *>(smem_dyn);
    __shared__ unsigned int h_count[2][BINS];  // double-buffered as in tl_sample
    __shared__ unsigned int t_count[BINS];
    __shared__ float w_v[SAMPLE_WARPS];
    __shared__ int w_i[SAMPLE_WARPS];
    __shared__ unsigned long long w_s[SAMPLE_WARPS];
    __shared__ unsigned int w_c[SAMPLE_WARPS];
    __shared__ Best pub_max;  // read by the other CTAs of the cluster
    __shared__ unsigned long long pub_s;
    __shared__ unsigned int pub_c;
    __shared__ int pub_n;
    __shared__ float pub_v[LOGPROBS_MAX_N];
    __shared__ int pub_i[LOGPROBS_MAX_N];
    __shared__ Best row_max;
    __shared__ float s_xt, s_log_s;
    __shared__ uint32_t s_prefix, s_tau;
    __shared__ unsigned int s_want, s_eq;
    __shared__ int s_ids;
    __shared__ int s_target, s_want_n, s_out_row;

    cg::cluster_group cluster = cg::this_cluster();
    const int rank = static_cast<int>(cluster.block_rank());
    const int C = static_cast<int>(cluster.num_blocks());
    const int row = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int begin = rank * slice;
    const int n = max(0, min(vocab, begin + slice) - begin);

    for (int i = threadIdx.x; i < 2 * BINS; i += SAMPLE_THREADS) (&h_count[0][0])[i] = 0;
    griddep_wait();  // the logits and the targets are the previous launches' output (tl_argmax / tl_sample in a decode graph)
    if (threadIdx.x == 0) {
        s_target = targets ? targets[row] : -1;
        s_want_n = max(0, min(max_n, top_n ? top_n[row] : max_n));
        const int at = out_index ? out_index[0] : 0;  // a log row outside the buffer writes nothing (decode_advance's rule)
        s_out_row = (at >= 0 && at < out_capacity) ? at * static_cast<int>(gridDim.y) + row : -1;
    }
    stage_slice(logits + static_cast<size_t>(row) * vocab + begin, xs, n, vec != 0);
    __syncthreads();

    // ---- 1. row maximum (first maximum wins, NaN never) and the target's value
    Best mine{-INFINITY, INT_MAX};
    for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) mine = better(mine, Best{xs[i], begin + i});
    mine = warp_best(mine);
    if (lane == 0) w_v[warp] = mine.v, w_i[warp] = mine.i;
    __syncthreads();
    if (warp == 0) {
        mine = warp_best(lane < SAMPLE_WARPS ? Best{w_v[lane], w_i[lane]} : Best{-INFINITY, INT_MAX});
        if (lane == 0) pub_max = mine;
    }
    cluster.sync();
    if (threadIdx.x == 0) {
        Best m{-INFINITY, INT_MAX};
        for (int r = 0; r < C; ++r) m = better(m, *cluster.map_shared_rank(&pub_max, r));
        row_max = m;
        const int t = s_target;
        s_xt = (t >= 0 && t < vocab) ? *cluster.map_shared_rank(xs + (t - (t / slice) * slice), t / slice) : NAN;
    }
    __syncthreads();
    const float m = row_max.v;
    const bool finite = isfinite(m);  // false: +inf, or no entry above -inf, or every entry NaN
    const float xt = s_xt;

    // ---- 2. fixed-point mass and the target's rank count
    unsigned long long s = 0;
    unsigned int above = 0;
    for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
        const float x = xs[i];
        if (x == x) {
            if (finite) s += __float2ull_rn(expf(x - m) * MASS_SCALE);
            above += x > xt ? 1u : 0u;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o), above += __shfl_xor_sync(0xffffffffu, above, o);
    if (lane == 0) w_s[warp] = s, w_c[warp] = above;
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0, above = 0;
        for (int w = 0; w < SAMPLE_WARPS; ++w) s += w_s[w], above += w_c[w];
        pub_s = s, pub_c = above;
    }
    cluster.sync();
    if (threadIdx.x == 0) {
        s = 0, above = 0;
        for (int r = 0; r < C; ++r) s += *cluster.map_shared_rank(&pub_s, r), above += *cluster.map_shared_rank(&pub_c, r);
        // S >= 1 (the maximum adds exactly 2^40), so the scaling by 2^-40 is exact; logf is the last rounding but one
        s_log_s = finite ? logf(__ull2float_rn(s) * MASS_UNSCALE) : NAN;
        const int out_row = s_out_row;
        if (rank == 0 && out_row >= 0) {
            lse_out[out_row] = finite ? __fadd_rn(m, s_log_s) : (row_max.i == INT_MAX ? NAN : m);
            lp_out[out_row] = xt == xt ? log_prob(xt, m, s_log_s) : NAN;
            rank_out[out_row] = xt == xt ? static_cast<int>(above) + 1 : 0;
        }
    }
    __syncthreads();
    const float log_s = s_log_s;

    // ---- 3. the want_n largest entries
    if (max_n > 0) {
        constexpr int KSHIFT = 32 - 8 * LEVELS;  // the key bits a value of this dtype can differ in
        if (threadIdx.x == 0) s_prefix = 0, s_want = s_want_n, s_ids = 0, s_tau = 0, s_eq = 0, pub_n = 0;
        __syncthreads();
        for (int level = 0; level < LEVELS + ID_LEVELS && s_want > 0 && (level < LEVELS || s_ids); ++level) {
            const int buf = level & 1;
            const bool ids = level >= LEVELS;
            const int shift = ids ? 16 - 8 * (level - LEVELS) : 24 - 8 * level;
            const uint32_t prefix = s_prefix, tau = s_tau;
            unsigned int *cnt = h_count[buf];
            for (int base = warp * 32; base < n; base += SAMPLE_THREADS) {
                const int i = base + lane;
                int bin = -1;
                if (i < n) {
                    const float x = xs[i];
                    if (x == x) {
                        const uint32_t key = order_key(x);
                        if (!ids) {
                            if (level == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) bin = static_cast<int>((key >> shift) & 0xffu);
                        } else if ((key >> KSHIFT) == (tau >> KSHIFT)) {
                            const uint32_t idk = ~static_cast<uint32_t>(begin + i) & 0xffffffu;  // larger key: lower id
                            if ((idk >> (shift + 8)) == (prefix >> (shift + 8))) bin = static_cast<int>((idk >> shift) & 0xffu);
                        }
                    }
                }
                bin_add(cnt, nullptr, bin, 0ull, false);
            }
            cluster.sync();
            if (threadIdx.x < BINS) {
                unsigned int c = 0;
                for (int r = 0; r < C; ++r) c += *cluster.map_shared_rank(&cnt[threadIdx.x], r);
                t_count[threadIdx.x] = c;
            }
            // the buffer of the next level is free again: every CTA read it (level - 1) before this level's barrier
            for (int i = threadIdx.x; i < BINS; i += SAMPLE_THREADS) h_count[buf ^ 1][i] = 0;
            __syncthreads();
            if (warp == 0) {
                // lane owns bins 8 lane .. 8 lane + 7; suffix sums from the top bin down
                unsigned int c[8];
                unsigned int lc = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) c[j] = t_count[8 * lane + j], lc += c[j];
                unsigned int ca = lc;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned int oc = __shfl_down_sync(0xffffffffu, ca, o);
                    if (lane + o < 32) ca += oc;
                }
                const unsigned int total = __shfl_sync(0xffffffffu, ca, 0);
                const unsigned int want = level == 0 ? min(s_want, total) : s_want;  // never more than the non-NaN entries
                unsigned int acc = ca - lc;
                int bk = -1;
                unsigned int bk_above = 0, bk_count = 0;
#pragma unroll
                for (int j = 7; j >= 0; --j) {
                    if (bk < 0 && acc < want && want <= acc + c[j]) bk = 8 * lane + j, bk_above = acc, bk_count = c[j];
                    acc += c[j];
                }
                const unsigned kb = __ballot_sync(0xffffffffu, bk >= 0);
                __syncwarp();
                if (!kb) {
                    if (lane == 0) s_want = 0;  // no non-NaN entry: an empty list
                } else if (lane == __ffs(kb) - 1) {
                    s_prefix = prefix | (static_cast<uint32_t>(bk) << shift);
                    s_want = want - bk_above;  // entries still to take inside the chosen bin
                    s_eq = bk_count;
                }
                __syncwarp();
                if (lane == 0 && level == LEVELS - 1 && s_want > 0) {
                    s_tau = s_prefix;             // the N-th largest key
                    s_ids = s_want < s_eq;        // ties straddle the N-th place: select the lowest ids among them
                    s_prefix = 0;
                }
            }
            __syncthreads();
        }
        // collect: keys above tau, and keys equal to it (with an id key >= the selected one when ties straddle)
        const unsigned int take = s_want;
        const uint32_t tau = s_tau, idt = s_prefix;
        const bool ids = s_ids != 0;
        if (take > 0) {
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float x = xs[i];
                if (x != x) continue;
                const uint32_t kh = order_key(x) >> KSHIFT, th = tau >> KSHIFT;
                const uint32_t idk = ~static_cast<uint32_t>(begin + i) & 0xffffffu;
                if (kh > th || (kh == th && (!ids || idk >= idt))) {
                    const int j = atomicAdd(&pub_n, 1);
                    if (j < LOGPROBS_MAX_N) pub_v[j] = x, pub_i[j] = begin + i;
                }
            }
        }
        cluster.sync();
        if (rank == 0 && s_out_row >= 0) {
            __shared__ float cv[LOGPROBS_MAX_N];
            __shared__ int ci[LOGPROBS_MAX_N];
            __shared__ int s_total;
            if (threadIdx.x == 0) {
                int total = 0;
                for (int r = 0; r < C; ++r) {
                    const int k = min(*cluster.map_shared_rank(&pub_n, r), LOGPROBS_MAX_N);
                    for (int j = 0; j < k && total < LOGPROBS_MAX_N; ++j, ++total)
                        cv[total] = *cluster.map_shared_rank(&pub_v[j], r), ci[total] = *cluster.map_shared_rank(&pub_i[j], r);
                }
                s_total = min(total, s_want_n);
            }
            __syncthreads();
            const int total = s_total, out_row = s_out_row;
            int32_t *ids_row = top_ids + static_cast<size_t>(out_row) * max_n;
            float *lp_row = top_lp + static_cast<size_t>(out_row) * max_n;
            if (threadIdx.x < total) {
                const Best me{cv[threadIdx.x], ci[threadIdx.x]};
                int pos = 0;
                for (int k = 0; k < total; ++k) pos += (cv[k] > me.v || (cv[k] == me.v && ci[k] < me.i)) ? 1 : 0;
                if (pos < total) ids_row[pos] = me.i, lp_row[pos] = log_prob(me.v, m, log_s);  // log_s is NaN when m is not finite
            } else if (threadIdx.x < max_n) {
                ids_row[threadIdx.x] = -1, lp_row[threadIdx.x] = -INFINITY;
            }
        }
    }
    cluster.sync();  // no CTA leaves while another may still read its shared memory
}

template <typename T, int LEVELS>
int launch_logprobs_t(const void *logits, const int32_t *targets, const int32_t *top_n, const int32_t *out_index, float *lse, float *lp,
                      int32_t *rank, int32_t *top_ids, float *top_lp, int rows, int vocab, int max_n, int out_capacity, int cluster, int slice,
                      int vec, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(logprobs_kernel<T, LEVELS>, cudaFuncAttributeMaxDynamicSharedMemorySize, SAMPLE_MAX_SMEM) != cudaSuccess)
            return fail(TL_ECUDA, "logprobs: cannot raise shared memory limit");
        configured = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cluster, rows);
    cfg.blockDim = dim3(SAMPLE_THREADS);
    cfg.dynamicSmemBytes = static_cast<size_t>(slice) * sizeof(float);
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
    const T *x = static_cast<const T *>(logits);
    cudaError_t e = cudaLaunchKernelEx(&cfg, logprobs_kernel<T, LEVELS>, x, targets, top_n, out_index, lse, lp, rank, top_ids, top_lp, vocab,
                                       slice, vec, max_n, out_capacity);
    if (e != cudaSuccess) return fail(TL_ECUDA, "logprobs: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("logprobs");
    return TL_OK;
}

}  // namespace

int launch_logprobs(const void *logits, const int32_t *targets, const int32_t *top_n, const int32_t *out_index, float *lse, float *lp,
                    int32_t *rank, int32_t *top_ids, float *top_lp, int rows, int vocab, int max_n, int out_capacity, int dtype,
                    cudaStream_t st) {
    if (rows == 0) return TL_OK;
    int cluster = 0, slice = 0;
    if (int e = sample_plan(vocab, &cluster, &slice)) return e;
    const int per16 = dtype == TL_F32 ? 4 : 8;
    const int vec = (vocab % per16 == 0 && aligned16(logits)) ? 1 : 0;
    switch (dtype) {
        case TL_F32:
            return launch_logprobs_t<float, 4>(logits, targets, top_n, out_index, lse, lp, rank, top_ids, top_lp, rows, vocab, max_n,
                                               out_capacity, cluster, slice, vec, st);
        case TL_F16:
            return launch_logprobs_t<__half, 4>(logits, targets, top_n, out_index, lse, lp, rank, top_ids, top_lp, rows, vocab, max_n,
                                                out_capacity, cluster, slice, vec, st);
        case TL_BF16:  // a bf16 value's key has 16 significant bits: two levels
            return launch_logprobs_t<__nv_bfloat16, 2>(logits, targets, top_n, out_index, lse, lp, rank, top_ids, top_lp, rows, vocab, max_n,
                                                       out_capacity, cluster, slice, vec, st);
        default: return fail(TL_EDTYPE, "logprobs: expected float32, float16, or bfloat16");
    }
}

}  // namespace tl
