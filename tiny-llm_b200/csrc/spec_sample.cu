// Speculative sampling: the rejection rule that turns a draft's sampled proposals into draws of the target's
// distribution (DESIGN.md section 8d).  One launch covers the T = k + 1 rows of a verify pass; row j < k checks the
// proposal d_j against target row x_j and draft row y_j, row k draws the bonus token as tl_sample does.
//
// Each row is one cluster of C CTAs, planned as tl_sample's (sample_plan).  CTA r stages the r-th slice of BOTH rows
// in shared memory as fp32 (2 * slice floats), then:
//   1. the first-maximum argmax of each row; greedy rows and rows with a non-finite maximum are the point mass at it;
//   2. each row's keep threshold with tl_sample's own code (TL_ROW_KEEP_THRESHOLD, row_cluster.cuh);
//   3. one pass sums the temperature masses E_i = rn(exp((x_i - m) / T) 2^40) over each keep set, 64-bit integers,
//      so S_p and S_q are exact in any order.  p_i = E^x_i / S_p and q_i = E^y_i / S_q;
//   4. p_d and q_d come from the CTA that holds d, over distributed shared memory.  Accept iff q_d > 0 and
//      u q_d <= p_d, u = (2 (w >> 9) + 1) 2^-24 from word 0 of Philox at counter (0, n_j, 1, 0); the test is done
//      on the integers, u' E^y_d S_p <= 2^24 E^x_d S_q, in 128 bits;
//   5. on rejection, argmax over {i : p_i > q_i} (again an integer comparison, E^x_i S_q > E^y_i S_p) of
//      log(p_i - q_i) + g_i, g_i the Gumbel noise of Philox stream 2 (counter (i >> 2, n_j, 2, 0)).
// Because the comparisons are exact on the kernel's own masses, sum p = sum q = 1 holds exactly and a rejection
// (p_d < q_d) always leaves an i with p_i > q_i: the residual set is never empty.  Should it be, the row returns x's
// argmax token, so the kernel always writes a token.
#include <cooperative_groups.h>

#include <climits>

#include "common.cuh"
#include "kernels.h"
#include "row_cluster.cuh"

namespace cg = cooperative_groups;

namespace tl {

namespace {

using u128 = unsigned __int128;

__device__ __forceinline__ double u128_to_double(u128 v) {
    return static_cast<double>(static_cast<unsigned long long>(v >> 64)) * 18446744073709551616.0 +
           static_cast<double>(static_cast<unsigned long long>(v));
}

// The fixed-point temperature mass of a kept entry (m: the row maximum, so the term is <= 1).
__device__ __forceinline__ unsigned long long temp_mass(float x, float m, float temp) {
    return static_cast<unsigned long long>(__float2ull_rn(expf(__fdiv_rn(__fsub_rn(x, m), temp)) * MASS_SCALE));
}

// One row's distribution as the kernel holds it: the point mass at `a`, or the keep set {order_key(x) >= tau} with
// masses temp_mass(x, m, temp) over the total S.
struct RowDist {
    bool point;
    int a;
    uint32_t tau;
    float m;
    unsigned long long S;
};

__device__ __forceinline__ unsigned long long mass_of(const RowDist &r, float x, int i, float temp) {
    if (r.point) return i == r.a ? 1ull : 0ull;
    return (x == x && order_key(x) >= r.tau) ? temp_mass(x, r.m, temp) : 0ull;
}

// Block then cluster first-maximum merge of every thread's candidate; pub must not be reused before a cluster barrier.
__device__ __forceinline__ Best cluster_best(Best mine, float *w_v, int *w_i, Best &pub, Best &res, cg::cluster_group &cluster) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    mine = warp_best(mine);
    if (lane == 0) w_v[warp] = mine.v, w_i[warp] = mine.i;
    __syncthreads();
    if (warp == 0) {
        mine = warp_best(lane < SAMPLE_WARPS ? Best{w_v[lane], w_i[lane]} : Best{-INFINITY, INT_MAX});
        if (lane == 0) pub = mine;
    }
    cluster.sync();
    if (threadIdx.x == 0) {
        Best b{-INFINITY, INT_MAX};
        for (int r = 0; r < static_cast<int>(cluster.num_blocks()); ++r) b = better(b, *cluster.map_shared_rank(&pub, r));
        res = b;
    }
    __syncthreads();
    return res;
}

template <typename T, int LEVELS>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
    spec_sample_kernel(const T *__restrict__ target, const T *__restrict__ draft, const int32_t *__restrict__ proposals,
                       const float *__restrict__ temperature, const int32_t *__restrict__ top_k, const float *__restrict__ top_p,
                       const int64_t *__restrict__ seed, const int32_t *__restrict__ positions, int32_t *__restrict__ out, int rows,
                       int vocab, int slice, int vec) {
    extern __shared__ float4 smem_dyn[];
    float *xs = reinterpret_cast<float *>(smem_dyn);  // target slice
    float *ys = xs + slice;                           // draft slice
    __shared__ unsigned int h_count[2][BINS];
    __shared__ unsigned long long h_mass[2][BINS];
    __shared__ unsigned int t_count[BINS];
    __shared__ unsigned long long t_mass[BINS];
    __shared__ float w_v[SAMPLE_WARPS];
    __shared__ int w_i[SAMPLE_WARPS];
    __shared__ unsigned long long w_s[2][SAMPLE_WARPS];
    __shared__ Best pub_mx, pub_my, pub_draw, res_mx, res_my, res_draw;
    __shared__ unsigned long long pub_s[2], tot_s[2];
    __shared__ uint32_t s_prefix;
    __shared__ int s_k_on, s_p_on;
    __shared__ unsigned int s_count_above;
    __shared__ unsigned long long s_mass_above;
    __shared__ double s_p_mass;
    __shared__ int s_bk, s_bp;
    __shared__ unsigned int s_bk_above;
    __shared__ unsigned long long s_bp_above;

    cg::cluster_group cluster = cg::this_cluster();
    const int rank = static_cast<int>(cluster.block_rank());
    const int C = static_cast<int>(cluster.num_blocks());
    const int row = blockIdx.y;
    const bool bonus = row == rows - 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int begin = rank * slice;
    const int n = max(0, min(vocab, begin + slice) - begin);

    for (int i = threadIdx.x; i < 2 * BINS; i += SAMPLE_THREADS) (&h_count[0][0])[i] = 0, (&h_mass[0][0])[i] = 0;
    griddep_wait();  // logits, proposals, parameters and positions are the previous launches' output
    const float temp = temperature[row];
    const uint32_t pos = static_cast<uint32_t>(positions[row]);
    const uint64_t sd = static_cast<uint64_t>(seed[row]);
    const uint32_t k0 = static_cast<uint32_t>(sd), k1 = static_cast<uint32_t>(sd >> 32);
    stage_slice(target + static_cast<size_t>(row) * vocab + begin, xs, n, vec != 0);
    if (!bonus) stage_slice(draft + static_cast<size_t>(row) * vocab + begin, ys, n, vec != 0);
    __syncthreads();

    // ---- 1. row maxima (first maximum wins) and the point-mass rows
    Best mine{-INFINITY, INT_MAX};
    for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) mine = better(mine, Best{xs[i], begin + i});
    const Best mx = cluster_best(mine, w_v, w_i, pub_mx, res_mx, cluster);
    Best my{-INFINITY, INT_MAX};
    if (!bonus) {
        mine = Best{-INFINITY, INT_MAX};
        for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) mine = better(mine, Best{ys[i], begin + i});
        my = cluster_best(mine, w_v, w_i, pub_my, res_my, cluster);
    }
    RowDist P{!(temp > 0.f) || !isfinite(mx.v), mx.i == INT_MAX ? 0 : mx.i, 0u, mx.v, 1ull};
    RowDist Q{!(temp > 0.f) || !isfinite(my.v), my.i == INT_MAX ? 0 : my.i, 0u, my.v, 1ull};

    // ---- 2. keep thresholds, tl_sample's code on each row
    if (!P.point) {
        const float m = P.m;
        TL_ROW_KEEP_THRESHOLD(LEVELS);
        P.tau = s_prefix;
    }
    if (bonus) {  // tl_sample's draw on x_k, stream 0
        int token = P.a;
        if (!P.point) {
            const uint32_t tau = P.tau;
            const float m = P.m;
            mine = Best{-INFINITY, INT_MAX};
            TL_ROW_GUMBEL_PASS(0u);
            const Best d = cluster_best(mine, w_v, w_i, pub_draw, res_draw, cluster);
            token = d.i == INT_MAX ? P.a : d.i;
        }
        if (rank == 0 && threadIdx.x == 0) out[row] = token;
        cluster.sync();  // no CTA leaves while another may still read its shared memory
        return;
    }
    if (!Q.point) {
        cluster.sync();  // every CTA has read the other CTAs' histograms of x's last level
        for (int i = threadIdx.x; i < 2 * BINS; i += SAMPLE_THREADS) (&h_count[0][0])[i] = 0, (&h_mass[0][0])[i] = 0;
        __syncthreads();
        const float *xs = ys;
        const float m = Q.m;
        TL_ROW_KEEP_THRESHOLD(LEVELS);
        Q.tau = s_prefix;
    }

    // ---- 3. temperature masses of both keep sets, exact integer sums
    unsigned long long sp = 0, sq = 0;
    for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
        if (!P.point) sp += mass_of(P, xs[i], begin + i, temp);
        if (!Q.point) sq += mass_of(Q, ys[i], begin + i, temp);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sp += __shfl_xor_sync(0xffffffffu, sp, o), sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if (lane == 0) w_s[0][warp] = sp, w_s[1][warp] = sq;
    __syncthreads();
    if (threadIdx.x < 2) {
        unsigned long long s = 0;
        for (int w = 0; w < SAMPLE_WARPS; ++w) s += w_s[threadIdx.x][w];
        pub_s[threadIdx.x] = s;
    }
    cluster.sync();
    if (threadIdx.x < 2) {
        unsigned long long s = 0;
        for (int r = 0; r < C; ++r) s += *cluster.map_shared_rank(&pub_s[threadIdx.x], r);
        tot_s[threadIdx.x] = s;
    }
    __syncthreads();
    if (!P.point) P.S = tot_s[0];  // >= 2^40: the maximum is kept and weighs exactly 1
    if (!Q.point) Q.S = tot_s[1];

    // ---- 4. acceptance: p_d and q_d from the CTA that holds d
    const int d = proposals[row];
    unsigned long long pd = 0, qd = 0;
    if (d >= 0 && d < vocab) {
        const int owner = d / slice, at = d - owner * slice;
        pd = mass_of(P, *cluster.map_shared_rank(xs + at, owner), d, temp);
        qd = mass_of(Q, *cluster.map_shared_rank(ys + at, owner), d, temp);
    }
    const uint32_t w_acc = philox4x32_10(make_uint4(0u, pos, 1u, 0u), k0, k1).x;
    const u128 u_odd = 2u * (w_acc >> 9) + 1u;  // u = u_odd 2^-24
    if (qd > 0 && u_odd * qd * P.S <= (static_cast<u128>(pd) << 24) * Q.S) {
        if (rank == 0 && threadIdx.x == 0) out[row] = d;
        cluster.sync();
        return;
    }

    // ---- 5. residual: argmax over {p_i > q_i} of log(p_i - q_i) + g_i, Philox stream 2
    const double denom = static_cast<double>(P.S) * static_cast<double>(Q.S);
    mine = Best{-INFINITY, INT_MAX};
    for (int g = threadIdx.x * 4; g < n; g += SAMPLE_THREADS * 4) {
        u128 diff[4];
        bool any = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            diff[j] = 0;
            if (g + j < n) {
                const u128 a = static_cast<u128>(mass_of(P, xs[g + j], begin + g + j, temp)) * Q.S;
                const u128 b = static_cast<u128>(mass_of(Q, ys[g + j], begin + g + j, temp)) * P.S;
                if (a > b) diff[j] = a - b, any = true;
            }
        }
        if (!any) continue;
        const uint4 w = philox4x32_10(make_uint4(static_cast<uint32_t>(begin + g) >> 2, pos, 2u, 0u), k0, k1);
        const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (diff[j] != 0)
                mine = better(mine, Best{__fadd_rn(static_cast<float>(log(u128_to_double(diff[j]) / denom)), gumbel(ws[j])), begin + g + j});
    }
    const Best r = cluster_best(mine, w_v, w_i, pub_draw, res_draw, cluster);
    if (rank == 0 && threadIdx.x == 0) out[row] = r.i == INT_MAX ? P.a : r.i;
    cluster.sync();
}

template <typename T, int LEVELS>
int launch_spec_t(const void *target, const void *draft, const int32_t *proposals, const float *temperature, const int32_t *top_k,
                  const float *top_p, const int64_t *seed, const int32_t *positions, int32_t *out, int rows, int vocab, int cluster,
                  int slice, int vec, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(spec_sample_kernel<T, LEVELS>, cudaFuncAttributeMaxDynamicSharedMemorySize, SAMPLE_MAX_SMEM) != cudaSuccess)
            return fail(TL_ECUDA, "speculative_sample: cannot raise shared memory limit");
        configured = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(cluster, rows);
    cfg.blockDim = dim3(SAMPLE_THREADS);
    cfg.dynamicSmemBytes = 2 * static_cast<size_t>(slice) * sizeof(float);
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
    cudaError_t e = cudaLaunchKernelEx(&cfg, spec_sample_kernel<T, LEVELS>, static_cast<const T *>(target), static_cast<const T *>(draft),
                                       proposals, temperature, top_k, top_p, seed, positions, out, rows, vocab, slice, vec);
    if (e != cudaSuccess) return fail(TL_ECUDA, "speculative_sample: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("speculative_sample");
    return TL_OK;
}

// dst[out_index] = src (after the dependency wait: the index and the rows are earlier launches' output); 16 bytes per
// thread when both rows are 16-byte aligned and whole words, else one byte.
__global__ void log_rows_kernel(const unsigned char *__restrict__ src, unsigned char *__restrict__ dst, const int32_t *__restrict__ out_index,
                                int capacity, long long bytes, int vec) {
    griddep_wait();
    const int o = *out_index;
    if (o < 0 || o >= capacity) return;
    unsigned char *d = dst + static_cast<long long>(o) * bytes;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    const long long first = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (vec) {
        for (long long i = first; i < bytes / 16; i += stride)
            reinterpret_cast<uint4 *>(d)[i] = reinterpret_cast<const uint4 *>(src)[i];
    } else {
        for (long long i = first; i < bytes; i += stride) d[i] = src[i];
    }
}

}  // namespace

int launch_log_rows(const void *src, void *dst, const int32_t *out_index, int capacity, long long bytes, cudaStream_t st) {
    const int vec = (bytes % 16 == 0 && aligned16(src) && aligned16(dst)) ? 1 : 0;
    const long long items = vec ? bytes / 16 : bytes;
    const int blocks = static_cast<int>(ceil_div_ll(items, 256) < 132 ? ceil_div_ll(items, 256) : 132);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(blocks);
    cfg.blockDim = dim3(256);
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, log_rows_kernel, static_cast<const unsigned char *>(src), static_cast<unsigned char *>(dst), out_index,
                                       capacity, bytes, vec);
    if (e != cudaSuccess) return fail(TL_ECUDA, "log_rows: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("log_rows");
    return TL_OK;
}

int speculative_sample_plan(int vocab, int *cluster, int *slice) {
    int c = 0, s = 0;
    if (vocab <= 0) return fail(TL_EINVAL, "speculative_sample: bad shape");
    if (vocab > TL_SPECULATIVE_SAMPLE_MAX_VOCAB)
        return fail(TL_EINVAL, "speculative_sample: vocab %d exceeds %d", vocab, TL_SPECULATIVE_SAMPLE_MAX_VOCAB);
    if (int e = sample_plan(vocab, &c, &s)) return e;
    if (2 * static_cast<size_t>(s) * sizeof(float) > SAMPLE_MAX_SMEM)  // both slices staged: cannot happen below the limit
        return fail(TL_EINVAL, "speculative_sample: vocab %d exceeds %d", vocab, TL_SPECULATIVE_SAMPLE_MAX_VOCAB);
    if (cluster) *cluster = c;
    if (slice) *slice = s;
    return TL_OK;
}

int launch_speculative_sample(const void *target, const void *draft, const int32_t *proposals, const float *temperature,
                              const int32_t *top_k, const float *top_p, const int64_t *seed, const int32_t *positions, int32_t *out,
                              int rows, int vocab, int dtype, cudaStream_t st) {
    int cluster = 0, slice = 0;
    if (int e = speculative_sample_plan(vocab, &cluster, &slice)) return e;
    const int per16 = dtype == TL_F32 ? 4 : 8;
    const int vec = (vocab % per16 == 0 && aligned16(target) && (rows == 1 || aligned16(draft))) ? 1 : 0;
    switch (dtype) {
        case TL_F32:
            return launch_spec_t<float, 4>(target, draft, proposals, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster, slice,
                                           vec, st);
        case TL_F16:
            return launch_spec_t<__half, 4>(target, draft, proposals, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster, slice,
                                            vec, st);
        case TL_BF16:  // raw bf16 rows: two radix levels, as tl_sample
            return launch_spec_t<__nv_bfloat16, 2>(target, draft, proposals, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster,
                                                   slice, vec, st);
        default: return fail(TL_EDTYPE, "speculative_sample: expected float32, float16, or bfloat16");
    }
}

}  // namespace tl
