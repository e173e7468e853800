// Seeded temperature / top-k / top-p sampling of one token per logits row (DESIGN.md section 8).
//
// Each row is drawn by a cluster of C CTAs (C = ceil(V / 4096), at most 8).  CTA r of the cluster stages the r-th slice
// of the row in shared memory once, as fp32, and every later pass reads it from there.  What the CTAs of a cluster
// exchange (row maximum, histograms, argmax candidates) goes through distributed shared memory between cluster
// barriers: one launch, no global workspace.  Every CTA of a cluster takes the same decisions from the same merged
// integers, so the CTAs never disagree about a branch or the number of barriers.
//
//   1. load the slice, fp32; the first-maximum-wins argmax of the raw values (tl_argmax's rules) gives the row
//      maximum m.  Greedy rows (temperature == 0) and rows whose maximum is not finite return that argmax.
//   2. keep set {x >= tau}: the logits map to order-preserving 32-bit keys; each radix level (2 for bf16, 4 for
//      fp16 / fp32) is one pass that adds a count and a mass e_i = exp(x_i - m) per 256-entry bin, for the elements
//      that share the prefix chosen so far.  Masses are 2^-40 fixed point in 64 bits, so their sums are exact in any
//      order.  Counts locate x_(k) and masses locate v* (the smallest value whose mass strictly above is < top_p * S)
//      in the same pass; where the two searches pick different bins the higher one is tau's and the other search ends.
//   3. one Gumbel pass: argmax over the kept i of x_i / T + g_i, g_i = -log(-log u_i), u_i from Philox4x32-10 at
//      counter (i >> 2, pos, 0, 0) and key (seed lo, seed hi); then the cluster argmax.
// Integer sums and first-maximum-wins merges make every launch give the same bits, whatever the row count.
//
// The penalised form (PEN, tl_sample_penalized, DESIGN.md section 8b) reads the row's int32 token state (bit 30: in
// the prompt, bits 0-29: times drawn) right after staging and rewrites the staged values in place with the repetition,
// frequency and presence penalties; every later step runs on that penalised row.  min-p adds a third lower bound on
// the keep threshold after the radix levels, and rank 0 adds 1 to the drawn token's count once every CTA has read
// its state slice.
#include <cooperative_groups.h>

#include <climits>

#include "common.cuh"
#include "kernels.h"
#include "row_cluster.cuh"

namespace cg = cooperative_groups;

namespace tl {

namespace {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

// Gumbel noise of one Philox word: u = (2 (w >> 9) + 1) 2^-24 is an odd multiple of 2^-24 in (0, 1), exact in fp32.
__device__ __forceinline__ float gumbel(uint32_t w) {
    const float u = static_cast<float>(2u * (w >> 9) + 1u) * 5.9604644775390625e-8f;
    return -logf(-logf(u));
}

// Per-row arrays of the penalised form; state is [rows, vocab].  Unused (all null) by the plain form.
struct Penalties {
    const float *repetition, *presence, *frequency, *min_p;
    int32_t *state;
    int svec;  // the state rows are 16-byte aligned (vocab % 4 == 0 and an aligned base)
};

constexpr int32_t STATE_PROMPT = 1 << 30;
constexpr int32_t STATE_COUNT = STATE_PROMPT - 1;

// x1 = seen && r != 1 ? (x > 0 ? x / r : x * r) : x;  x2 = c > 0 ? x1 - f c : x1;  x3 = c > 0 ? x2 - pres : x2, each
// operation rounded on its own (no contraction into an fma).
__device__ __forceinline__ float penalize(float x, int32_t s, float r, float pres, float f) {
    const int32_t c = s & STATE_COUNT;
    if ((s & STATE_PROMPT) || c > 0) {
        if (r != 1.f) x = x > 0.f ? __fdiv_rn(x, r) : __fmul_rn(x, r);
    }
    if (c > 0) x = __fsub_rn(__fsub_rn(x, __fmul_rn(f, __int2float_rn(c))), pres);
    return x;
}

template <typename T, int LEVELS, bool PEN>
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(const T *__restrict__ logits, const float *__restrict__ temperature,
                                                                const int32_t *__restrict__ top_k, const float *__restrict__ top_p,
                                                                const int64_t *__restrict__ seed, const int32_t *__restrict__ positions,
                                                                int32_t *__restrict__ out, int vocab, int slice, int vec, Penalties pen) {
    extern __shared__ float4 smem_dyn[];
    float *xs = reinterpret_cast<float *>(smem_dyn);
    __shared__ unsigned int h_count[2][BINS];  // double-buffered: level l + 2 reuses l's buffer after all remote reads of it
    __shared__ unsigned long long h_mass[2][BINS];
    __shared__ unsigned int t_count[BINS];  // cluster totals of the current level
    __shared__ unsigned long long t_mass[BINS];
    __shared__ float w_v[SAMPLE_WARPS];
    __shared__ int w_i[SAMPLE_WARPS];
    __shared__ Best pub_max, pub_draw;  // read by the other CTAs of the cluster
    __shared__ Best row_max;
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
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int begin = rank * slice;
    const int n = max(0, min(vocab, begin + slice) - begin);

    for (int i = threadIdx.x; i < 2 * BINS; i += SAMPLE_THREADS) (&h_count[0][0])[i] = 0, (&h_mass[0][0])[i] = 0;
    griddep_wait();  // the logits and the parameters are the previous launches' output
    const float temp = temperature[row];
    stage_slice(logits + static_cast<size_t>(row) * vocab + begin, xs, n, vec != 0);
    __syncthreads();
    if constexpr (PEN) {
        const float r = pen.repetition[row], pres = pen.presence[row], f = pen.frequency[row];
        if (r != 1.f || pres != 0.f || f != 0.f) {  // with every penalty off the values stay as staged: no state read
            const int32_t *st = pen.state + static_cast<size_t>(row) * vocab + begin;
            if (pen.svec) {  // n is a multiple of 4 here: the slice start is, and so is vocab
                for (int i = threadIdx.x * 4; i < n; i += SAMPLE_THREADS * 4) {
                    const int4 s = *reinterpret_cast<const int4 *>(st + i);
                    float4 x = *reinterpret_cast<const float4 *>(xs + i);
                    x.x = penalize(x.x, s.x, r, pres, f);
                    x.y = penalize(x.y, s.y, r, pres, f);
                    x.z = penalize(x.z, s.z, r, pres, f);
                    x.w = penalize(x.w, s.w, r, pres, f);
                    *reinterpret_cast<float4 *>(xs + i) = x;
                }
            } else {
                for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) xs[i] = penalize(xs[i], st[i], r, pres, f);
            }
            __syncthreads();
        }
    }

    // ---- 1. first-maximum-wins argmax of the (penalised) row
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
    }
    __syncthreads();
    const Best best = row_max;
    if (!(temp > 0.f) || !isfinite(best.v)) {
        if (rank == 0 && threadIdx.x == 0) {
            const int token = best.i == INT_MAX ? 0 : best.i;
            out[row] = token;
            if constexpr (PEN) {  // every CTA read its state slice before the cluster barrier above
                if (positions[row] > 0) pen.state[static_cast<size_t>(row) * vocab + token] += 1;
            }
        }
        cluster.sync();  // no CTA leaves while another may still read its pub_max
        return;
    }
    const float m = best.v;

    // ---- 2. keep set {key >= tau}
    if (threadIdx.x == 0) {
        const int k = top_k[row];
        const float p = top_p[row];
        s_k_on = k > 0 && k < vocab;
        s_p_on = p > 0.f && p < 1.f;
        s_prefix = 0;
        s_count_above = 0;
        s_mass_above = 0;
    }
    __syncthreads();
    const unsigned int k_want = static_cast<unsigned int>(top_k[row]);
    const float p_want = top_p[row];
    for (int level = 0; level < LEVELS && (s_k_on || s_p_on); ++level) {
        const int buf = level & 1;
        const int shift = 24 - 8 * level;
        const uint32_t prefix = s_prefix;
        const bool with_mass = s_p_on;
        unsigned int *cnt = h_count[buf];
        unsigned long long *mass = h_mass[buf];
        for (int base = warp * 32; base < n; base += SAMPLE_THREADS) {
            const int i = base + lane;
            int bin = -1;
            unsigned long long e = 0;
            if (i < n) {
                const float x = xs[i];
                if (x == x) {
                    const uint32_t key = order_key(x);
                    if (level == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) {
                        bin = static_cast<int>((key >> shift) & 0xffu);
                        if (with_mass) e = static_cast<unsigned long long>(__float2ull_rn(expf(x - m) * MASS_SCALE));
                    }
                }
            }
            bin_add(cnt, mass, bin, e, with_mass);
        }
        cluster.sync();
        if (threadIdx.x < BINS) {
            unsigned int c = 0;
            unsigned long long s = 0;
            for (int r = 0; r < C; ++r) {
                c += *cluster.map_shared_rank(&cnt[threadIdx.x], r);
                if (with_mass) s += *cluster.map_shared_rank(&mass[threadIdx.x], r);
            }
            t_count[threadIdx.x] = c;
            t_mass[threadIdx.x] = s;
        }
        // the buffer of the next level is free again: every CTA read it (level - 1) before this level's barrier
        for (int i = threadIdx.x; i < BINS; i += SAMPLE_THREADS) h_count[buf ^ 1][i] = 0, h_mass[buf ^ 1][i] = 0;
        __syncthreads();
        if (warp == 0) {
            // lane owns bins 8 lane .. 8 lane + 7; suffix sums from the top bin down
            unsigned int c[8];
            unsigned long long s[8];
            unsigned int lc = 0;
            unsigned long long ls = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) c[j] = t_count[8 * lane + j], s[j] = t_mass[8 * lane + j], lc += c[j], ls += s[j];
            unsigned int ca = lc;
            unsigned long long sa = ls;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned int oc = __shfl_down_sync(0xffffffffu, ca, o);
                const unsigned long long os = __shfl_down_sync(0xffffffffu, sa, o);
                if (lane + o < 32) ca += oc, sa += os;
            }
            const unsigned int total_c = __shfl_sync(0xffffffffu, ca, 0);
            const unsigned long long total_s = __shfl_sync(0xffffffffu, sa, 0);
            if (level == 0 && lane == 0) {
                if (total_c < k_want) s_k_on = 0;  // fewer non-NaN entries than k: top-k keeps them all
                s_p_mass = static_cast<double>(p_want) * static_cast<double>(total_s);
            }
            __syncwarp();
            const bool k_on = s_k_on, p_on = s_p_on;
            const double p_mass = s_p_mass;
            unsigned int above_c = s_count_above + (ca - lc);
            unsigned long long above_s = s_mass_above + (sa - ls);
            int bk = -1, bp = -1;
            unsigned int bk_above = 0;
            unsigned long long bp_above = 0;
#pragma unroll
            for (int j = 7; j >= 0; --j) {
                if (k_on && bk < 0 && above_c < k_want && k_want <= above_c + c[j]) bk = 8 * lane + j, bk_above = above_c;
                if (p_on && c[j] > 0 && static_cast<double>(above_s) < p_mass) bp = 8 * lane + j, bp_above = above_s;  // lowest wins
                above_c += c[j];
                above_s += s[j];
            }
            const unsigned kb = __ballot_sync(0xffffffffu, bk >= 0);
            const unsigned pb = __ballot_sync(0xffffffffu, bp >= 0);
            if (kb && lane == __ffs(kb) - 1) s_bk = bk, s_bk_above = bk_above;
            if (pb && lane == __ffs(pb) - 1) s_bp = bp, s_bp_above = bp_above;
            __syncwarp();
            if (lane == 0) {
                const int kbin = k_on ? s_bk : -1, pbin = p_on ? s_bp : -1;
                const int bin = max(kbin, pbin);  // tau = max(x_(k), v*): the higher bin holds it
                s_k_on = kbin == bin;
                s_p_on = pbin == bin;
                s_prefix = prefix | (static_cast<uint32_t>(bin) << shift);
                s_count_above = s_k_on ? s_bk_above : 0;
                s_mass_above = s_p_on ? s_bp_above : 0;
            }
        }
        __syncthreads();
    }
    uint32_t tau = s_prefix;
    if constexpr (PEN) {  // min-p: x >= m + T log(min_p), a bound on the whole row like the two above
        const float mp = pen.min_p[row];
        if (mp > 0.f) {
            const float log_p = static_cast<float>(log(static_cast<double>(fminf(mp, 1.f))));
            tau = max(tau, order_key(__fadd_rn(m, __fmul_rn(temp, log_p))));
        }
    }

    // ---- 3. Gumbel-max over the kept entries, 4 consecutive entries per Philox call
    const uint32_t pos = static_cast<uint32_t>(positions[row]);
    const uint64_t sd = static_cast<uint64_t>(seed[row]);
    const uint32_t k0 = static_cast<uint32_t>(sd), k1 = static_cast<uint32_t>(sd >> 32);
    mine = Best{-INFINITY, INT_MAX};
    for (int g = threadIdx.x * 4; g < n; g += SAMPLE_THREADS * 4) {
        bool any = false;
        float x[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            x[j] = g + j < n ? xs[g + j] : NAN;
            any |= x[j] == x[j] && order_key(x[j]) >= tau;
        }
        if (!any) continue;
        const uint4 w = philox4x32_10(make_uint4(static_cast<uint32_t>(begin + g) >> 2, pos, 0u, 0u), k0, k1);
        const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (x[j] == x[j] && order_key(x[j]) >= tau) mine = better(mine, Best{__fdiv_rn(x[j], temp) + gumbel(ws[j]), begin + g + j});
    }
    mine = warp_best(mine);
    if (lane == 0) w_v[warp] = mine.v, w_i[warp] = mine.i;
    __syncthreads();
    if (warp == 0) {
        mine = warp_best(lane < SAMPLE_WARPS ? Best{w_v[lane], w_i[lane]} : Best{-INFINITY, INT_MAX});
        if (lane == 0) pub_draw = mine;
    }
    cluster.sync();
    if (rank == 0 && threadIdx.x == 0) {
        Best d{-INFINITY, INT_MAX};
        for (int r = 0; r < C; ++r) d = better(d, *cluster.map_shared_rank(&pub_draw, r));
        const int token = d.i == INT_MAX ? best.i : d.i;  // the row maximum is always kept: INT_MAX cannot happen
        out[row] = token;
        if constexpr (PEN) {
            if (positions[row] > 0) pen.state[static_cast<size_t>(row) * vocab + token] += 1;
        }
    }
    cluster.sync();
}

template <typename T, int LEVELS, bool PEN>
int launch_sample_t(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                    const int32_t *positions, int32_t *out, int rows, int vocab, int cluster, int slice, int vec, const Penalties &pen,
                    cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(sample_kernel<T, LEVELS, PEN>, cudaFuncAttributeMaxDynamicSharedMemorySize, SAMPLE_MAX_SMEM) != cudaSuccess)
            return fail(TL_ECUDA, "sample: cannot raise shared memory limit");
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
    cudaError_t e =
        cudaLaunchKernelEx(&cfg, sample_kernel<T, LEVELS, PEN>, x, temperature, top_k, top_p, seed, positions, out, vocab, slice, vec, pen);
    if (e != cudaSuccess) return fail(TL_ECUDA, "sample: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("sample");
    return TL_OK;
}

template <bool PEN>
int launch_sample_any(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                      const int32_t *positions, int32_t *out, int rows, int vocab, int dtype, const Penalties &pen, cudaStream_t st) {
    if (rows == 0) return TL_OK;
    int cluster = 0, slice = 0;
    if (int e = sample_plan(vocab, &cluster, &slice)) return e;
    const int per16 = dtype == TL_F32 ? 4 : 8;
    const int vec = (vocab % per16 == 0 && aligned16(logits)) ? 1 : 0;
    switch (dtype) {
        case TL_F32:
            return launch_sample_t<float, 4, PEN>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster, slice, vec, pen,
                                                  st);
        case TL_F16:
            return launch_sample_t<__half, 4, PEN>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster, slice, vec,
                                                   pen, st);
        case TL_BF16:  // a bf16 value's key has 16 significant bits: two levels
            return launch_sample_t<__nv_bfloat16, 2, PEN>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster, slice,
                                                           vec, pen, st);
        default: return fail(TL_EDTYPE, "sample: expected float32, float16, or bfloat16");
    }
}

}  // namespace

int sample_plan(int vocab, int *cluster, int *slice) {
    if (vocab <= 0) return fail(TL_EINVAL, "sample: bad shape");
    const int c = ceil_div(vocab, SAMPLE_SLICE_MIN) < SAMPLE_MAX_CLUSTER ? ceil_div(vocab, SAMPLE_SLICE_MIN) : SAMPLE_MAX_CLUSTER;
    const int s = ceil_div(ceil_div(vocab, c), 8) * 8;  // a multiple of 8 entries: 16-byte slice starts, whole Philox groups
    if (static_cast<size_t>(s) * sizeof(float) > SAMPLE_MAX_SMEM)
        return fail(TL_EINVAL, "sample: vocab %d exceeds %d", vocab, SAMPLE_MAX_CLUSTER * (SAMPLE_MAX_SMEM / 4));
    if (cluster) *cluster = c;
    if (slice) *slice = s;
    return TL_OK;
}

int launch_sample(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                  const int32_t *positions, int32_t *out, int rows, int vocab, int dtype, cudaStream_t st) {
    return launch_sample_any<false>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, Penalties{}, st);
}

int launch_sample_penalized(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                            const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                            const float *min_p, int32_t *state, int32_t *out, int rows, int vocab, int dtype, cudaStream_t st) {
    const Penalties pen{repetition, presence, frequency, min_p, state, (vocab % 4 == 0 && aligned16(state)) ? 1 : 0};
    return launch_sample_any<true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, st);
}

}  // namespace tl
