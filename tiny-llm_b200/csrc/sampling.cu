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
//   2. keep set {x >= tau}: the logits map to order-preserving 32-bit keys; each radix level (2 for raw bf16 rows, 4
//      once a penalty can move a value off the bf16 grid, 4 for fp16 / fp32) is one pass that adds a count and a mass e_i = exp(x_i - m) per 256-entry bin, for the elements
//      that share the prefix chosen so far.  Masses are 2^-40 fixed point in 64 bits, so their sums are exact in any
//      order.  Counts locate x_(k) and masses locate v* (the smallest value whose mass strictly above is < top_p * S)
//      in the same pass; where the two searches pick different bins the higher one is tau's and the other search ends.
//      Top-k with k above the non-NaN count is off, and with top-p off too every non-NaN entry is kept.
//   3. one Gumbel pass: argmax over the kept i of (x_i - m) / T + g_i, g_i = -log(-log u_i), u_i from Philox4x32-10 at
//      counter (i >> 2, pos, 0, 0) and key (seed lo, seed hi); then the cluster argmax.  The maximum's term is exactly
//      0, so a temperature near the bottom of fp32 sends the others to -inf instead of every kept term to +-inf: the
//      draw is x_i / T + g_i's in exact arithmetic.
// Integer sums and first-maximum-wins merges make every launch give the same bits, whatever the row count.
//
// The penalised form (PEN, tl_sample_penalized, DESIGN.md section 8b) reads the row's int32 token state (bit 30: in
// the prompt, bits 0-29: times drawn) right after staging and rewrites the staged values in place with the repetition,
// frequency and presence penalties; every later step runs on that penalised row.  min-p adds a third lower bound on
// the keep threshold after the radix levels, and rank 0 adds 1 to the drawn token's count once every CTA has read
// its state slice.
//
// The constrained form (MASK, tl_sample_constrained, DESIGN.md section 8c) reads the row's tl_constraint_row after
// the wait.  For a row with a mask, the staged entries of disallowed tokens become NaN after the penalty rewrite:
// NaN entries are never counted, weighed, kept or drawn, so every later step runs on the allowed entries alone.  Rank 0
// walks the drawn token's bytes through the DFA and writes the row's new state, for rows with position > 0.
//
// The XTC forms (XTC, DESIGN.md section 24) add one step after the keep threshold: with probability q, drawn from
// Philox stream 3 at the row's position, the kept entries whose share of the kept mass is at least theta, all but the
// least likely of them, become NaN when there are two or more.  Two integer passes over the staged slice (the kept
// mass, then the count and minimum key of the entries at or above theta's share) decide it, so every CTA of the
// cluster drops the same entries.
#include <cooperative_groups.h>

#include <climits>

#include "common.cuh"
#include "kernels.h"
#include "row_cluster.cuh"

namespace cg = cooperative_groups;

namespace tl {

namespace {

// Per-row arrays of the penalised form; state is [rows, vocab].  Unused (all null) by the plain form.
struct Penalties {
    const float *repetition, *presence, *frequency, *min_p;
    int32_t *state;
    int svec;  // the state rows are 16-byte aligned (vocab % 4 == 0 and an aligned base)
};

// Per-row arrays of the XTC forms.  Unused (all null) by the others.
struct Xtc {
    const float *threshold, *probability;
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

// The constrained row's state after `token`: S (terminal) after an allowed token without bytes (EOS) or in S, else the
// DFA walk of the token's bytes (-1 once dead, which an allowed token never reaches).  A state outside [0, S] stays.
__device__ __forceinline__ int32_t constraint_advance(const tl_constraint_row &c, int token) {
    int32_t s = c.state;
    if (s < 0 || s >= c.num_states) return s;
    const int b0 = c.token_offsets[token], b1 = c.token_offsets[token + 1];
    if (b0 == b1) return c.num_states;
    for (int j = b0; j < b1 && s >= 0; ++j) s = c.dfa[s * 256 + c.token_bytes[j]];
    return s;
}

// The lowest id the row's mask allows (0 when it allows none): the token of a row without an allowed non-NaN entry.
__device__ __forceinline__ int constraint_lowest(const tl_constraint_row &c, int vocab) {
    if (c.state < 0 || c.state > c.num_states) return 0;
    const int words = (vocab + 31) >> 5;
    const uint32_t *m = c.mask + static_cast<size_t>(c.state) * words;
    for (int w = 0; w < words; ++w)
        if (m[w]) return min(vocab - 1, 32 * w + __ffs(m[w]) - 1);
    return 0;
}

template <typename T, int LEVELS, bool PEN, bool MASK, bool XTC>
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(const T *__restrict__ logits, const float *__restrict__ temperature,
                                                                const int32_t *__restrict__ top_k, const float *__restrict__ top_p,
                                                                const int64_t *__restrict__ seed, const int32_t *__restrict__ positions,
                                                                int32_t *__restrict__ out, int vocab, int slice, int vec, Penalties pen,
                                                                tl_constraint_row *con, Xtc xtc) {
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
    if constexpr (MASK) {
        const uint32_t *mask = con[row].mask;
        if (mask) {  // disallowed entries (and every entry of a state outside [0, S]) become NaN
            const int32_t state = con[row].state, S = con[row].num_states;
            const bool known = state >= 0 && state <= S;
            const uint32_t *m = mask + static_cast<size_t>(known ? state : 0) * ((vocab + 31) >> 5);
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const int t = begin + i;
                if (!known || !((__ldg(m + (t >> 5)) >> (t & 31)) & 1u)) xs[i] = NAN;
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
            int token = best.i == INT_MAX ? 0 : best.i;
            if constexpr (MASK) {
                if (con[row].mask && best.i == INT_MAX) token = constraint_lowest(con[row], vocab);
            }
            out[row] = token;
            if constexpr (PEN) {  // every CTA read its state slice before the cluster barrier above
                if (positions[row] > 0) pen.state[static_cast<size_t>(row) * vocab + token] += 1;
            }
            if constexpr (MASK) {  // and its constraint state
                if (con[row].mask && positions[row] > 0) con[row].state = constraint_advance(con[row], token);
            }
        }
        cluster.sync();  // no CTA leaves while another may still read its pub_max
        return;
    }
    const float m = best.v;

    // ---- 2. keep set {key >= tau}
    TL_ROW_KEEP_THRESHOLD(LEVELS);
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
    if constexpr (XTC) {
        __shared__ unsigned long long x_mass;
        __shared__ unsigned int x_count, x_min, x_hi;
        const uint4 w = philox4x32_10(make_uint4(0u, pos, 3u, 0u), k0, k1);
        const float u = static_cast<float>(2u * (w.x >> 9) + 1u) * 5.9604644775390625e-8f;
        if (u < xtc.probability[row]) {  // the same decision in every CTA of the cluster
            if (threadIdx.x == 0) x_mass = 0, x_count = 0, x_min = UINT_MAX;
            __syncthreads();
            // e_i = exp((x_i - m) / T) in 2^-40 fixed point: integer sums, exact in any order
            unsigned long long s = 0;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (v == v && order_key(v) >= tau) s += __float2ull_rn(expf(__fdiv_rn(__fsub_rn(v, m), temp)) * MASS_SCALE);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0 && s) atomicAdd(&x_mass, s);
            cluster.sync();
            unsigned long long total = 0;
            for (int r = 0; r < C; ++r) total += *cluster.map_shared_rank(&x_mass, r);
            const double thr = static_cast<double>(xtc.threshold[row]) * static_cast<double>(total);
            unsigned int c = 0, lowest = UINT_MAX;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (v == v && order_key(v) >= tau &&
                    static_cast<double>(__float2ull_rn(expf(__fdiv_rn(__fsub_rn(v, m), temp)) * MASS_SCALE)) >= thr)
                    ++c, lowest = min(lowest, order_key(v));
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                c += __shfl_xor_sync(0xffffffffu, c, o);
                lowest = min(lowest, __shfl_xor_sync(0xffffffffu, lowest, o));
            }
            if (lane == 0 && c) atomicAdd(&x_count, c), atomicMin(&x_min, lowest);
            cluster.sync();
            if (threadIdx.x == 0) {
                unsigned int cnt = 0, lo = UINT_MAX;
                for (int r = 0; r < C; ++r) cnt += *cluster.map_shared_rank(&x_count, r), lo = min(lo, *cluster.map_shared_rank(&x_min, r));
                x_hi = cnt >= 2 ? lo : UINT_MAX;  // ties at the least likely value stay
            }
            __syncthreads();
            const uint32_t hi = x_hi;
            if (hi != UINT_MAX) {
                for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS)
                    if (xs[i] == xs[i] && order_key(xs[i]) > hi) xs[i] = NAN;
                __syncthreads();
            }
        }
    }
    mine = Best{-INFINITY, INT_MAX};
    TL_ROW_GUMBEL_PASS(0u);
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
        if constexpr (MASK) {
            if (con[row].mask && positions[row] > 0) con[row].state = constraint_advance(con[row], token);
        }
    }
    cluster.sync();
}

template <typename T, int LEVELS, bool PEN, bool MASK, bool XTC>
int launch_sample_t(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                    const int32_t *positions, int32_t *out, int rows, int vocab, int cluster, int slice, int vec, const Penalties &pen,
                    tl_constraint_row *con, const Xtc &xtc, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(sample_kernel<T, LEVELS, PEN, MASK, XTC>, cudaFuncAttributeMaxDynamicSharedMemorySize, SAMPLE_MAX_SMEM) != cudaSuccess)
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
        cudaLaunchKernelEx(&cfg, sample_kernel<T, LEVELS, PEN, MASK, XTC>, x, temperature, top_k, top_p, seed, positions, out, vocab, slice, vec, pen, con, xtc);
    if (e != cudaSuccess) return fail(TL_ECUDA, "sample: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("sample");
    return TL_OK;
}

template <bool PEN, bool MASK, bool XTC = false>
int launch_sample_any(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                      const int32_t *positions, int32_t *out, int rows, int vocab, int dtype, const Penalties &pen, tl_constraint_row *con,
                      cudaStream_t st, const Xtc &xtc = Xtc{}) {
    if (rows == 0) return TL_OK;
    int cluster = 0, slice = 0;
    if (int e = sample_plan(vocab, &cluster, &slice)) return e;
    const int per16 = dtype == TL_F32 ? 4 : 8;
    const int vec = (vocab % per16 == 0 && aligned16(logits)) ? 1 : 0;
    switch (dtype) {
        case TL_F32:
            return launch_sample_t<float, 4, PEN, MASK, XTC>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster, slice,
                                                             vec, pen, con, xtc, st);
        case TL_F16:
            return launch_sample_t<__half, 4, PEN, MASK, XTC>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster,
                                                              slice, vec, pen, con, xtc, st);
        case TL_BF16:  // a raw bf16 value's key has 16 significant bits: two levels.  A penalty rewrites the staged values
                       // (x / r, x * r, x - f c, x - pres) into arbitrary fp32 values: four levels, or tau would stop
                       // at a 16-bit prefix and keep every entry of its bucket below x_(k) or v*
            return launch_sample_t<__nv_bfloat16, PEN ? 4 : 2, PEN, MASK, XTC>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab,
                                                                      cluster, slice, vec, pen, con, xtc, st);
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
    return launch_sample_any<false, false>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, Penalties{}, nullptr, st);
}

int launch_sample_penalized(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                            const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                            const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability, int32_t *out,
                            int rows, int vocab, int dtype, cudaStream_t st) {
    const Penalties pen{repetition, presence, frequency, min_p, state, (vocab % 4 == 0 && aligned16(state)) ? 1 : 0};
    if (xtc_threshold)
        return launch_sample_any<true, false, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, nullptr, st,
                                                    Xtc{xtc_threshold, xtc_probability});
    return launch_sample_any<true, false>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, nullptr, st);
}

int launch_sample_constrained(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                              const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                              const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability,
                              tl_constraint_row *constraints, int32_t *out, int rows, int vocab, int dtype, cudaStream_t st) {
    if (!state)
        return launch_sample_any<false, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, Penalties{},
                                              constraints, st);
    const Penalties pen{repetition, presence, frequency, min_p, state, (vocab % 4 == 0 && aligned16(state)) ? 1 : 0};
    if (xtc_threshold)
        return launch_sample_any<true, true, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, constraints,
                                                   st, Xtc{xtc_threshold, xtc_probability});
    return launch_sample_any<true, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, constraints, st);
}

}  // namespace tl
