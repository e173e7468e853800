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
//
// The truncation forms (TRUNC, DESIGN.md section 25; always with XTC's code, which they skip when no XTC array is
// given) add top-n-sigma, locally typical sampling and Mirostat 2.0 after min-p.  Top-n-sigma is two fixed-order double
// reductions (mean, then squared deviations) and one more lower bound on tau.  Typical sums the kept T = 1 masses and
// sum e_i z_i, runs up to four radix levels over the key of d_i = |z_bar - z_i| ascending in the same bins, and sends
// the kept entries above the boundary d to NaN.  Mirostat sums the tempered masses, sends every entry below S 2^-mu to
// NaN, sums the rest, and after the draw rank 0 reads the token's value over distributed shared memory to update mu.
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

// Per-row arrays of the truncation forms (DESIGN.md section 25); any of them may be null when no row uses it.  Mirostat
// is on for a row with mirostat_tau > 0, and mu (fp32, one per row) is then read and, at position > 0, written.
struct Trunc {
    const float *typical_p, *top_n_sigma, *mirostat_tau, *mirostat_eta;
    float *mu;
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

// TRUNC: the cluster totals of a pair of per-thread partial sums, added in one fixed order (each thread's entries, a
// warp butterfly, the warps in order, the ranks in order), so every CTA of the cluster gets the same bits in every
// launch; integer pairs give the same total in any order.  `pub` is published to the other CTAs: each reduction of a
// launch uses a slot of its own, since a slower CTA may still read the previous one after this CTA went on.
template <typename V>
struct Pair {
    V a, b;
};
template <typename V>
__device__ __forceinline__ Pair<V> cluster_sum(cg::cluster_group &cluster, Pair<V> p, Pair<V> *w, Pair<V> *pub, Pair<V> *res, int C) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) p.a += __shfl_xor_sync(0xffffffffu, p.a, o), p.b += __shfl_xor_sync(0xffffffffu, p.b, o);
    if (lane == 0) w[warp] = p;
    __syncthreads();
    if (threadIdx.x == 0) {
        Pair<V> s{0, 0};
        for (int i = 0; i < SAMPLE_WARPS; ++i) s.a += w[i].a, s.b += w[i].b;
        *pub = s;
    }
    cluster.sync();
    if (threadIdx.x == 0) {
        Pair<V> t{0, 0};
        for (int r = 0; r < C; ++r) {
            const Pair<V> q = *cluster.map_shared_rank(pub, r);
            t.a += q.a, t.b += q.b;
        }
        *res = t;
    }
    __syncthreads();
    return *res;
}

template <typename T, int LEVELS, bool PEN, bool MASK, bool XTC, bool TRUNC = false>
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(const T *__restrict__ logits, const float *__restrict__ temperature,
                                                                const int32_t *__restrict__ top_k, const float *__restrict__ top_p,
                                                                const int64_t *__restrict__ seed, const int32_t *__restrict__ positions,
                                                                int32_t *__restrict__ out, int vocab, int slice, int vec, Penalties pen,
                                                                tl_constraint_row *con, Xtc xtc, Trunc trn) {
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
    // ---- 2b. truncation (TRUNC, DESIGN.md section 25): top-n-sigma joins tau, typical sends the kept entries it drops
    //      to NaN, and Mirostat replaces the keep set with its own (NaN outside it, tau = 0)
    // (nothing of it stays in registers across the draw: rank 0 reads mu, S_K and the parameters again to update mu)
    __shared__ unsigned long long s_miro_kept;  // Mirostat: the kept mass S_K (unused by the other forms)
    if constexpr (TRUNC) {
        __shared__ Pair<double> tr_wd[SAMPLE_WARPS], tr_pd[2], tr_rd;
        __shared__ Pair<unsigned long long> tr_wu[SAMPLE_WARPS], tr_pu[3], tr_ru;
        __shared__ uint32_t s_dprefix;
        __shared__ unsigned long long s_dbelow;
        __shared__ double s_dwant;
        const bool miro = trn.mirostat_tau && trn.mirostat_tau[row] > 0.f;
        const float nsig = trn.top_n_sigma && !miro ? trn.top_n_sigma[row] : 0.f;
        const float typ = trn.typical_p && !miro ? trn.typical_p[row] : 1.f;
        if (nsig > 0.f) {  // x >= m - n sigma over the finite entries (population sigma), the bound rounded up to fp32
            double sx = 0, cnt = 0;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (isfinite(v)) sx += v, cnt += 1;
            }
            const Pair<double> t1 = cluster_sum(cluster, Pair<double>{sx, cnt}, tr_wd, &tr_pd[0], &tr_rd, C);
            const double mean = t1.a / t1.b;
            double sq = 0;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (isfinite(v)) sq += (static_cast<double>(v) - mean) * (static_cast<double>(v) - mean);
            }
            const Pair<double> t2 = cluster_sum(cluster, Pair<double>{sq, 0.0}, tr_wd, &tr_pd[1], &tr_rd, C);
            const double bound = static_cast<double>(m) - static_cast<double>(nsig) * sqrt(t2.a / t1.b);
            tau = max(tau, order_key(__double2float_ru(bound)));
        }
        if (typ > 0.f && typ < 1.f) {
            // the T = 1 masses of the keep set K: S_K and sum e_i z_i (z_i = x_i - m, 2^-4 fixed point, signed), so
            // z_bar = sum p_i z_i and d_i = |z_bar - z_i| = |-ln p_i - H|
            unsigned long long se = 0, sz = 0;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (v == v && order_key(v) >= tau) {
                    const unsigned long long e = __float2ull_rn(expf(v - m) * MASS_SCALE);
                    se += e;
                    if (e) sz += static_cast<unsigned long long>(__double2ll_rn(static_cast<double>(e) * static_cast<double>(v - m) * 16.0));
                }
            }
            const Pair<unsigned long long> tk = cluster_sum(cluster, Pair<unsigned long long>{se, sz}, tr_wu, &tr_pu[0], &tr_ru, C);
            const double zbar = static_cast<double>(static_cast<long long>(tk.b)) * 0.0625 / static_cast<double>(tk.a);
            // every CTA has read the keep threshold's bins (the barrier above): both buffers are free again
            for (int i = threadIdx.x; i < 2 * BINS; i += SAMPLE_THREADS) (&h_count[0][0])[i] = 0, (&h_mass[0][0])[i] = 0;
            if (threadIdx.x == 0) s_dprefix = 0, s_dbelow = 0, s_dwant = static_cast<double>(typ) * static_cast<double>(tk.a);
            __syncthreads();
            // d* = the smallest key of d with mass(key <= d*) >= typical_p S_K: 4 radix levels, ascending
            for (int level = 0; level < 4; ++level) {
                const int buf = level & 1;
                const int shift = 24 - 8 * level;
                const uint32_t prefix = s_dprefix;
                for (int base = warp * 32; base < n; base += SAMPLE_THREADS) {
                    const int i = base + lane;
                    int bin = -1;
                    unsigned long long e = 0;
                    if (i < n) {
                        const float v = xs[i];
                        if (v == v && order_key(v) >= tau) {
                            const uint32_t dk = __float_as_uint(__double2float_rn(fabs(zbar - static_cast<double>(v - m))));
                            if (level == 0 || (dk >> (shift + 8)) == (prefix >> (shift + 8))) {
                                bin = static_cast<int>((dk >> shift) & 0xffu);
                                e = __float2ull_rn(expf(v - m) * MASS_SCALE);
                            }
                        }
                    }
                    bin_add(h_count[buf], h_mass[buf], bin, e, true);
                }
                cluster.sync();
                if (threadIdx.x < BINS) {
                    unsigned long long s = 0;
                    for (int r = 0; r < C; ++r) s += *cluster.map_shared_rank(&h_mass[buf][threadIdx.x], r);
                    t_mass[threadIdx.x] = s;
                }
                for (int i = threadIdx.x; i < BINS; i += SAMPLE_THREADS) h_count[buf ^ 1][i] = 0, h_mass[buf ^ 1][i] = 0;
                __syncthreads();
                if (warp == 0) {  // lane owns bins 8 lane .. 8 lane + 7; prefix sums from bin 0 up
                    unsigned long long s[8], ls = 0;
#pragma unroll
                    for (int j = 0; j < 8; ++j) s[j] = t_mass[8 * lane + j], ls += s[j];
                    unsigned long long incl = ls;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned long long up = __shfl_up_sync(0xffffffffu, incl, o);
                        if (lane >= o) incl += up;
                    }
                    const double want = s_dwant;  // typical_p S_K
                    unsigned long long below = s_dbelow + (incl - ls);
                    int hit = -1;
                    unsigned long long hit_below = 0;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        if (hit < 0 && static_cast<double>(below + s[j]) >= want) hit = 8 * lane + j, hit_below = below;
                        below += s[j];
                    }
                    const unsigned hb = __ballot_sync(0xffffffffu, hit >= 0);
                    // the crossing bin adds mass, so it holds an entry; no crossing cannot happen (want < S_K)
                    if (hb && lane == __ffs(hb) - 1) s_dprefix = prefix | (static_cast<uint32_t>(hit) << shift), s_dbelow = hit_below;
                }
                __syncthreads();
            }
            const uint32_t dstar = s_dprefix;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (v == v && order_key(v) >= tau && __float_as_uint(__double2float_rn(fabs(zbar - static_cast<double>(v - m)))) > dstar)
                    xs[i] = NAN;
            }
            __syncthreads();
        }
        if (miro) {  // keep {e_i >= S 2^-mu} at the row's temperature, the maximum always (its e is 2^40)
            const float mu = trn.mu[row];
            unsigned long long se = 0;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (v == v) se += __float2ull_rn(expf(__fdiv_rn(__fsub_rn(v, m), temp)) * MASS_SCALE);
            }
            const unsigned long long S = cluster_sum(cluster, Pair<unsigned long long>{se, 0ull}, tr_wu, &tr_pu[1], &tr_ru, C).a;
            const double thr = fmin(static_cast<double>(S) * exp2(-static_cast<double>(mu)), static_cast<double>(MASS_SCALE));
            unsigned long long sk = 0;
            for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) {
                const float v = xs[i];
                if (v == v) {
                    const unsigned long long e = __float2ull_rn(expf(__fdiv_rn(__fsub_rn(v, m), temp)) * MASS_SCALE);
                    if (static_cast<double>(e) >= thr)
                        sk += e;
                    else
                        xs[i] = NAN;
                }
            }
            const unsigned long long kept = cluster_sum(cluster, Pair<unsigned long long>{sk, 0ull}, tr_wu, &tr_pu[2], &tr_ru, C).a;
            if (threadIdx.x == 0) s_miro_kept = kept;
            tau = 0;
        }
    }
    if constexpr (XTC) {
        __shared__ unsigned long long x_mass;
        __shared__ unsigned int x_count, x_min, x_hi;
        const uint4 w = philox4x32_10(make_uint4(0u, pos, 3u, 0u), k0, k1);
        const float u = static_cast<float>(2u * (w.x >> 9) + 1u) * 5.9604644775390625e-8f;
        if ((!TRUNC || (xtc.probability && !(trn.mirostat_tau && trn.mirostat_tau[row] > 0.f))) && u < xtc.probability[row]) {  // the same decision in every CTA of the cluster
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
        // the row maximum is always kept: INT_MAX cannot happen (TRUNC reads it back from shared memory rather than keep
        // a register across its passes)
        const int token = d.i == INT_MAX ? (TRUNC ? row_max.i : best.i) : d.i;
        out[row] = token;
        if constexpr (PEN) {
            if (positions[row] > 0) pen.state[static_cast<size_t>(row) * vocab + token] += 1;
        }
        if constexpr (MASK) {
            if (con[row].mask && positions[row] > 0) con[row].state = constraint_advance(con[row], token);
        }
        if constexpr (TRUNC) {  // mu' = mu - eta (s - tau), s = log2 S_K - log2 e_token: the surprise over the kept mass
            if (trn.mirostat_tau && trn.mirostat_tau[row] > 0.f && positions[row] > 0) {
                const int owner = token / slice;
                const float xt = *cluster.map_shared_rank(xs + (token - owner * slice), owner);
                const unsigned long long et = __float2ull_rn(expf(__fdiv_rn(__fsub_rn(xt, m), temp)) * MASS_SCALE);
                const double s = log2(static_cast<double>(s_miro_kept)) - log2(static_cast<double>(et));
                trn.mu[row] = static_cast<float>(static_cast<double>(trn.mu[row]) -
                                                 static_cast<double>(trn.mirostat_eta[row]) * (s - static_cast<double>(trn.mirostat_tau[row])));
            }
        }
    }
    cluster.sync();
}

template <typename T, int LEVELS, bool PEN, bool MASK, bool XTC, bool TRUNC>
int launch_sample_t(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                    const int32_t *positions, int32_t *out, int rows, int vocab, int cluster, int slice, int vec, const Penalties &pen,
                    tl_constraint_row *con, const Xtc &xtc, const Trunc &trn, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(sample_kernel<T, LEVELS, PEN, MASK, XTC, TRUNC>, cudaFuncAttributeMaxDynamicSharedMemorySize, SAMPLE_MAX_SMEM) != cudaSuccess)
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
        cudaLaunchKernelEx(&cfg, sample_kernel<T, LEVELS, PEN, MASK, XTC, TRUNC>, x, temperature, top_k, top_p, seed, positions, out, vocab, slice, vec, pen, con, xtc, trn);
    if (e != cudaSuccess) return fail(TL_ECUDA, "sample: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("sample");
    return TL_OK;
}

template <bool PEN, bool MASK, bool XTC = false, bool TRUNC = false>
int launch_sample_any(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                      const int32_t *positions, int32_t *out, int rows, int vocab, int dtype, const Penalties &pen, tl_constraint_row *con,
                      cudaStream_t st, const Xtc &xtc = Xtc{}, const Trunc &trn = Trunc{}) {
    if (rows == 0) return TL_OK;
    int cluster = 0, slice = 0;
    if (int e = sample_plan(vocab, &cluster, &slice)) return e;
    const int per16 = dtype == TL_F32 ? 4 : 8;
    const int vec = (vocab % per16 == 0 && aligned16(logits)) ? 1 : 0;
    switch (dtype) {
        case TL_F32:
            return launch_sample_t<float, 4, PEN, MASK, XTC, TRUNC>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster, slice,
                                                             vec, pen, con, xtc, trn, st);
        case TL_F16:
            return launch_sample_t<__half, 4, PEN, MASK, XTC, TRUNC>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, cluster,
                                                              slice, vec, pen, con, xtc, trn, st);
        case TL_BF16:  // a raw bf16 value's key has 16 significant bits: two levels.  A penalty rewrites the staged values
                       // (x / r, x * r, x - f c, x - pres) into arbitrary fp32 values: four levels, or tau would stop
                       // at a 16-bit prefix and keep every entry of its bucket below x_(k) or v*
            return launch_sample_t<__nv_bfloat16, PEN ? 4 : 2, PEN, MASK, XTC, TRUNC>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab,
                                                                      cluster, slice, vec, pen, con, xtc, trn, st);
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
                            const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability,
                            const float *typical_p, const float *top_n_sigma, const float *mirostat_tau, const float *mirostat_eta,
                            float *mirostat_mu, int32_t *out, int rows, int vocab, int dtype, cudaStream_t st) {
    const Penalties pen{repetition, presence, frequency, min_p, state, (vocab % 4 == 0 && aligned16(state)) ? 1 : 0};
    if (typical_p || top_n_sigma || mirostat_tau)
        return launch_sample_any<true, false, true, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, nullptr,
                                                          st, Xtc{xtc_threshold, xtc_probability},
                                                          Trunc{typical_p, top_n_sigma, mirostat_tau, mirostat_eta, mirostat_mu});
    if (xtc_threshold)
        return launch_sample_any<true, false, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, nullptr, st,
                                                    Xtc{xtc_threshold, xtc_probability});
    return launch_sample_any<true, false>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, nullptr, st);
}

int launch_sample_constrained(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                              const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                              const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability,
                              const float *typical_p, const float *top_n_sigma, const float *mirostat_tau, const float *mirostat_eta,
                              float *mirostat_mu, tl_constraint_row *constraints, int32_t *out, int rows, int vocab, int dtype, cudaStream_t st) {
    if (!state)
        return launch_sample_any<false, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, Penalties{},
                                              constraints, st);
    const Penalties pen{repetition, presence, frequency, min_p, state, (vocab % 4 == 0 && aligned16(state)) ? 1 : 0};
    if (typical_p || top_n_sigma || mirostat_tau)
        return launch_sample_any<true, true, true, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen,
                                                         constraints, st, Xtc{xtc_threshold, xtc_probability},
                                                         Trunc{typical_p, top_n_sigma, mirostat_tau, mirostat_eta, mirostat_mu});
    if (xtc_threshold)
        return launch_sample_any<true, true, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, constraints,
                                                   st, Xtc{xtc_threshold, xtc_probability});
    return launch_sample_any<true, true>(logits, temperature, top_k, top_p, seed, positions, out, rows, vocab, dtype, pen, constraints, st);
}

}  // namespace tl
