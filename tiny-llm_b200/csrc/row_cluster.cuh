// Building blocks of the kernels that reduce one logits row per thread-block cluster: tl_sample (sampling.cu),
// tl_speculative_sample (spec_sample.cu) and tl_logprobs (logprobs.cu).  A row of V entries is split over
// C = ceil(V / SAMPLE_SLICE_MIN) CTAs (at most SAMPLE_MAX_CLUSTER; sample_plan() in sampling.cu is the rule), each CTA
// stages its slice once in shared memory as fp32, and the CTAs merge integers and first-maximum-wins candidates over
// distributed shared memory.
#pragma once

#include <cstdint>

#include "common.cuh"

namespace tl {

namespace {

constexpr int SAMPLE_THREADS = 512;
constexpr int SAMPLE_WARPS = SAMPLE_THREADS / 32;
constexpr int SAMPLE_MAX_CLUSTER = 8;
constexpr int SAMPLE_SLICE_MIN = 4096;      // vocabulary entries per CTA before the cluster grows
constexpr int SAMPLE_MAX_SMEM = 200 << 10;  // staged slice: fp32, 51,200 entries per CTA
constexpr int BINS = 256;
constexpr float MASS_SCALE = 1099511627776.f;  // 2^40: e_i <= 1, so a row of < 2^23 entries sums below 2^63

struct Best {
    float v;
    int i;
};
__device__ __forceinline__ Best better(Best a, Best b) {
    return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;  // first maximum wins; NaN never does
}
__device__ __forceinline__ Best warp_best(Best m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = better(m, Best{__shfl_xor_sync(0xffffffffu, m.v, o), __shfl_xor_sync(0xffffffffu, m.i, o)});
    return m;
}

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

// Order-preserving key of a non-NaN float (-0 is folded onto +0 first, so equal values have equal keys).
__device__ __forceinline__ uint32_t order_key(float x) {
    const uint32_t b = __float_as_uint(x == 0.f ? 0.f : x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

template <typename T>
__device__ __forceinline__ void stage_slice(const T *__restrict__ src, float *xs, int n, bool vec) {
    if (vec) {  // the slice start and the row pitch are 16-byte aligned, n a multiple of 16 / sizeof(T)
        constexpr int PER = 16 / sizeof(T);
        for (int i = threadIdx.x * PER; i < n; i += SAMPLE_THREADS * PER) {
            const uint4 raw = *reinterpret_cast<const uint4 *>(src + i);
            if constexpr (sizeof(T) == 4) {
                *reinterpret_cast<float4 *>(xs + i) = make_float4(__uint_as_float(raw.x), __uint_as_float(raw.y), __uint_as_float(raw.z),
                                                                  __uint_as_float(raw.w));
            } else {
                const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = unpack2<T>(w[j]);
                    xs[i + 2 * j] = f.x;
                    xs[i + 2 * j + 1] = f.y;
                }
            }
        }
    } else {
        for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) xs[i] = to_f(src[i]);
    }
}

// One 32-bit broadcast per warp-uniform loop step: the lanes of `peers` share a bin; the lowest of them adds their
// count and mass to it.
__device__ __forceinline__ void bin_add(unsigned int *count, unsigned long long *mass, int bin, unsigned long long e, bool with_mass) {
    const unsigned active = __ballot_sync(0xffffffffu, bin >= 0);
    if (!active) return;
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    const int lane = threadIdx.x & 31;
    unsigned long long sum = 0;
    if (with_mass) {
#pragma unroll 8
        for (int j = 0; j < 32; ++j) {
            const unsigned long long v = __shfl_sync(0xffffffffu, e, j);
            if ((peers >> j) & 1u) sum += v;
        }
    }
    if (bin >= 0 && lane == __ffs(peers) - 1) {
        atomicAdd(&count[bin], static_cast<unsigned>(__popc(peers)));
        if (with_mass) atomicAdd(&mass[bin], sum);
    }
}

}  // namespace

}  // namespace tl

// The keep threshold and the Gumbel pass of a staged row (DESIGN.md section 8, steps 2 and 3), shared by tl_sample and
// tl_speculative_sample.  They are statement macros over the caller's names, not functions: expanded in place, the
// existing sample_kernel instantiations compile to the instructions they had before the speculative kernel shared them
// (an inlined function moved their reconvergence points).
//
// TL_ROW_KEEP_THRESHOLD(LEVELS) leaves tau in s_prefix: the row keeps its non-NaN entries with order_key(x) >= tau,
// tau = max(x_(k), v*).  It reads xs, n (this CTA's staged slice), m (the row's finite maximum), top_k[row],
// top_p[row], vocab, cluster, C, warp, lane and the shared scratch h_count / h_mass [2][BINS] (zero on entry),
// t_count / t_mass [BINS], s_prefix, s_k_on, s_p_on, s_count_above, s_mass_above, s_p_mass, s_bk, s_bp, s_bk_above,
// s_bp_above.  Every CTA of the cluster takes the same branches and barriers and ends with the same tau.
#define TL_ROW_KEEP_THRESHOLD(LEVELS) \
    do {                              \
    if (threadIdx.x == 0) {                                                                                                              \
        const int k = top_k[row];                                                                                                        \
        const float p = top_p[row];                                                                                                      \
        s_k_on = k > 0 && k < vocab;                                                                                                     \
        s_p_on = p > 0.f && p < 1.f;                                                                                                     \
        s_prefix = 0;                                                                                                                    \
        s_count_above = 0;                                                                                                               \
        s_mass_above = 0;                                                                                                                \
    }                                                                                                                                    \
    __syncthreads();                                                                                                                     \
    const unsigned int k_want = static_cast<unsigned int>(top_k[row]);                                                                   \
    const float p_want = top_p[row];                                                                                                     \
    for (int level = 0; level < LEVELS && (s_k_on || s_p_on); ++level) {                                                                 \
        const int buf = level & 1;                                                                                                       \
        const int shift = 24 - 8 * level;                                                                                                \
        const uint32_t prefix = s_prefix;                                                                                                \
        const bool with_mass = s_p_on;                                                                                                   \
        unsigned int *cnt = h_count[buf];                                                                                                \
        unsigned long long *mass = h_mass[buf];                                                                                          \
        for (int base = warp * 32; base < n; base += SAMPLE_THREADS) {                                                                   \
            const int i = base + lane;                                                                                                   \
            int bin = -1;                                                                                                                \
            unsigned long long e = 0;                                                                                                    \
            if (i < n) {                                                                                                                 \
                const float x = xs[i];                                                                                                   \
                if (x == x) {                                                                                                            \
                    const uint32_t key = order_key(x);                                                                                   \
                    if (level == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) {                                                 \
                        bin = static_cast<int>((key >> shift) & 0xffu);                                                                  \
                        if (with_mass) e = static_cast<unsigned long long>(__float2ull_rn(expf(x - m) * MASS_SCALE));                    \
                    }                                                                                                                    \
                }                                                                                                                        \
            }                                                                                                                            \
            bin_add(cnt, mass, bin, e, with_mass);                                                                                       \
        }                                                                                                                                \
        cluster.sync();                                                                                                                  \
        if (threadIdx.x < BINS) {                                                                                                        \
            unsigned int c = 0;                                                                                                          \
            unsigned long long s = 0;                                                                                                    \
            for (int r = 0; r < C; ++r) {                                                                                                \
                c += *cluster.map_shared_rank(&cnt[threadIdx.x], r);                                                                     \
                if (with_mass) s += *cluster.map_shared_rank(&mass[threadIdx.x], r);                                                     \
            }                                                                                                                            \
            t_count[threadIdx.x] = c;                                                                                                    \
            t_mass[threadIdx.x] = s;                                                                                                     \
        }                                                                                                                                \
        /* the buffer of the next level is free again: every CTA read it (level - 1) before this level's barrier */                      \
        for (int i = threadIdx.x; i < BINS; i += SAMPLE_THREADS) h_count[buf ^ 1][i] = 0, h_mass[buf ^ 1][i] = 0;                        \
        __syncthreads();                                                                                                                 \
        if (warp == 0) {                                                                                                                 \
            /* lane owns bins 8 lane .. 8 lane + 7; suffix sums from the top bin down */                                                 \
            unsigned int c[8];                                                                                                           \
            unsigned long long s[8];                                                                                                     \
            unsigned int lc = 0;                                                                                                         \
            unsigned long long ls = 0;                                                                                                   \
_Pragma("unroll")                                                                                                                        \
            for (int j = 0; j < 8; ++j) c[j] = t_count[8 * lane + j], s[j] = t_mass[8 * lane + j], lc += c[j], ls += s[j];               \
            unsigned int ca = lc;                                                                                                        \
            unsigned long long sa = ls;                                                                                                  \
_Pragma("unroll")                                                                                                                        \
            for (int o = 1; o < 32; o <<= 1) {                                                                                           \
                const unsigned int oc = __shfl_down_sync(0xffffffffu, ca, o);                                                            \
                const unsigned long long os = __shfl_down_sync(0xffffffffu, sa, o);                                                      \
                if (lane + o < 32) ca += oc, sa += os;                                                                                   \
            }                                                                                                                            \
            const unsigned int total_c = __shfl_sync(0xffffffffu, ca, 0);                                                                \
            const unsigned long long total_s = __shfl_sync(0xffffffffu, sa, 0);                                                          \
            if (level == 0 && lane == 0) {                                                                                               \
                if (total_c < k_want) s_k_on = 0;  /* fewer non-NaN entries than k: top-k keeps them all */                              \
                s_p_mass = static_cast<double>(p_want) * static_cast<double>(total_s);                                                   \
            }                                                                                                                            \
            __syncwarp();                                                                                                                \
            const bool k_on = s_k_on, p_on = s_p_on;                                                                                     \
            const double p_mass = s_p_mass;                                                                                              \
            unsigned int above_c = s_count_above + (ca - lc);                                                                            \
            unsigned long long above_s = s_mass_above + (sa - ls);                                                                       \
            int bk = -1, bp = -1;                                                                                                        \
            unsigned int bk_above = 0;                                                                                                   \
            unsigned long long bp_above = 0;                                                                                             \
_Pragma("unroll")                                                                                                                        \
            for (int j = 7; j >= 0; --j) {                                                                                               \
                if (k_on && bk < 0 && above_c < k_want && k_want <= above_c + c[j]) bk = 8 * lane + j, bk_above = above_c;               \
                if (p_on && c[j] > 0 && static_cast<double>(above_s) < p_mass) bp = 8 * lane + j, bp_above = above_s;  /* lowest wins */ \
                above_c += c[j];                                                                                                         \
                above_s += s[j];                                                                                                         \
            }                                                                                                                            \
            const unsigned kb = __ballot_sync(0xffffffffu, bk >= 0);                                                                     \
            const unsigned pb = __ballot_sync(0xffffffffu, bp >= 0);                                                                     \
            if (kb && lane == __ffs(kb) - 1) s_bk = bk, s_bk_above = bk_above;                                                           \
            if (pb && lane == __ffs(pb) - 1) s_bp = bp, s_bp_above = bp_above;                                                           \
            __syncwarp();                                                                                                                \
            if (lane == 0) {                                                                                                             \
                const int kbin = k_on ? s_bk : -1, pbin = p_on ? s_bp : -1;                                                              \
                const int bin = max(kbin, pbin);  /* tau = max(x_(k), v*): the higher bin holds it */                                    \
                /* bin < 0: level 0 turned top-k off and top-p is off, so tau stays 0 and every non-NaN entry is kept */                 \
                s_k_on = bin >= 0 && kbin == bin;                                                                                        \
                s_p_on = bin >= 0 && pbin == bin;                                                                                        \
                if (bin >= 0) s_prefix = prefix | (static_cast<uint32_t>(bin) << shift);                                                 \
                s_count_above = s_k_on ? s_bk_above : 0;                                                                                 \
                s_mass_above = s_p_on ? s_bp_above : 0;                                                                                  \
            }                                                                                                                            \
        }                                                                                                                                \
        __syncthreads();                                                                                                                 \
    }                                                                                                                                    \
    } while (0)

// TL_ROW_GUMBEL_PASS(STREAM) folds into `mine` this thread's candidates (x_i - m) / temp + g_i over the kept entries
// (order_key(x) >= tau) of the slice starting at row index `begin`; g_i is the Gumbel noise of word i % 4 of
// Philox4x32-10 at counter (i >> 2, pos, STREAM, 0) under the key (k0, k1).  Stream 0 is the draw of tl_sample.
#define TL_ROW_GUMBEL_PASS(STREAM) \
    do {                           \
    for (int g = threadIdx.x * 4; g < n; g += SAMPLE_THREADS * 4) {                                                  \
        bool any = false;                                                                                            \
        float x[4];                                                                                                  \
_Pragma("unroll")                                                                                                    \
        for (int j = 0; j < 4; ++j) {                                                                                \
            x[j] = g + j < n ? xs[g + j] : NAN;                                                                      \
            any |= x[j] == x[j] && order_key(x[j]) >= tau;                                                           \
        }                                                                                                            \
        if (!any) continue;                                                                                          \
        const uint4 w = philox4x32_10(make_uint4(static_cast<uint32_t>(begin + g) >> 2, pos, (STREAM), 0u), k0, k1); \
        const uint32_t ws[4] = {w.x, w.y, w.z, w.w};                                                                 \
_Pragma("unroll")                                                                                                    \
        for (int j = 0; j < 4; ++j)                                                                                  \
            if (x[j] == x[j] && order_key(x[j]) >= tau)                                                              \
                mine = better(mine, Best{__fdiv_rn(__fsub_rn(x[j], m), temp) + gumbel(ws[j]), begin + g + j});       \
    }                                                                                                                \
    } while (0)
