// Fused decode attention for the Week-3 Qwen3 model (bf16, paged KV, L == 1): one launch does
// q/k RMSNorm -> RoPE -> K/V append -> paged GQA attention for every (request, KV head), i.e. the
// operator sequence rms_norm x2 -> rope x2 -> paged_cache_update x2 -> paged_attention of
// src/tiny_llm_ref/qwen3_week3.py:62-105 with the kernel arithmetic of
// src/extensions_ref/src/paged_attention.metal:108-248, every rounding point kept.
//
// A request may carry R <= 8 consecutive query rows (the verify pass of speculative decoding): row j
// is the decode step of one more token, so its output equals, bit for bit, R = 1 run on that row alone
// with rows < j already appended (see mk_attention).
//
// (An earlier whole-step persistent kernel in this file lost to the CUDA-graph + programmatic-dependent-launch
// path - its time went to grid barriers and staging - and was retired.)
#include <algorithm>
#include <stdlib.h>
#include <math_constants.h>

#include "common.cuh"
#include "kernels.h"
#include "w4a16_item.cuh"
#include "trace.cuh"

namespace tl {

constexpr int MK_WARPS = 16;
constexpr int MK_THREADS = MK_WARPS * 32;
constexpr float MK_LOG2E = 1.44269504089f;
constexpr float MK_NEG = -1e30f;
constexpr int MK_MAX_ROWS = 8;  // query rows per request

typedef __nv_bfloat16 bf16;

// Launch-constant arguments (plain pointers and sizes; filled by launch_decode_attention_fused).
struct MkLayer {
    const void *q_norm, *k_norm;  // bf16 [D]
    void *k_pages, *v_pages;      // bf16 [P, Hkv, page, D]
    const int32_t *table;         // int32 [B, max_pages], -1 padded
};
struct MkArgs {
    int B, Hq, Hkv, D;
    int R, HR;                              // query rows per request; staged (head, row) pairs, max(4, G R)
    float eps, attn_scale;
    int page_size, max_pages, num_pages;
    const int32_t *offsets, *context_lens;  // [B R]: RoPE positions, post-append lengths
    const void *qkv;                        // bf16 [B R, (Hq + 2 Hkv) D]
    void *y;                                // bf16 [B R, Hq D]
    float *attn_ws;                         // [B*R*Hq*nsplit*(D+2)] when nsplit > 1
    int nsplit, tokens_per_split;
    const double *rope_inv_freq;            // [D/2]
};

__device__ __forceinline__ float mk_bf(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float mk_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

struct Prof {
    __device__ __forceinline__ void stamp(int) {}
};

// --------------------------------------------------------------- attention --
// One CTA per (request, kv head, split).  The phase is pure latency (8 CTAs x 64 KB of
// K/V at context 128), so it is organised around dependent round trips and wide parallelism, not
// bandwidth.  Per round of up to MK_ATT_TOK tokens:
//   A  page ids of the round -> shared; the first q-path task of each warp already holds its norm
//      weights and rope frequencies in registers (loaded before anything else)
//   B  cp.async ALL K/V rows of the round into shared memory (row stride 528 B: bank spread)
//   C  while those are in flight: q/k RMSNorm + RoPE (rounded like rms_norm -> rope), V copy, for
//      the (G + 2) R head rows of the request's R query rows
//   S  scores = Q K^T on the tensor cores: mma.sync m16n8k16, A = the G R (head, row) pairs (rows
//      past them zero; a second m16 block beyond 16 pairs), B = K rows straight from shared memory;
//      8 tokens per MMA tile, 16 warps
//   V  out = P V on CUDA cores with fp32 probabilities: thread = (pair, 8 dims, token subset)
//   then the running (max, sum, out) of thread (pair, dim) absorbs the round.
// R rows: row j's keys end at context_lens[j] (causal mask, applied like the slots past the round's
// end); the new K/V rows of all R rows are staged from shared memory, never re-read from the pages
// another CTA is writing in the same launch.  A row takes part in exactly the rounds the R = 1 kernel
// runs for it alone: its later rounds leave its running state untouched.
constexpr int MK_ATT_TOK = 256;     // K/V rows staged per round
constexpr int MK_KV_STRIDE = 528;   // bytes per staged token: K row | V row | 16 B pad

// dynamic shared memory for HR staged (head, row) pairs and R rows
__host__ __device__ constexpr size_t mk_att_bytes(int HR, int R) {
    return static_cast<size_t>(HR) * 128 * 2 + 2 * static_cast<size_t>(R) * 128 * 2 + static_cast<size_t>(HR) * MK_ATT_TOK * 4 +
           static_cast<size_t>(HR) * 64 * 4 + (MK_ATT_TOK + 4) * 4 + static_cast<size_t>(MK_ATT_TOK) * MK_KV_STRIDE;
}

// beyond 16 pairs the running (max, sum, out) of the output threads lives in shared memory, [HR][16][m | l | out[8]]
// (in registers it would spill)
__host__ __device__ constexpr size_t mk_state_bytes(int HR) { return static_cast<size_t>(HR) * 16 * 10 * 4; }

__device__ __forceinline__ void mk_cp16(void *dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))), "l"(src) : "memory");
}

// DEPWAIT (stand-alone kernel under programmatic dependent launch): everything that does not read
// this step's qkv row - page ids, the K/V rows of older tokens - is requested BEFORE
// griddepcontrol.wait, i.e. while the qkv projection is still draining.
// NP: (head, row) pairs per output thread, >= ceil(G R / 4); NP == 1 exactly when R == 1 (the decode step).
template <bool DEPWAIT, int NP>
__device__ void mk_attention(const MkArgs &a, const MkLayer &l, unsigned char *dyn, Prof &prof) {
    constexpr int MB = NP > 4 ? 2 : 1;   // m16 blocks of the score MMA
    constexpr bool HI8 = NP > 2;         // rows g + 8 of a block carry pairs
    constexpr bool SMEM_STATE = NP > 4;  // running state in shared memory (mk_state_bytes)
    constexpr int NPR = SMEM_STATE ? 1 : NP;
    // NP == 1 is the single-row step (R == 1, G <= 4): its row count and shared layout are compile-time
    const int D = a.D, G = a.Hq / a.Hkv, R = NP == 1 ? 1 : a.R, GR = G * R;
    const int HR = NP == 1 ? 4 : a.HR;  // max(4, G R)
    const int items = a.B * a.Hkv * a.nsplit;
    if (static_cast<int>(blockIdx.x) >= items) return;
    const int split = blockIdx.x % a.nsplit;
    const int kvh = (blockIdx.x / a.nsplit) % a.Hkv;
    const int b = blockIdx.x / (a.nsplit * a.Hkv);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qkv_w = (a.Hq + 2 * a.Hkv) * D;

    bf16 *q_s = reinterpret_cast<bf16 *>(dyn);                      // [HR][128] rope output (unscaled), pair = row * G + head
    bf16 *k_cur = q_s + HR * 128;                                   // [R][128] new tokens
    bf16 *v_cur = k_cur + R * 128;                                  // [R][128]
    float *s_s = reinterpret_cast<float *>(v_cur + R * 128);        // [HR][MK_ATT_TOK] scores, then probabilities
    float *st_s = s_s + HR * MK_ATT_TOK;                            // per (pair, tile): max [HR][32], then sum [HR][32]
    int *pg_s = reinterpret_cast<int *>(st_s + HR * 64);            // page ids of the round
    unsigned char *kv_s = reinterpret_cast<unsigned char *>(pg_s + MK_ATT_TOK + 4);  // [MK_ATT_TOK][528]
    float *state_s = reinterpret_cast<float *>(kv_s + MK_ATT_TOK * MK_KV_STRIDE);    // SMEM_STATE only

    // ---- head rows for the q path: task = (row j, head slot w), w < G query heads, G the k head, G + 1 the v head
    const int ntask = (G + 2) * R;
    float re[2] = {0.f, 0.f}, im[2] = {0.f, 0.f}, wre[2] = {0.f, 0.f}, wim[2] = {0.f, 0.f};
    double freq[2] = {0.0, 0.0};
    int position = 0;
    auto load_w = [&](int tk) {  // norm weights, rope frequencies and position of task tk
        const int w = NP == 1 ? tk : tk % (G + 2);
        const bool is_q = w < G, is_k = w == G;
        const bf16 *wt = static_cast<const bf16 *>(is_q ? l.q_norm : l.k_norm);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (is_q || is_k) {
                wre[h] = mk_bf(wt[lane + 32 * h]);
                wim[h] = mk_bf(wt[lane + 32 * h + 64]);
                freq[h] = a.rope_inv_freq[lane + 32 * h];
            }
        }
        position = a.offsets[b * R + (NP == 1 ? 0 : tk / (G + 2))];
    };
    auto load_q = [&](int tk) {
        const int w = NP == 1 ? tk : tk % (G + 2);
        const int head_off = w < G ? (kvh * G + w) * D : (w == G ? (a.Hq + kvh) * D : (a.Hq + a.Hkv + kvh) * D);
        const bf16 *src = static_cast<const bf16 *>(a.qkv) + static_cast<size_t>(b * R + (NP == 1 ? 0 : tk / (G + 2))) * qkv_w + head_off;
#pragma unroll
        for (int h = 0; h < 2; ++h) {  // lane owns pairs (i, i+64) for i = lane, lane+32   (D == 128)
            re[h] = mk_bf(ld_cg(src + lane + 32 * h));
            im[h] = mk_bf(ld_cg(src + lane + 32 * h + 64));
        }
    };
    if (warp < ntask) {
        load_w(warp);
        if (!DEPWAIT) load_q(warp);
    }
    // page ids of the first round do not need the context length: request them together with it
    const int begin = split * a.tokens_per_split;
    {
        const int lp_first = begin / a.page_size + static_cast<int>(threadIdx.x);
        if (static_cast<int>(threadIdx.x) <= MK_ATT_TOK && lp_first < a.max_pages)
            pg_s[threadIdx.x] = l.table[static_cast<size_t>(b) * a.max_pages + lp_first];
    }
    const int cap = a.max_pages * a.page_size;
    auto row_end = [&](int j) { return min(min(a.context_lens[b * R + j], cap), begin + a.tokens_per_split); };
    // the rows' contexts are consecutive: the new tokens are [new_lo, new_hi], the last row sees the most keys
    const int ctx_lo = min(a.context_lens[b * R], cap), ctx_hi = min(a.context_lens[b * R + R - 1], cap);
    const int end = min(ctx_hi, begin + a.tokens_per_split);
    const int new_lo = ctx_lo - 1, new_hi = ctx_hi - 1;
    const int gidx = warp * 2 + (lane >> 4), c8 = lane & 15;   // copy mapping: lane group of 16 per token row
    const int g = lane >> 2, t = lane & 3;                      // MMA fragment coordinates
    const int oh = threadIdx.x >> 7;                            // first pair whose output this thread helps to form
    const int sub = threadIdx.x & 7, d8 = (threadIdx.x >> 3) & 15;
    const float scale2 = a.attn_scale * MK_LOG2E;
    // keys visible to the score rows of this lane ([mb][g / g + 8]) and to the output pairs of this thread
    int s_end[MB][2];
#pragma unroll
    for (int mb = 0; mb < MB; ++mb)
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
            const int p = mb * 16 + hf * 8 + g;
            s_end[mb][hf] = NP == 1 ? (p < GR ? end : 0) : (p < GR ? row_end(p / G) : 0);
        }
    int v_end[NP];
    float m_run[NPR], l_run[NPR], o_run[NPR][8];  // kept by the (threadIdx & 7) == 0 lanes
#pragma unroll
    for (int i = 0; i < NP; ++i) {
        const int p = oh + 4 * i;
        v_end[i] = NP == 1 ? end : (p < GR ? row_end(p / G) : 0);
        if constexpr (SMEM_STATE) {
            if (p < GR && sub == 0) {
                float *S = state_s + (p * 16 + d8) * 10;
                S[0] = MK_NEG, S[1] = 0.f;
#pragma unroll
                for (int k = 0; k < 8; ++k) S[2 + k] = 0.f;
            }
        } else {
            m_run[i] = MK_NEG, l_run[i] = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) o_run[i][k] = 0.f;
        }
    }
    prof.stamp(50001);

    for (int rb = begin; rb < end || rb == begin; rb += MK_ATT_TOK) {  // one pass even for an empty split (q path, barriers)
        const int rend = min(end, rb + MK_ATT_TOK);
        const int cnt = max(rend - rb, 0);
        const int lp0 = rb / a.page_size;
        const int npg = cnt > 0 ? (rend - 1) / a.page_size - lp0 + 1 : 0;
        if (rb != begin && static_cast<int>(threadIdx.x) < npg) pg_s[threadIdx.x] = l.table[static_cast<size_t>(b) * a.max_pages + lp0 + threadIdx.x];
        __syncthreads();
        prof.stamp(50002);
        // ---- B: all K/V rows of the round in flight
        {
            int lpi = (rb + gidx) / a.page_size;        // logical page and row inside it of this lane group's next token,
            int row = rb + gidx - lpi * a.page_size;    // advanced by 32 tokens per step without further divisions
            const size_t head_rows = static_cast<size_t>(a.Hkv) * a.page_size;
            unsigned char *dst = kv_s + gidx * MK_KV_STRIDE + c8 * 16;
#pragma unroll
            for (int j = 0; j < MK_ATT_TOK / 32; ++j) {
                const int tok = rb + j * 32 + gidx;
                if (tok < rend && (tok < new_lo || tok > new_hi)) {
                    const int pid = pg_s[lpi - lp0];
                    if (pid >= 0 && pid < a.num_pages) {
                        const size_t off = ((pid * head_rows + static_cast<size_t>(kvh) * a.page_size + row) << 7) + c8 * 8;  // D == 128
                        mk_cp16(dst, static_cast<const bf16 *>(l.k_pages) + off);
                        mk_cp16(dst + 256, static_cast<const bf16 *>(l.v_pages) + off);
                    }
                }
                dst += 32 * MK_KV_STRIDE;
                row += 32;
                while (row >= a.page_size) row -= a.page_size, lpi += 1;
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        prof.stamp(50003);
        if (DEPWAIT && rb == begin) {
            TL_TRACE_STAMP(21);
            asm volatile("griddepcontrol.wait;" ::: "memory");  // the qkv row of this step exists now
            TL_TRACE_STAMP(22);
            if (warp < ntask) load_q(warp);
        }
        // ---- C: q path (first round only)
        if (rb == begin) {
            for (int tk = warp; tk < ntask; tk += NP == 1 ? ntask : MK_WARPS) {  // NP == 1: one task per warp at most
                if (NP > 1 && tk != warp) load_w(tk), load_q(tk);
                const int j = NP == 1 ? 0 : tk / (G + 2), w = NP == 1 ? tk : tk % (G + 2);
                const bool is_q = w < G, is_k = w == G;
                if (is_q || is_k) {
                    float ss = re[0] * re[0] + im[0] * im[0] + re[1] * re[1] + im[1] * im[1];
                    ss = warp_sum(ss);
                    const float inv = rsqrtf(ss / static_cast<float>(D) + a.eps);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int i = lane + 32 * h;
                        const float nre = mk_round(re[h] * inv * wre[h]);
                        const float nim = mk_round(im[h] * inv * wim[h]);
                        const float angle = static_cast<float>(static_cast<double>(position) * freq[h]);
                        float sn, cs;
                        sincosf(angle, &sn, &cs);
                        const bf16 ore = __float2bfloat16_rn(nre * cs - nim * sn), oim = __float2bfloat16_rn(nim * cs + nre * sn);
                        bf16 *dst = is_q ? q_s + (j * G + w) * 128 : k_cur + j * 128;
                        dst[i] = ore, dst[i + 64] = oim;
                    }
                } else {
                    bf16 *dst = v_cur + j * 128;
#pragma unroll
                    for (int h = 0; h < 2; ++h) dst[lane + 32 * h] = __float2bfloat16_rn(re[h]), dst[lane + 32 * h + 64] = __float2bfloat16_rn(im[h]);
                }
            }
        }
        prof.stamp(50004);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();  // q_s / k_cur / v_cur and every lane's K/V pieces are visible
        // the new tokens: their K/V rows join the staged rows, and the split that owns each appends it
        // to the cache (paged_cache_update semantics).  Rows clamped to the same slot: the last one writes.
        if (static_cast<int>(threadIdx.x) < R * 2 * (D / 8)) {
            const int j = threadIdx.x / (2 * (D / 8)), tj = threadIdx.x % (2 * (D / 8));
            const int ctx_j = NP == 1 ? ctx_hi : min(a.context_lens[b * R + j], cap);  // no reload on the decode step's path
            const int cur = ctx_j - 1;
            const bool last = NP == 1 || j + 1 == R || min(a.context_lens[b * R + j + 1], cap) != ctx_j;
            if (ctx_j > 0 && last && cur >= rb && cur < rend) {
                const bool kk = tj < D / 8;
                const int ch = kk ? tj : tj - D / 8;
                const uint4 row = *reinterpret_cast<const uint4 *>((kk ? k_cur : v_cur) + j * 128 + ch * 8);
                *reinterpret_cast<uint4 *>(kv_s + (cur - rb) * MK_KV_STRIDE + (kk ? 0 : 256) + ch * 16) = row;
                const int lp = cur / a.page_size;
                const int pid = pg_s[lp - lp0];
                if (pid >= 0 && pid < a.num_pages) {
                    bf16 *dst = static_cast<bf16 *>(kk ? l.k_pages : l.v_pages) + ((static_cast<size_t>(pid) * a.Hkv + kvh) * a.page_size + (cur - lp * a.page_size)) * D + ch * 8;
                    *reinterpret_cast<uint4 *>(dst) = row;
                }
            }
        }
        __syncthreads();
        prof.stamp(50005);
        if (DEPWAIT) TL_TRACE_STAMP(23);
        // ---- S: scores of 8 tokens x the (head, row) pairs per MMA tile, with the tile's softmax statistics
        for (int tile = warp; tile * 8 < cnt; tile += MK_WARPS) {
            float d[MB][4], d2[MB][4];  // two independent MMA chains per block
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int k = 0; k < 4; ++k) d[mb][k] = 0.f, d2[mb][k] = 0.f;
            const unsigned char *krow = kv_s + (tile * 8 + g) * MK_KV_STRIDE + t * 4;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const uint32_t b0 = *reinterpret_cast<const uint32_t *>(krow + ks * 32);
                const uint32_t b1 = *reinterpret_cast<const uint32_t *>(krow + ks * 32 + 16);
#pragma unroll
                for (int mb = 0; mb < MB; ++mb) {
                    const int p = mb * 16 + g;
                    const bf16 *qrow = q_s + (p < GR ? p : 0) * 128 + 2 * t;
                    uint32_t a0 = *reinterpret_cast<const uint32_t *>(qrow + ks * 16);
                    uint32_t a2 = *reinterpret_cast<const uint32_t *>(qrow + ks * 16 + 8);
                    if (p >= GR) a0 = a2 = 0u;
                    uint32_t a1 = 0u, a3 = 0u;
                    if (HI8) {
                        const int p8 = p + 8;
                        const bf16 *qrow8 = q_s + (p8 < GR ? p8 : 0) * 128 + 2 * t;
                        a1 = *reinterpret_cast<const uint32_t *>(qrow8 + ks * 16);
                        a3 = *reinterpret_cast<const uint32_t *>(qrow8 + ks * 16 + 8);
                        if (p8 >= GR) a1 = a3 = 0u;
                    }
                    if (ks & 1)
                        W4Num<bf16>::mma(d2[mb], a0, a1, a2, a3, b0, b1);
                    else
                        W4Num<bf16>::mma(d[mb], a0, a1, a2, a3, b0, b1);
                }
            }
            // lane (g, t) holds pairs g (and g + 8) of each block, tokens 2t and 2t+1 of the tile
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int hf = 0; hf < (HI8 ? 2 : 1); ++hf) {
                    const int p = mb * 16 + hf * 8 + g;
                    float sc[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int slot = tile * 8 + 2 * t + e;
                        bool ok = rb + slot < s_end[mb][hf];
                        if (ok) {
                            const int pid = pg_s[(rb + slot) / a.page_size - lp0];
                            ok = pid >= 0 && pid < a.num_pages;
                        }
                        sc[e] = ok ? (d[mb][2 * hf + e] + d2[mb][2 * hf + e]) * scale2 : -CUDART_INF_F;
                    }
                    float mx = fmaxf(sc[0], sc[1]);
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    const float ref = mx == -CUDART_INF_F ? 0.f : mx;  // a fully masked tile: probabilities 0, not NaN
                    const float p0 = exp2f(sc[0] - ref), p1 = exp2f(sc[1] - ref);
                    float ls = p0 + p1;
                    ls += __shfl_xor_sync(0xffffffffu, ls, 1);
                    ls += __shfl_xor_sync(0xffffffffu, ls, 2);
                    if (p < GR) {
                        *reinterpret_cast<float2 *>(s_s + p * MK_ATT_TOK + tile * 8 + 2 * t) = make_float2(p0, p1);
                        if (t == 0) st_s[p * 32 + tile] = mx == -CUDART_INF_F ? MK_NEG : mx, st_s[HR * 32 + p * 32 + tile] = ls;
                    }
                }
        }
        __syncthreads();
        prof.stamp(50008);
        // ---- V: thread = (token of the tile, 8 dims, pair); one staged row per tile, then a shuffle
        // reduction over the 8 tokens of a tile position; the sub == 0 lane keeps the running state
        const int ntile = (cnt + 7) >> 3;
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            const int p = oh + 4 * i;
            if (NP > 1 && p >= GR) break;  // warp-uniform
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            float m_r = MK_NEG, l_r = 0.f;
            if (p < GR) {
                for (int tile = 0; tile < ntile; ++tile) m_r = fmaxf(m_r, st_s[p * 32 + tile]);
                for (int tile = 0; tile < ntile; ++tile) {
                    const float f = exp2f(st_s[p * 32 + tile] - m_r);
                    l_r += st_s[HR * 32 + p * 32 + tile] * f;
                    const int slot = tile * 8 + sub;
                    const float pr = s_s[p * MK_ATT_TOK + slot] * f;
                    if (pr != 0.f) {  // masked / padded slots hold no valid V row
                        const uint4 vr = *reinterpret_cast<const uint4 *>(kv_s + slot * MK_KV_STRIDE + 256 + d8 * 16);
                        const float2 f0 = unpack2<bf16>(vr.x), f1 = unpack2<bf16>(vr.y), f2 = unpack2<bf16>(vr.z), f3 = unpack2<bf16>(vr.w);
                        acc[0] += pr * f0.x, acc[1] += pr * f0.y, acc[2] += pr * f1.x, acc[3] += pr * f1.y;
                        acc[4] += pr * f2.x, acc[5] += pr * f2.y, acc[6] += pr * f3.x, acc[7] += pr * f3.y;
                    }
                }
            }
#pragma unroll
            for (int off = 1; off < 8; off <<= 1)
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], off);
            // a row whose keys ended before this round: the R = 1 kernel runs no such round for it
            if constexpr (SMEM_STATE) {
                if (p < GR && sub == 0 && (rb < v_end[i] || rb == begin)) {
                    float *S = state_s + (p * 16 + d8) * 10;
                    const float nm = fmaxf(S[0], m_r);
                    const float fr = exp2f(S[0] - nm), fn = exp2f(m_r - nm);
#pragma unroll
                    for (int k = 0; k < 8; ++k) S[2 + k] = S[2 + k] * fr + acc[k] * fn;
                    S[1] = S[1] * fr + l_r * fn;
                    S[0] = nm;
                }
            } else if (p < GR && sub == 0 && (NP == 1 || rb < v_end[i] || rb == begin)) {
                const float nm = fmaxf(m_run[i], m_r);
                const float fr = exp2f(m_run[i] - nm), fn = exp2f(m_r - nm);
#pragma unroll
                for (int k = 0; k < 8; ++k) o_run[i][k] = o_run[i][k] * fr + acc[k] * fn;
                l_run[i] = l_run[i] * fr + l_r * fn;
                m_run[i] = nm;
            }
        }
        prof.stamp(50006);
        __syncthreads();  // the round's page ids, rows and scores are dead: the next round may overwrite them
    }
    prof.stamp(50007);
#pragma unroll
    for (int i = 0; i < NP; ++i) {
        const int p = oh + 4 * i;
        if (p < GR && (threadIdx.x & 7) == 0) {  // this lane owns out[pair p][8 dims]
            if constexpr (SMEM_STATE) {
                const float *S = state_s + (p * 16 + d8) * 10;
                m_run[0] = S[0], l_run[0] = S[1];
#pragma unroll
                for (int k = 0; k < 8; ++k) o_run[0][k] = S[2 + k];
            }
            const int ii = SMEM_STATE ? 0 : i;
            const int head = kvh * G + p % G, qrow = b * R + p / G, d0 = ((threadIdx.x >> 3) & 15) * 8;
            if (a.nsplit == 1) {
                const float inv = l_run[ii] == 0.f ? 0.f : 1.0f / l_run[ii];
                uint4 o;
                o.x = pack2<bf16>(o_run[ii][0] * inv, o_run[ii][1] * inv), o.y = pack2<bf16>(o_run[ii][2] * inv, o_run[ii][3] * inv);
                o.z = pack2<bf16>(o_run[ii][4] * inv, o_run[ii][5] * inv), o.w = pack2<bf16>(o_run[ii][6] * inv, o_run[ii][7] * inv);
                *reinterpret_cast<uint4 *>(static_cast<bf16 *>(a.y) + (static_cast<size_t>(qrow) * a.Hq + head) * D + d0) = o;
            } else {
                const size_t row = (static_cast<size_t>(qrow) * a.Hq + head) * a.nsplit + split;
#pragma unroll
                for (int k = 0; k < 8; ++k) a.attn_ws[row * (D + 2) + d0 + k] = o_run[ii][k];
                if (d0 == 0) a.attn_ws[row * (D + 2) + D] = m_run[ii], a.attn_ws[row * (D + 2) + D + 1] = l_run[ii];
            }
        }
    }
}

__device__ void mk_attention_merge(const MkArgs &a) {
    const int D = a.D;
    const int heads = a.B * a.R * a.Hq;
    const int warp_global = blockIdx.x * MK_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    for (int h = warp_global; h < heads; h += gridDim.x * MK_WARPS) {
        const float *base = a.attn_ws + static_cast<size_t>(h) * a.nsplit * (D + 2);
        float gm = MK_NEG;
        for (int s = 0; s < a.nsplit; ++s) gm = fmaxf(gm, ld_cg(base + s * (D + 2) + D));
        float gl = 0.f, o[4] = {0.f, 0.f, 0.f, 0.f};
        for (int s = 0; s < a.nsplit; ++s) {
            const float f = exp2f(ld_cg(base + s * (D + 2) + D) - gm);
            gl += ld_cg(base + s * (D + 2) + D + 1) * f;
#pragma unroll
            for (int i = 0; i < 4; ++i) o[i] += ld_cg(base + s * (D + 2) + lane + 32 * i) * f;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) static_cast<bf16 *>(a.y)[static_cast<size_t>(h) * D + lane + 32 * i] = __float2bfloat16_rn(gl == 0.f ? 0.f : o[i] / gl);
    }
}

// ---- the attention phase as a kernel of its own (CUDA-graph decode path) ----
template <int NP>
__global__ void __launch_bounds__(MK_THREADS, 1) decode_attention_fused_kernel(const MkArgs a, const MkLayer l) {
    extern __shared__ __align__(128) unsigned char att_smem_raw[];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // the o_proj stream may prefetch its weights now
    TL_TRACE_STAMP(20);
    Prof prof;
    mk_attention<true, NP>(a, l, att_smem_raw, prof);
    TL_TRACE_STAMP(29);
}
#if TL_TRACE
void trace_bind_attention(unsigned long long *buf, unsigned int *n, unsigned int cap) { trace_bind(buf, n, cap); }
#endif
__global__ void __launch_bounds__(MK_THREADS, 1) decode_attention_merge_kernel(const MkArgs a) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    mk_attention_merge(a);
}

// splits depend on the number of requests, never on their rows: a row's split boundaries are those of
// the single-row decode step at the same max_context
static int attention_max_split(int batch, int num_kv_heads) {
    const int s = sm_count() / (batch * num_kv_heads);
    return s < 1 ? 1 : s;
}
size_t decode_attention_fused_workspace(int batch, int rows_per_request, int num_heads, int num_kv_heads) {
    return static_cast<size_t>(batch) * rows_per_request * num_heads * attention_max_split(batch, num_kv_heads) * (128 + 2);
}

template <int NP>
static int launch_mk(const MkArgs &a, const MkLayer &l, int grid, cudaStream_t st) {
    // the single-row launch keeps its shared-memory footprint (mk_att_bytes(4, 1))
    const size_t max_bytes = NP == 1 ? mk_att_bytes(4, 1) : mk_att_bytes(4 * NP, MK_MAX_ROWS) + (NP > 4 ? mk_state_bytes(4 * NP) : 0);
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(decode_attention_fused_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(max_bytes + 64)) != cudaSuccess)
            return fail(TL_ECUDA, "decode_attention_fused: cannot raise shared memory limit");
        configured = true;
    }
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(MK_THREADS);
    cfg.dynamicSmemBytes = mk_att_bytes(a.HR, a.R) + (NP > 4 ? mk_state_bytes(a.HR) : 0) + 64;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 1 : 0;  // without the attribute griddepcontrol.wait returns at once
    cudaError_t e = cudaLaunchKernelEx(&cfg, decode_attention_fused_kernel<NP>, a, l);
    if (e != cudaSuccess) return fail(TL_ECUDA, "decode_attention_fused: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("decode_attention_fused");
    return TL_OK;
}

int launch_decode_attention_fused(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                  const int32_t *block_table, const int32_t *context_lens, const double *rope_inv_freq,
                                  void *key_pages, void *value_pages, void *out, float *workspace, int batch, int rows_per_request,
                                  int num_heads, int num_kv_heads, int head_dim, float eps, float scale, int num_pages,
                                  int page_size, int max_pages, int max_context, int dtype, cudaStream_t st) {
    if (batch == 0) return TL_OK;
    if (dtype != TL_BF16 || head_dim != 128 || num_kv_heads < 1 || num_heads % num_kv_heads != 0 || num_heads / num_kv_heads > 4)
        return fail(TL_EINVAL, "decode_attention_fused: needs bfloat16, head_dim 128 and at most 4 query heads per KV head");
    if (rows_per_request < 1 || rows_per_request > MK_MAX_ROWS)
        return fail(TL_EINVAL, "decode_attention_fused: rows_per_request must be in [1, 8]");
    MkArgs a{};
    MkLayer l{};
    const int GR = num_heads / num_kv_heads * rows_per_request;
    a.B = batch, a.Hq = num_heads, a.Hkv = num_kv_heads, a.D = head_dim;
    a.R = rows_per_request, a.HR = GR < 4 ? 4 : GR;
    a.eps = eps, a.attn_scale = scale;
    a.page_size = page_size, a.max_pages = max_pages, a.num_pages = num_pages;
    a.offsets = const_cast<int32_t *>(offsets), a.context_lens = const_cast<int32_t *>(context_lens);
    a.rope_inv_freq = rope_inv_freq;
    a.qkv = const_cast<void *>(qkv), a.y = out, a.attn_ws = workspace;
    const int max_split = attention_max_split(batch, num_kv_heads);
    int tps = (max_context < 1 ? 1 : max_context + max_split - 1) / max_split;
    tps = tps < 2 * MK_ATT_TOK ? 2 * MK_ATT_TOK : tps;  // a split (extra merge launch) only pays beyond two rounds
    tps = (tps + 63) / 64 * 64;
    a.tokens_per_split = tps;
    a.nsplit = (max_context + tps - 1) / tps;
    a.nsplit = a.nsplit < 1 ? 1 : (a.nsplit > max_split ? max_split : a.nsplit);
    l.q_norm = q_norm_weight, l.k_norm = k_norm_weight, l.table = block_table;
    l.k_pages = key_pages, l.v_pages = value_pages;
    const int grid = batch * num_kv_heads * a.nsplit;
    const int np = rows_per_request == 1 ? 1 : std::max(2, (GR + 3) / 4);  // NP == 1: the single-row step only
    const int rc = np <= 1 ? launch_mk<1>(a, l, grid, st)
                 : np <= 2 ? launch_mk<2>(a, l, grid, st)
                 : np <= 4 ? launch_mk<4>(a, l, grid, st)
                           : launch_mk<8>(a, l, grid, st);
    if (rc != TL_OK) return rc;
    if (a.nsplit > 1) {
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cudaLaunchConfig_t cfg{};
        const int heads = batch * rows_per_request * num_heads;
        cfg.gridDim = dim3((heads + MK_WARPS - 1) / MK_WARPS);
        cfg.blockDim = dim3(MK_THREADS);
        cfg.dynamicSmemBytes = 0;
        cfg.stream = st;
        cfg.attrs = attr;
        cfg.numAttrs = use_pdl() ? 1 : 0;
        cudaError_t e = cudaLaunchKernelEx(&cfg, decode_attention_merge_kernel, a);
        if (e != cudaSuccess) return fail(TL_ECUDA, "decode_attention_merge: launch failed: %s", cudaGetErrorString(e));
        TL_LAUNCH_CHECK("decode_attention_merge");
    }
    return TL_OK;
}


}  // namespace tl
