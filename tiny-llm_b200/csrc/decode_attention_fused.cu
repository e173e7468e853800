// Fused decode attention for the Week-3 Qwen3 model (bf16, paged KV, L == 1): one launch does
// q/k RMSNorm -> RoPE -> K/V append -> paged GQA attention for every (request, KV head), i.e. the
// operator sequence rms_norm x2 -> rope x2 -> paged_cache_update x2 -> paged_attention of
// src/tiny_llm_ref/qwen3_week3.py:62-105 with the kernel arithmetic of
// src/extensions_ref/src/paged_attention.metal:108-248, every rounding point kept.
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

typedef __nv_bfloat16 bf16;

// Launch-constant arguments (plain pointers and sizes; filled by launch_decode_attention_fused).
struct MkLayer {
    const void *q_norm, *k_norm;  // bf16 [D]
    void *k_pages, *v_pages;      // bf16 [P, Hkv, page, D]
    const int32_t *table;         // int32 [B, max_pages], -1 padded
};
struct MkArgs {
    int B, Hq, Hkv, D;
    float eps, attn_scale;
    int page_size, max_pages, num_pages;
    const int32_t *offsets, *context_lens;  // [B]: RoPE positions, post-append lengths
    const void *qkv;                        // bf16 [B, (Hq + 2 Hkv) D]
    void *y;                                // bf16 [B, Hq D]
    float *attn_ws;                         // [B*Hq*nsplit*(D+2)] when nsplit > 1
    int nsplit, tokens_per_split;
    const double *rope_inv_freq;            // [D/2]
};

__device__ __forceinline__ float mk_bf(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float mk_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

struct Prof {
    __device__ __forceinline__ void stamp(int) {}
};

// --------------------------------------------------------------- attention --
// One CTA per (request, kv head, split), L == 1.  The phase is pure latency (8 CTAs x 64 KB of
// K/V at context 128), so it is organised around dependent round trips and wide parallelism, not
// bandwidth.  Per round of up to MK_ATT_TOK tokens:
//   A  page ids of the round -> shared; warps 0..G+1 already hold their q/k/v head rows, norm
//      weights and rope frequencies in registers (loaded before anything else)
//   B  cp.async ALL K/V rows of the round into shared memory (row stride 528 B: bank spread)
//   C  while those are in flight: q/k RMSNorm + RoPE (rounded like rms_norm -> rope), V copy
//   S  scores = Q K^T on the tensor cores: mma.sync m16n8k16, A = the G query heads (rows >= G
//      zero), B = K rows straight from shared memory; 8 tokens per MMA tile, 16 warps
//   M  one warp per head: max / exp2 / sum over the round's tokens (fp32)
//   V  out = P V on CUDA cores with fp32 probabilities: thread = (head, 8 dims, token subset)
//   then the running (max, sum, out) of thread (head, dim) absorbs the round.
constexpr int MK_ATT_TOK = 256;     // K/V rows staged per round
constexpr int MK_KV_STRIDE = 528;   // bytes per staged token: K row | V row | 16 B pad
constexpr size_t MK_ATT_BYTES = 4 * 128 * 2 + 2 * 128 * 2 + 4 * MK_ATT_TOK * 4 + 256 * 4 + (MK_ATT_TOK + 4) * 4 +
                                static_cast<size_t>(MK_ATT_TOK) * MK_KV_STRIDE;

__device__ __forceinline__ void mk_cp16(void *dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))), "l"(src) : "memory");
}

// DEPWAIT (stand-alone kernel under programmatic dependent launch): everything that does not read
// this step's qkv row - page ids, the K/V rows of older tokens - is requested BEFORE
// griddepcontrol.wait, i.e. while the qkv projection is still draining.
template <bool DEPWAIT>
__device__ void mk_attention(const MkArgs &a, const MkLayer &l, unsigned char *dyn, Prof &prof) {
    const int D = a.D, G = a.Hq / a.Hkv;
    const int items = a.B * a.Hkv * a.nsplit;
    if (static_cast<int>(blockIdx.x) >= items) return;
    const int split = blockIdx.x % a.nsplit;
    const int kvh = (blockIdx.x / a.nsplit) % a.Hkv;
    const int b = blockIdx.x / (a.nsplit * a.Hkv);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qkv_w = (a.Hq + 2 * a.Hkv) * D;

    bf16 *q_s = reinterpret_cast<bf16 *>(dyn);                      // [4][128] rope output (unscaled)
    bf16 *k_cur = q_s + 4 * 128;                                    // [128] newest token
    bf16 *v_cur = k_cur + 128;                                      // [128]
    float *s_s = reinterpret_cast<float *>(v_cur + 128);            // [4][MK_ATT_TOK] scores, then probabilities
    float *st_s = s_s + 4 * MK_ATT_TOK;                             // per (head, tile): max [4][32], then sum [4][32]
    int *pg_s = reinterpret_cast<int *>(st_s + 256);                // page ids of the round
    unsigned char *kv_s = reinterpret_cast<unsigned char *>(pg_s + MK_ATT_TOK + 4);  // [MK_ATT_TOK][528]

    // ---- head rows for the q path (registers; used after the K/V copies are in flight)
    const bool qpath = warp < G + 2;
    const bool is_q = warp < G, is_k = warp == G;
    float re[2] = {0.f, 0.f}, im[2] = {0.f, 0.f}, wre[2] = {0.f, 0.f}, wim[2] = {0.f, 0.f};
    double freq[2] = {0.0, 0.0};
    int position = 0;
    auto load_q = [&]() {
        if (qpath) {
            const int head_off = is_q ? (kvh * G + warp) * D : (is_k ? (a.Hq + kvh) * D : (a.Hq + a.Hkv + kvh) * D);
            const bf16 *src = static_cast<const bf16 *>(a.qkv) + static_cast<size_t>(b) * qkv_w + head_off;
#pragma unroll
            for (int h = 0; h < 2; ++h) {  // lane owns pairs (i, i+64) for i = lane, lane+32   (D == 128)
                re[h] = mk_bf(ld_cg(src + lane + 32 * h));
                im[h] = mk_bf(ld_cg(src + lane + 32 * h + 64));
            }
        }
    };
    if (qpath) {
        const bf16 *w = static_cast<const bf16 *>(is_q ? l.q_norm : l.k_norm);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (is_q || is_k) {
                wre[h] = mk_bf(w[lane + 32 * h]);
                wim[h] = mk_bf(w[lane + 32 * h + 64]);
                freq[h] = a.rope_inv_freq[lane + 32 * h];
            }
        }
        position = a.offsets[b];
    }
    if (!DEPWAIT) load_q();
    // page ids of the first round do not need the context length: request them together with it
    const int begin = split * a.tokens_per_split;
    {
        const int lp_first = begin / a.page_size + static_cast<int>(threadIdx.x);
        if (static_cast<int>(threadIdx.x) <= MK_ATT_TOK && lp_first < a.max_pages)
            pg_s[threadIdx.x] = l.table[static_cast<size_t>(b) * a.max_pages + lp_first];
    }
    const int ctx = min(a.context_lens[b], a.max_pages * a.page_size);
    const int end = min(ctx, begin + a.tokens_per_split);
    const int cur_tok = ctx - 1;
    const int gidx = warp * 2 + (lane >> 4), c8 = lane & 15;   // copy mapping: lane group of 16 per token row
    const int g = lane >> 2, t = lane & 3;                      // MMA fragment coordinates
    const int oh = threadIdx.x >> 7;                            // head whose output this thread helps to form
    const float scale2 = a.attn_scale * MK_LOG2E;
    float m_run = MK_NEG, l_run = 0.f, o_run[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};  // kept by the (threadIdx & 7) == 0 lanes
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
                if (tok < rend && tok != cur_tok) {
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
            load_q();
        }
        // ---- C: q path (first round only)
        if (rb == begin && qpath) {
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
                    bf16 *dst = is_q ? q_s + warp * 128 : k_cur;
                    dst[i] = ore, dst[i + 64] = oim;
                }
            } else {
#pragma unroll
                for (int h = 0; h < 2; ++h) v_cur[lane + 32 * h] = __float2bfloat16_rn(re[h]), v_cur[lane + 32 * h + 64] = __float2bfloat16_rn(im[h]);
            }
        }
        prof.stamp(50004);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();  // q_s / k_cur / v_cur and every lane's K/V pieces are visible
        // the newest token: its K/V rows join the staged rows, and the split that owns it appends it
        // to the cache (paged_cache_update semantics)
        if (ctx > 0 && cur_tok >= rb && cur_tok < rend && threadIdx.x < 2 * (D / 8)) {
            const bool kk = threadIdx.x < D / 8;
            const int ch = kk ? threadIdx.x : threadIdx.x - D / 8;
            const uint4 row = *reinterpret_cast<const uint4 *>((kk ? k_cur : v_cur) + ch * 8);
            *reinterpret_cast<uint4 *>(kv_s + (cur_tok - rb) * MK_KV_STRIDE + (kk ? 0 : 256) + ch * 16) = row;
            const int lp = cur_tok / a.page_size;
            const int pid = pg_s[lp - lp0];
            if (pid >= 0 && pid < a.num_pages) {
                bf16 *dst = static_cast<bf16 *>(kk ? l.k_pages : l.v_pages) + ((static_cast<size_t>(pid) * a.Hkv + kvh) * a.page_size + (cur_tok - lp * a.page_size)) * D + ch * 8;
                *reinterpret_cast<uint4 *>(dst) = row;
            }
        }
        __syncthreads();
        prof.stamp(50005);
        if (DEPWAIT) TL_TRACE_STAMP(23);
        // ---- S: scores of 8 tokens x G heads per MMA tile, with the tile's softmax statistics
        for (int tile = warp; tile * 8 < cnt; tile += MK_WARPS) {
            float d[4] = {0.f, 0.f, 0.f, 0.f}, d2[4] = {0.f, 0.f, 0.f, 0.f};  // two independent MMA chains
            const unsigned char *krow = kv_s + (tile * 8 + g) * MK_KV_STRIDE + t * 4;
            const bf16 *qrow = q_s + (g < G ? g : 0) * 128 + 2 * t;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                uint32_t a0 = *reinterpret_cast<const uint32_t *>(qrow + ks * 16);
                uint32_t a2 = *reinterpret_cast<const uint32_t *>(qrow + ks * 16 + 8);
                if (g >= G) a0 = a2 = 0u;
                const uint32_t b0 = *reinterpret_cast<const uint32_t *>(krow + ks * 32);
                const uint32_t b1 = *reinterpret_cast<const uint32_t *>(krow + ks * 32 + 16);
                if (ks & 1)
                    W4Num<bf16>::mma(d2, a0, 0u, a2, 0u, b0, b1);
                else
                    W4Num<bf16>::mma(d, a0, 0u, a2, 0u, b0, b1);
            }
            // lane (g, t) holds head g, tokens 2t and 2t+1 of the tile
            float sc[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int slot = tile * 8 + 2 * t + e;
                bool ok = slot < cnt;
                if (ok) {
                    const int pid = pg_s[(rb + slot) / a.page_size - lp0];
                    ok = pid >= 0 && pid < a.num_pages;
                }
                sc[e] = ok ? (d[e] + d2[e]) * scale2 : -CUDART_INF_F;
            }
            float mx = fmaxf(sc[0], sc[1]);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float ref = mx == -CUDART_INF_F ? 0.f : mx;  // a fully masked tile: probabilities 0, not NaN
            const float p0 = exp2f(sc[0] - ref), p1 = exp2f(sc[1] - ref);
            float ls = p0 + p1;
            ls += __shfl_xor_sync(0xffffffffu, ls, 1);
            ls += __shfl_xor_sync(0xffffffffu, ls, 2);
            if (g < G) {
                *reinterpret_cast<float2 *>(s_s + g * MK_ATT_TOK + tile * 8 + 2 * t) = make_float2(p0, p1);
                if (t == 0) st_s[g * 32 + tile] = mx == -CUDART_INF_F ? MK_NEG : mx, st_s[128 + g * 32 + tile] = ls;
            }
        }
        __syncthreads();
        prof.stamp(50008);
        // ---- V: thread = (token of the tile, 8 dims, head); one staged row per tile, then a shuffle
        // reduction over the 8 tokens of a tile position; the sub == 0 lane keeps the running state
        {
            const int sub = threadIdx.x & 7, d8 = (threadIdx.x >> 3) & 15;
            const int ntile = (cnt + 7) >> 3;
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            float m_r = MK_NEG, l_r = 0.f;
            if (oh < G) {
                for (int tile = 0; tile < ntile; ++tile) m_r = fmaxf(m_r, st_s[oh * 32 + tile]);
                for (int tile = 0; tile < ntile; ++tile) {
                    const float f = exp2f(st_s[oh * 32 + tile] - m_r);
                    l_r += st_s[128 + oh * 32 + tile] * f;
                    const int slot = tile * 8 + sub;
                    const float pr = s_s[oh * MK_ATT_TOK + slot] * f;
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
                for (int i = 0; i < 8; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
            if (oh < G && sub == 0) {
                const float nm = fmaxf(m_run, m_r);
                const float fr = exp2f(m_run - nm), fn = exp2f(m_r - nm);
#pragma unroll
                for (int i = 0; i < 8; ++i) o_run[i] = o_run[i] * fr + acc[i] * fn;
                l_run = l_run * fr + l_r * fn;
                m_run = nm;
            }
        }
        prof.stamp(50006);
        __syncthreads();  // the round's page ids, rows and scores are dead: the next round may overwrite them
    }
    prof.stamp(50007);
    if (oh < G && (threadIdx.x & 7) == 0) {  // this lane owns out[head oh][8 dims]
        const int head = kvh * G + oh, d0 = ((threadIdx.x >> 3) & 15) * 8;
        if (a.nsplit == 1) {
            const float inv = l_run == 0.f ? 0.f : 1.0f / l_run;
            uint4 o;
            o.x = pack2<bf16>(o_run[0] * inv, o_run[1] * inv), o.y = pack2<bf16>(o_run[2] * inv, o_run[3] * inv);
            o.z = pack2<bf16>(o_run[4] * inv, o_run[5] * inv), o.w = pack2<bf16>(o_run[6] * inv, o_run[7] * inv);
            *reinterpret_cast<uint4 *>(static_cast<bf16 *>(a.y) + (static_cast<size_t>(b) * a.Hq + head) * D + d0) = o;
        } else {
            const size_t row = (static_cast<size_t>(b) * a.Hq + head) * a.nsplit + split;
#pragma unroll
            for (int i = 0; i < 8; ++i) a.attn_ws[row * (D + 2) + d0 + i] = o_run[i];
            if (d0 == 0) a.attn_ws[row * (D + 2) + D] = m_run, a.attn_ws[row * (D + 2) + D + 1] = l_run;
        }
    }
}

__device__ void mk_attention_merge(const MkArgs &a) {
    const int D = a.D;
    const int heads = a.B * a.Hq;
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
__global__ void __launch_bounds__(MK_THREADS, 1) decode_attention_fused_kernel(const MkArgs a, const MkLayer l) {
    extern __shared__ __align__(128) unsigned char att_smem_raw[];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // the o_proj stream may prefetch its weights now
    TL_TRACE_STAMP(20);
    Prof prof;
    mk_attention<true>(a, l, att_smem_raw, prof);
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

static int attention_max_split(int batch, int num_kv_heads) {
    const int s = sm_count() / (batch * num_kv_heads);
    return s < 1 ? 1 : s;
}
size_t decode_attention_fused_workspace(int batch, int num_heads, int num_kv_heads) {
    return static_cast<size_t>(batch) * num_heads * attention_max_split(batch, num_kv_heads) * (128 + 2);
}

int launch_decode_attention_fused(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                  const int32_t *block_table, const int32_t *context_lens, const double *rope_inv_freq,
                                  void *key_pages, void *value_pages, void *out, float *workspace, int batch, int num_heads,
                                  int num_kv_heads, int head_dim, float eps, float scale, int num_pages, int page_size,
                                  int max_pages, int max_context, int dtype, cudaStream_t st) {
    if (batch == 0) return TL_OK;
    if (dtype != TL_BF16 || head_dim != 128 || num_kv_heads < 1 || num_heads % num_kv_heads != 0 || num_heads / num_kv_heads > 4)
        return fail(TL_EINVAL, "decode_attention_fused: needs bfloat16, head_dim 128 and at most 4 query heads per KV head");
    MkArgs a{};
    MkLayer l{};
    a.B = batch, a.Hq = num_heads, a.Hkv = num_kv_heads, a.D = head_dim;
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
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(decode_attention_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(MK_ATT_BYTES + 64)) != cudaSuccess)
            return fail(TL_ECUDA, "decode_attention_fused: cannot raise shared memory limit");
        configured = true;
    }
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(batch * num_kv_heads * a.nsplit);
    cfg.blockDim = dim3(MK_THREADS);
    cfg.dynamicSmemBytes = MK_ATT_BYTES + 64;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 1 : 0;  // without the attribute griddepcontrol.wait returns at once
    cudaError_t e = cudaLaunchKernelEx(&cfg, decode_attention_fused_kernel, a, l);
    if (e != cudaSuccess) return fail(TL_ECUDA, "decode_attention_fused: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("decode_attention_fused");
    if (a.nsplit > 1) {
        const int heads = batch * num_heads;
        cfg.gridDim = dim3((heads + MK_WARPS - 1) / MK_WARPS);
        cfg.dynamicSmemBytes = 0;
        e = cudaLaunchKernelEx(&cfg, decode_attention_merge_kernel, a);
        if (e != cudaSuccess) return fail(TL_ECUDA, "decode_attention_merge: launch failed: %s", cudaGetErrorString(e));
        TL_LAUNCH_CHECK("decode_attention_merge");
    }
    return TL_OK;
}


}  // namespace tl
