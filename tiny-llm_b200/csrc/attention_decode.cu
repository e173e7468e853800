// Decode-side attention kernels (HBM-bound K/V streaming, fp32 online softmax).
//
//  * decode_attention_kernel       - dense K/V, reference week2_decode_attention
//    (src/extensions_ref/src/week2_kernels.metal:119-235).
//  * paged_rowwise_kernel          - generic paged attention, one CTA per query
//    row; any dtype/head-dim/page-size (reference paged_attention_decode and the
//    f32 scalar path, paged_attention.metal:108-248, :508-674).
//  * paged_gqa_kernel + merge      - bf16, D=128 fast path: one CTA per
//    (request, KV head, row group, KV split).  All query heads that share a KV
//    head are processed together so K/V bytes are read ONCE per KV head (the
//    Metal kernel re-reads them per query head), the context is split across
//    CTAs (flash-decoding) so a single request still fills every SM, and every
//    K/V access is a 128-bit load of a fully used 32-byte sector.
//
// Causality is bottom-right aligned everywhere: query row l of an L-row chunk
// sees keys < clamp(ctx - L + l + 1, 0, ctx)   (paged_attention.metal:158-160),
// then at most the max_pages * page_size keys of the block table.  The shift uses
// the unclamped context, so every kernel keeps the same rows aligned when a
// context is longer than its table.
#include <math_constants.h>

#include "common.cuh"
#include "kernels.h"

namespace tl {

constexpr float LOG2E = 1.44269504089f;
constexpr float NEG_BIG = -1e30f;  // finite "minus infinity" of the reference kernels

// ------------------------------------------------------- dense decode (N10) --
template <typename T>
__global__ void __launch_bounds__(128) decode_attention_kernel(const T *__restrict__ q, const T *__restrict__ k,
                                                               const T *__restrict__ v, const float *__restrict__ mask,
                                                               T *__restrict__ out, int q_rows, int L, int S, int D,
                                                               int num_heads, int num_kv_heads, float scale,
                                                               int is_causal, int has_mask) {
    constexpr int WARPS = 4;
    constexpr int MAXV = 8;  // D <= 256
    extern __shared__ float sm[];
    float *p_acc = sm;                // [WARPS][D]
    float *p_max = sm + WARPS * D;    // [WARPS]
    float *p_sum = p_max + WARPS;     // [WARPS]
    const int query_index = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int query_row = query_index / L;
    const int query_pos = query_index - query_row * L;
    const int batch = query_row / num_heads;
    const int head = query_row - batch * num_heads;
    const int kv_row = batch * num_kv_heads + head / (num_heads / num_kv_heads);
    const int vpl = (D + 31) / 32;

    float qv[MAXV], acc[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int d = lane + 32 * i;
        acc[i] = 0.f;
        qv[i] = (i < vpl && d < D) ? to_f(q[static_cast<size_t>(query_index) * D + d]) * scale : 0.f;
    }
    float m = NEG_BIG, l = 0.f;
    for (int pos = warp; pos < S; pos += WARPS) {
        if (is_causal && pos > S - L + query_pos) continue;
        const T *kr = k + (static_cast<size_t>(kv_row) * S + pos) * D;
        const T *vr = v + (static_cast<size_t>(kv_row) * S + pos) * D;
        float part = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int d = lane + 32 * i;
            if (i < vpl && d < D) part += qv[i] * to_f(kr[d]);
        }
        float score = warp_sum(part);
        if (has_mask) score += mask[static_cast<size_t>(query_index) * S + pos];
        const float nm = fmaxf(m, score);
        const float f_old = __expf(m - nm);
        const float f_new = __expf(score - nm);
        l = l * f_old + f_new;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int d = lane + 32 * i;
            if (i < vpl && d < D) acc[i] = acc[i] * f_old + f_new * to_f(vr[d]);
        }
        m = nm;
    }
    if (lane == 0) p_max[warp] = m, p_sum[warp] = l;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int d = lane + 32 * i;
        if (i < vpl && d < D) p_acc[warp * D + d] = acc[i];
    }
    __syncthreads();
    float gm = NEG_BIG;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) gm = fmaxf(gm, p_max[w]);
    float gs = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) gs += p_sum[w] * __expf(p_max[w] - gm);
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        float o = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) o += p_acc[w * D + d] * __expf(p_max[w] - gm);
        out[static_cast<size_t>(query_index) * D + d] = from_f<T>(o / gs);
    }
}

template <typename T>
static int decode_attention_t(const void *q, const void *k, const void *v, const float *mask, void *out, int q_rows,
                              int L, int S, int D, int nh, int nkv, float scale, int causal, int has_mask,
                              cudaStream_t st) {
    const size_t smem = (4 * static_cast<size_t>(D) + 8) * sizeof(float);
    decode_attention_kernel<T><<<q_rows * L, 128, smem, st>>>(static_cast<const T *>(q), static_cast<const T *>(k),
                                                              static_cast<const T *>(v), mask, static_cast<T *>(out),
                                                              q_rows, L, S, D, nh, nkv, scale, causal, has_mask);
    TL_LAUNCH_CHECK("decode_attention");
    return TL_OK;
}

int launch_decode_attention(const void *q, const void *k, const void *v, const float *mask, void *out, int q_rows,
                            int L, int S, int D, int num_heads, int num_kv_heads, float scale, int is_causal,
                            int has_mask, int dtype, cudaStream_t st) {
    if (q_rows * L == 0) return TL_OK;
    switch (dtype) {
        case TL_F32: return decode_attention_t<float>(q, k, v, mask, out, q_rows, L, S, D, num_heads, num_kv_heads, scale, is_causal, has_mask, st);
        case TL_F16: return decode_attention_t<__half>(q, k, v, mask, out, q_rows, L, S, D, num_heads, num_kv_heads, scale, is_causal, has_mask, st);
        case TL_BF16: return decode_attention_t<__nv_bfloat16>(q, k, v, mask, out, q_rows, L, S, D, num_heads, num_kv_heads, scale, is_causal, has_mask, st);
    }
    return fail(TL_EDTYPE, "decode_attention: expected float32, float16, or bfloat16");
}

// ------------------------------------------------- generic paged, row-wise --
template <typename T>
__global__ void __launch_bounds__(128) paged_rowwise_kernel(const T *__restrict__ q, const T *__restrict__ kp,
                                                            const T *__restrict__ vp, const int32_t *__restrict__ bt,
                                                            const int32_t *__restrict__ cl, T *__restrict__ out, int L,
                                                            int D, int num_pages, int page_size, int max_pages,
                                                            float scale, int is_causal, int num_kv_heads,
                                                            int num_heads) {
    constexpr int WARPS = 4;
    constexpr int MAXV = 4;  // D <= 128
    __shared__ float p_acc[WARPS][128];
    __shared__ float p_max[WARPS], p_sum[WARPS];
    const int query_index = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = query_index / L;
    const int query_pos = query_index - n * L;
    const int batch = n / num_heads;
    const int head = n - batch * num_heads;
    const int kv_head = head / (num_heads / num_kv_heads);
    const int ctx = cl[batch];
    const int vpl = (D + 31) / 32;
    const float scale2 = scale * LOG2E;

    float qv[MAXV], acc[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int d = lane + 32 * i;
        acc[i] = 0.f;
        qv[i] = (i < vpl && d < D) ? to_f(q[static_cast<size_t>(query_index) * D + d]) * scale2 : 0.f;
    }
    int visible = is_causal ? min(max(ctx - L + query_pos + 1, 0), ctx) : ctx;
    visible = min(visible, max_pages * page_size);
    float m = NEG_BIG, l = 0.f;
    for (int tok = warp; tok < visible; tok += WARPS) {
        const int lp = tok / page_size;
        const int pid = bt[static_cast<size_t>(batch) * max_pages + lp];
        if (pid < 0 || pid >= num_pages) continue;
        const size_t off = ((static_cast<size_t>(pid) * num_kv_heads + kv_head) * page_size + (tok - lp * page_size)) * D;
        float part = 0.f;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int d = lane + 32 * i;
            if (i < vpl && d < D) part += qv[i] * to_f(kp[off + d]);
        }
        const float score = warp_sum(part);
        const float nm = fmaxf(m, score);
        const float f_old = exp2f(m - nm);
        const float f_new = exp2f(score - nm);
        l = l * f_old + f_new;
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int d = lane + 32 * i;
            if (i < vpl && d < D) acc[i] = acc[i] * f_old + f_new * to_f(vp[off + d]);
        }
        m = nm;
    }
    if (lane == 0) p_max[warp] = m, p_sum[warp] = l;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int d = lane + 32 * i;
        if (i < vpl && d < D) p_acc[warp][d] = acc[i];
    }
    __syncthreads();
    float gm = NEG_BIG;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) gm = fmaxf(gm, p_max[w]);
    float gs = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) gs += p_sum[w] * exp2f(p_max[w] - gm);
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
        float o = 0.f;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) o += p_acc[w][d] * exp2f(p_max[w] - gm);
        out[static_cast<size_t>(query_index) * D + d] = from_f<T>(gs == 0.f ? 0.f : o / gs);  // metal :238-240
    }
}

int launch_paged_rowwise(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl,
                         void *out, int rows, int L, int D, int num_pages, int page_size, int max_pages, float scale,
                         int is_causal, int num_kv_heads, int num_heads, int dtype, cudaStream_t st) {
    if (rows * L == 0) return TL_OK;
    if (dtype == TL_F32)
        paged_rowwise_kernel<float><<<rows * L, 128, 0, st>>>(static_cast<const float *>(q), static_cast<const float *>(kp),
                                                             static_cast<const float *>(vp), bt, cl,
                                                             static_cast<float *>(out), L, D, num_pages, page_size,
                                                             max_pages, scale, is_causal, num_kv_heads, num_heads);
    else if (dtype == TL_BF16)
        paged_rowwise_kernel<__nv_bfloat16><<<rows * L, 128, 0, st>>>(
            static_cast<const __nv_bfloat16 *>(q), static_cast<const __nv_bfloat16 *>(kp),
            static_cast<const __nv_bfloat16 *>(vp), bt, cl, static_cast<__nv_bfloat16 *>(out), L, D, num_pages,
            page_size, max_pages, scale, is_causal, num_kv_heads, num_heads);
    else
        return fail(TL_EDTYPE, "paged_attention: q, key_pages, and value_pages must have the same float32 or bfloat16 dtype");
    TL_LAUNCH_CHECK("paged_rowwise");
    return TL_OK;
}

// ------------------------------------ bf16 D=128 GQA-grouped split-KV path --
constexpr int GQA_D = 128;
constexpr int GQA_WARPS = 4;
constexpr int GQA_THREADS = GQA_WARPS * 32;
constexpr int GQA_STEP = GQA_WARPS * 4;  // tokens per CTA iteration (4 per warp, 8 lanes each)
constexpr int GQA_RING = 6;          // cp.async steps in flight per lane (64 B each)
constexpr int GQA_PAGE_CACHE = 264;  // page ids of one split kept in shared memory

// Rows of one KV head are ordered r = head_in_group * L + l.
template <int RG>
__global__ void __launch_bounds__(GQA_THREADS) paged_gqa_kernel(
    const __nv_bfloat16 *__restrict__ q, const __nv_bfloat16 *__restrict__ kp, const __nv_bfloat16 *__restrict__ vp,
    const int32_t *__restrict__ bt, const int32_t *__restrict__ cl, __nv_bfloat16 *__restrict__ out,
    float *__restrict__ ws_o, float *__restrict__ ws_m, float *__restrict__ ws_l, int L, int num_pages, int page_size,
    int max_pages, float scale, int is_causal, int num_kv_heads, int num_heads, int row_groups, int splits,
    int tokens_per_split) {
    const int split = blockIdx.x % splits;
    const int rgi = blockIdx.x / splits;
    const int kv_head = blockIdx.y;
    const int batch = blockIdx.z;
    const int G = num_heads / num_kv_heads;
    const int R = G * L;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = lane >> 3;  // token slot of this lane group
    const int c = lane & 7;   // 16-dim chunk owned by this lane
    const int ctx = cl[batch];
    const int cap = max_pages * page_size;  // keys the block table can hold
    const float scale2 = scale * LOG2E;

    float qv[RG][16], acc[RG][16], m[RG], l[RG];
    int vis[RG];
    int vis_max = 0;
#pragma unroll
    for (int r = 0; r < RG; ++r) {
        const int row = rgi * RG + r;
        m[r] = NEG_BIG;
        l[r] = 0.f;
        vis[r] = 0;
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[r][i] = 0.f, qv[r][i] = 0.f;
        if (row < R) {
            const int hl = row / L, pos = row - hl * L;
            const int qi = (batch * num_heads + kv_head * G + hl) * L + pos;
            vis[r] = min(is_causal ? min(max(ctx - L + pos + 1, 0), ctx) : ctx, cap);  // causal shift first, as paged_rowwise_kernel
            vis_max = max(vis_max, vis[r]);
            const uint4 *src = reinterpret_cast<const uint4 *>(q + static_cast<size_t>(qi) * GQA_D + c * 16);
            const uint4 a = src[0], b = src[1];
            const uint32_t raw[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float2 f = unpack2<__nv_bfloat16>(raw[i]);
                qv[r][2 * i] = f.x * scale2;
                qv[r][2 * i + 1] = f.y * scale2;
            }
        }
    }

    const int begin = split * tokens_per_split;
    const int end = min(vis_max, begin + tokens_per_split);

    // Page ids of this split, resolved once (no dependent global load inside the token loop).
    __shared__ int s_pages[GQA_PAGE_CACHE];
    const int first_page = begin / page_size;
    {
        const int last_page = end > begin ? (end - 1) / page_size : first_page - 1;
        for (int i = threadIdx.x; i <= last_page - first_page && i < GQA_PAGE_CACHE; i += GQA_THREADS)
            s_pages[i] = bt[static_cast<size_t>(batch) * max_pages + first_page + i];
    }
    __syncthreads();
    auto page_of = [&](int lp) -> int {
        const int i = lp - first_page;
        return i < GQA_PAGE_CACHE ? s_pages[i] : bt[static_cast<size_t>(batch) * max_pages + lp];
    };

    // Each lane owns 32 B of K and 32 B of V of one token per step; those bytes travel through a
    // PRIVATE shared-memory ring filled by cp.async, GQA_RING steps deep (8-12 KiB in flight per
    // warp), so the HBM latency is paid once per split instead of once per 4 tokens.
    extern __shared__ __align__(16) unsigned char s_ring[];  // GQA_THREADS * GQA_RING * 64 bytes (dynamic)
    unsigned char *my_ring = s_ring + static_cast<size_t>(threadIdx.x) * GQA_RING * 64;
    const uint32_t my_ring_s = static_cast<uint32_t>(__cvta_generic_to_shared(my_ring));
    const int steps = end > begin + warp * 4 ? (end - begin - warp * 4 + GQA_STEP - 1) / GQA_STEP : 0;
    auto token_src = [&](int step, size_t &off) -> bool {
        const int tok = begin + warp * 4 + step * GQA_STEP + j;
        if (step >= steps || tok >= end) return false;
        const int lp = tok / page_size;
        const int pid = page_of(lp);
        if (pid < 0 || pid >= num_pages) return false;
        off = ((static_cast<size_t>(pid) * num_kv_heads + kv_head) * page_size + (tok - lp * page_size)) * GQA_D + c * 16;
        return true;
    };
    auto issue = [&](int step) {
        size_t off;
        if (token_src(step, off)) {
            const uint32_t dst = my_ring_s + (step % GQA_RING) * 64;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(kp + off) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16), "l"(kp + off + 8) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 32), "l"(vp + off) : "memory");
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 48), "l"(vp + off + 8) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
#pragma unroll
    for (int i = 0; i < GQA_RING - 1; ++i) issue(i);

    for (int step = 0; step < steps; ++step) {
        const int tok = begin + warp * 4 + step * GQA_STEP + j;
        size_t unused;
        const bool valid = token_src(step, unused);
        asm volatile("cp.async.wait_group %0;" ::"n"(GQA_RING - 2) : "memory");
        uint4 k0 = make_uint4(0, 0, 0, 0), k1 = k0, v0 = k0, v1 = k0;
        if (valid) {  // a lane reads back only the bytes it copied itself: no cross-lane sync needed
            const uint4 *slot = reinterpret_cast<const uint4 *>(my_ring + (step % GQA_RING) * 64);
            k0 = slot[0], k1 = slot[1], v0 = slot[2], v1 = slot[3];
        }
        issue(step + GQA_RING - 1);
        float kf[16];
        {
            const uint32_t raw[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float2 f = unpack2<__nv_bfloat16>(raw[i]);
                kf[2 * i] = f.x, kf[2 * i + 1] = f.y;
            }
        }
        float p[RG], corr[RG];
#pragma unroll
        for (int r = 0; r < RG; ++r) {
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) s += qv[r][i] * kf[i];
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            s += __shfl_xor_sync(0xffffffffu, s, 4);
            if (!valid || tok >= vis[r]) s = -CUDART_INF_F;
            const float nm = fmaxf(m[r], s);
            corr[r] = exp2f(m[r] - nm);
            p[r] = exp2f(s - nm);
            l[r] = l[r] * corr[r] + p[r];
            m[r] = nm;
        }
        float vf[16];
        {
            const uint32_t raw[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float2 f = unpack2<__nv_bfloat16>(raw[i]);
                vf[2 * i] = f.x, vf[2 * i + 1] = f.y;
            }
        }
#pragma unroll
        for (int r = 0; r < RG; ++r)
#pragma unroll
            for (int i = 0; i < 16; ++i) acc[r][i] = acc[r][i] * corr[r] + p[r] * vf[i];
    }

    // merge the 4 lane groups of the warp (same dims, disjoint tokens)
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
#pragma unroll
        for (int r = 0; r < RG; ++r) {
            const float mo = __shfl_xor_sync(0xffffffffu, m[r], o);
            const float lo = __shfl_xor_sync(0xffffffffu, l[r], o);
            const float nm = fmaxf(m[r], mo);
            const float fs = exp2f(m[r] - nm), fo = exp2f(mo - nm);
            l[r] = l[r] * fs + lo * fo;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float ao = __shfl_xor_sync(0xffffffffu, acc[r][i], o);
                acc[r][i] = acc[r][i] * fs + ao * fo;
            }
            m[r] = nm;
        }
    }
    // the ring is drained: reuse its memory for the cross-warp merge
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    float(*s_acc)[RG][GQA_D] = reinterpret_cast<float(*)[RG][GQA_D]>(s_ring);
    __shared__ float s_m[GQA_WARPS][RG], s_l[GQA_WARPS][RG];
    if (j == 0) {
#pragma unroll
        for (int r = 0; r < RG; ++r) {
#pragma unroll
            for (int i = 0; i < 16; ++i) s_acc[warp][r][c * 16 + i] = acc[r][i];
            if (c == 0) s_m[warp][r] = m[r], s_l[warp][r] = l[r];
        }
    }
    __syncthreads();
    const int d = threadIdx.x;  // GQA_THREADS == GQA_D
#pragma unroll
    for (int r = 0; r < RG; ++r) {
        const int row = rgi * RG + r;
        if (row >= R) continue;
        float gm = NEG_BIG;
#pragma unroll
        for (int w = 0; w < GQA_WARPS; ++w) gm = fmaxf(gm, s_m[w][r]);
        float gl = 0.f, o = 0.f;
#pragma unroll
        for (int w = 0; w < GQA_WARPS; ++w) {
            const float f = exp2f(s_m[w][r] - gm);
            gl += s_l[w][r] * f;
            o += s_acc[w][r][d] * f;
        }
        const int hl = row / L, pos = row - hl * L;
        const size_t qi = static_cast<size_t>(batch * num_heads + kv_head * G + hl) * L + pos;
        if (splits == 1) {
            out[qi * GQA_D + d] = __float2bfloat16_rn(gl == 0.f ? 0.f : o / gl);
        } else {
            ws_o[(qi * splits + split) * GQA_D + d] = o;
            if (d == 0) ws_m[qi * splits + split] = gm, ws_l[qi * splits + split] = gl;
        }
    }
}

__global__ void __launch_bounds__(GQA_THREADS) paged_gqa_merge_kernel(const float *ws_o, const float *ws_m, const float *ws_l,
                                                                      __nv_bfloat16 *out, int splits, int L, int Hq, int token_major) {
    // Dependent launch (common.cuh): the partials are the attention kernel's output, in a workspace every layer rewrites
    // - read them through L2.
    griddep_launch();
    griddep_wait();
    const size_t qi = blockIdx.x;
    const int d = threadIdx.x, lane = d & 31;
    const float *pm = ws_m + qi * splits, *pl = ws_l + qi * splits;
    // Latency matters here (the whole long-context decode attention of one request is a few microseconds): every warp reduces the
    // split scalars on its own with ONE load round per lane (splits <= 32) and a shuffle tree, then the output column is
    // gathered eight independent loads at a time.  (The first version walked the splits in two dependent loops: 2 x
    // splits L2 round trips per thread.)  Fixed order everywhere: same bits on every run.
    float gm = NEG_BIG;
    for (int s = lane; s < splits; s += 32) gm = fmaxf(gm, ld_cg(pm + s));
    gm = warp_max(gm);
    float gl = 0.f;
    for (int s = lane; s < splits; s += 32) gl += ld_cg(pl + s) * exp2f(ld_cg(pm + s) - gm);
    gl = warp_sum(gl);
    float o = 0.f;
    const float *po = ws_o + qi * splits * GQA_D + d;
    for (int s0 = 0; s0 < splits; s0 += 8) {
        float v[8], f[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const bool live = s0 + j < splits;
            v[j] = live ? ld_cg(po + static_cast<size_t>(s0 + j) * GQA_D) : 0.f;
            f[j] = live ? ld_cg(pm + s0 + j) : gm;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (s0 + j < splits) o += v[j] * exp2f(f[j] - gm);
    }
    // partial row qi is (b * Hq + head) * L + l; token-major output (the o projection's layout) is (b * L + l) * Hq + head.
    // A split whose tiles all lie past a row's last visible key left m = -1e30, l = 0 for that row: weight 0 here.
    size_t oi = qi;
    if (token_major) {
        const size_t l = qi % L, bh = qi / L;
        oi = (bh / Hq * L + l) * Hq + bh % Hq;
    }
    out[oi * GQA_D + d] = __float2bfloat16_rn(gl == 0.f ? 0.f : o / gl);
}

int launch_paged_gqa_merge(const float *ws_o, const float *ws_m, const float *ws_l, void *out, int rows_total, int splits, cudaStream_t st,
                           int L, int Hq, bool token_major) {
    launch_chained(paged_gqa_merge_kernel, dim3(static_cast<unsigned>(rows_total)), dim3(GQA_THREADS), 0, st, ws_o, ws_m, ws_l,
                   static_cast<__nv_bfloat16 *>(out), splits, L, Hq, token_major ? 1 : 0);
    TL_LAUNCH_CHECK("paged_gqa_merge");
    return TL_OK;
}

int launch_paged_gqa(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl, void *out,
                     int rows, int L, int num_pages, int page_size, int max_pages, float scale, int is_causal,
                     int num_kv_heads, int num_heads, bool allow_split, void *ws, size_t ws_bytes, cudaStream_t st) {
    if (rows * L == 0) return TL_OK;
    const int batch = rows / num_heads;
    const int G = num_heads / num_kv_heads;
    const int R = G * L;
    const int RG = R >= 3 ? 4 : R;
    const int row_groups = ceil_div(R, RG);
    const long long bound = static_cast<long long>(max_pages) * page_size;
    const long long base_ctas = static_cast<long long>(batch) * num_kv_heads * row_groups;
    int splits = 1;
    if (allow_split) {
        const long long target = 4LL * sm_count();
        long long want = ceil_div_ll(target, base_ctas);
        const long long most = bound / 128 > 0 ? bound / 128 : 1;  // at least 128 tokens per split (larger minimums lengthen the per-step chain at short contexts)
        if (want > most) want = most;
        if (want > PAGED_MAX_SPLITS) want = PAGED_MAX_SPLITS;
        if (want < 1) want = 1;
        splits = static_cast<int>(want);
    }
    int tps = static_cast<int>(ceil_div_ll(bound, splits));
    tps = ceil_div(tps, GQA_STEP) * GQA_STEP;
    splits = static_cast<int>(ceil_div_ll(bound, tps));
    if (splits < 1) splits = 1;
    float *ws_o = nullptr, *ws_m = nullptr, *ws_l = nullptr;
    if (splits > 1) {
        const size_t rows_total = static_cast<size_t>(rows) * L;
        const size_t need = rows_total * splits * (GQA_D + 2) * sizeof(float);
        if (ws == nullptr || ws_bytes < need) return fail(TL_EWORKSPACE, "paged_attention: workspace too small (%zu < %zu)", ws_bytes, need);
        ws_o = static_cast<float *>(ws);
        ws_m = ws_o + rows_total * splits * GQA_D;
        ws_l = ws_m + rows_total * splits;
    }
    if (num_kv_heads > 65535 || batch > 65535) return fail(TL_EINVAL, "paged_attention: grid too large");
    dim3 grid(static_cast<unsigned>(splits) * row_groups, num_kv_heads, batch);
    auto qp = static_cast<const __nv_bfloat16 *>(q);
    auto kpp = static_cast<const __nv_bfloat16 *>(kp);
    auto vpp = static_cast<const __nv_bfloat16 *>(vp);
    auto op = static_cast<__nv_bfloat16 *>(out);
    constexpr size_t ring_bytes = static_cast<size_t>(GQA_THREADS) * GQA_RING * 64;
    static_assert(ring_bytes >= sizeof(float) * GQA_WARPS * 4 * GQA_D, "merge scratch aliases the ring");
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(paged_gqa_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ring_bytes));
        cudaFuncSetAttribute(paged_gqa_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ring_bytes));
        cudaFuncSetAttribute(paged_gqa_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ring_bytes));
        configured = true;
    }
#define TL_GQA(RGV)                                                                                                   \
    paged_gqa_kernel<RGV><<<grid, GQA_THREADS, ring_bytes, st>>>(qp, kpp, vpp, bt, cl, op, ws_o, ws_m, ws_l, L, num_pages,     \
                                                       page_size, max_pages, scale, is_causal, num_kv_heads,         \
                                                       num_heads, row_groups, splits, tps)
    if (RG == 4)
        TL_GQA(4);
    else if (RG == 2)
        TL_GQA(2);
    else
        TL_GQA(1);
#undef TL_GQA
    TL_LAUNCH_CHECK("paged_gqa");
    if (splits > 1) {
        launch_chained(paged_gqa_merge_kernel, dim3(static_cast<unsigned>(rows * L)), dim3(GQA_THREADS), 0, st, static_cast<const float *>(ws_o),
                       static_cast<const float *>(ws_m), static_cast<const float *>(ws_l), op, splits, L, num_heads, 0);
        TL_LAUNCH_CHECK("paged_gqa_merge");
    }
    return TL_OK;
}

}  // namespace tl
