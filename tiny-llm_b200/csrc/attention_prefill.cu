// Paged causal prefill attention on the tensor cores (bf16, head_dim 128).
//
// Replaces paged_attention_prefill / the tiled FlashAttention of the reference
// (src/extensions_ref/src/paged_attention.metal:250-506,
// flash_attention.metal) for L > 8, where the CUDA-core GQA kernel would dominate a Qwen3-4B prefill.
//
// Shape of the computation (FlashAttention-2 style, one pass, online softmax):
//   grid  = (ceil(L / 64) query tiles, B * Hq heads), longest (last) query tiles first
//   CTA   = 4 warps, 16 query rows each; Q fragments live in registers for the whole kernel
//   loop  = 64-key tiles of the request's paged K/V, cp.async'ed row by row through the block
//           table into a double-buffered shared-memory stage (row stride 272 B: conflict-free
//           ldmatrix), S = Q K^T and O += P V with mma.sync.m16n8k16 (fp32 accumulate),
//           probabilities rounded to bf16 for the second product (as every flash kernel does)
//   mask  = bottom-right aligned causal limit clamp(ctx - L + l + 1, 0, ctx) per query row
//           (attention.py:40-58 semantics), then at most the block table's keys; rows/pages
//           outside the context contribute nothing
//
// This is the mma.sync version; page sizes that are a multiple of 64 take the wgmma + TMA kernel
// (attention_prefill_tc.cu, DESIGN.md section 4).
#include <math_constants.h>

#include "common.cuh"
#include "kernels.h"

namespace tl {

constexpr int FA_BM = 64, FA_BN = 64, FA_D = 128;
constexpr int FA_WARPS = 4, FA_THREADS = FA_WARPS * 32;
constexpr int FA_STRIDE = FA_D + 8;  // bf16 elements per shared-memory row
constexpr size_t FA_TILE_BYTES = static_cast<size_t>(FA_BN) * FA_STRIDE * 2;
constexpr size_t FA_SMEM_BYTES = 5 * FA_TILE_BYTES;  // Q + 2 x (K, V)

typedef __nv_bfloat16 bf16;

__device__ __forceinline__ uint32_t fa_smem(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void fa_cp16(uint32_t dst, const void *src, bool valid) {  // invalid rows are zero-filled
    const int bytes = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fa_ldsm4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void fa_ldsm4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ float fa_exp2(float x) {  // ex2.approx: 2 ulp, exp2(-inf) = 0; inputs are <= 0 here
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ void fa_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(FA_THREADS) paged_prefill_fa_kernel(const bf16 *__restrict__ q, const bf16 *__restrict__ kp,
                                                                      const bf16 *__restrict__ vp, const int32_t *__restrict__ bt,
                                                                      const int32_t *__restrict__ cl, bf16 *__restrict__ out, int L,
                                                                      int Hq, int Hkv, int page_size, int max_pages, int num_pages,
                                                                      float scale, int causal) {
    extern __shared__ __align__(128) unsigned char fa_raw[];
    __shared__ int bad[2];  // (tile index + 1) of the last tile loaded into the stage that had a row with an invalid page id
    bf16 *q_s = reinterpret_cast<bf16 *>(fa_raw);
    bf16 *k_s = q_s + FA_BM * FA_STRIDE;      // [2][64][136]
    bf16 *v_s = k_s + 2 * FA_BN * FA_STRIDE;  // [2][64][136]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int qt = gridDim.x - 1 - blockIdx.x;  // long tiles first
    const int head_row = blockIdx.y;
    const int b = head_row / Hq, h = head_row - b * Hq;
    const int kvh = h / (Hq / Hkv);
    const int ctx_all = cl[b];
    const int ctx = min(ctx_all, max_pages * page_size);  // keys the block table holds
    const int q0 = qt * FA_BM;
    // the causal shift uses the whole context, the block table clamps afterwards (attention_decode.cu)
    auto limit = [&](int l) { return min(causal ? max(0, min(ctx_all, ctx_all - L + l + 1)) : ctx_all, ctx); };
    const int kmax = limit(min(q0 + FA_BM - 1, L - 1));  // keys any row of this tile may see
    const int nkt = (kmax + FA_BN - 1) / FA_BN;
    if (threadIdx.x < 2) bad[threadIdx.x] = 0;
    __syncthreads();  // the loaders below may set the flags

    // ---- Q tile -> shared (rows past L are zero)
    const bf16 *q_head = q + static_cast<size_t>(head_row) * L * FA_D;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = threadIdx.x + i * FA_THREADS, row = c >> 4, col = (c & 15) * 8;
        const bool ok = q0 + row < L;
        fa_cp16(fa_smem(q_s + row * FA_STRIDE + col), q_head + static_cast<size_t>(ok ? q0 + row : 0) * FA_D + col, ok);
    }
    const bool tile_in_page = page_size % FA_BN == 0;  // a 64-key tile never straddles pages: one table lookup per tile
    auto load_kv = [&](int kt, int stage) {
        bf16 *ks = k_s + stage * FA_BN * FA_STRIDE, *vs = v_s + stage * FA_BN * FA_STRIDE;
        int tile_pid = -1, tile_row0 = 0;
        if (tile_in_page) {
            const int lp = kt * FA_BN / page_size;
            tile_pid = bt[static_cast<size_t>(b) * max_pages + lp];
            tile_row0 = kt * FA_BN - lp * page_size;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int c = threadIdx.x + i * FA_THREADS, row = c >> 4, col = (c & 15) * 8;
            const int j = kt * FA_BN + row;
            bool ok = j < ctx;
            size_t off = 0;
            if (ok) {
                int pid = tile_pid, prow = tile_row0 + row;
                if (!tile_in_page) {
                    const int lp = j / page_size;
                    pid = bt[static_cast<size_t>(b) * max_pages + lp];
                    prow = j - lp * page_size;
                }
                ok = pid >= 0 && pid < num_pages;
                if (ok)
                    off = ((static_cast<size_t>(pid) * Hkv + kvh) * page_size + prow) * FA_D + col;
                else if ((c & 15) == 0)
                    bad[stage] = kt + 1;
            }
            fa_cp16(fa_smem(ks + row * FA_STRIDE + col), kp + off, ok);
            fa_cp16(fa_smem(vs + row * FA_STRIDE + col), vp + off, ok);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    if (nkt > 0) load_kv(0, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();

    // ---- Q fragments (A operand): 8 k-steps x 4 registers
    uint32_t qa[8][4];
    {
        const int row = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) fa_ldsm4(qa[ks], fa_smem(q_s + row * FA_STRIDE + ks * 16 + ((lane >> 4) & 1) * 8));
    }
    const int l0 = q0 + warp * 16 + g, l1 = l0 + 8;  // the two query rows of this thread
    const int lim0 = l0 < L ? limit(l0) : 0, lim1 = l1 < L ? limit(l1) : 0;
    const int lim_min = limit(min(q0 + warp * 16, L - 1));  // smallest limit among this warp's rows
    const float c2 = scale * 1.44269504089f;
    float o[16][4];
#pragma unroll
    for (int n = 0; n < 16; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
    float m0 = -CUDART_INF_F, m1 = -CUDART_INF_F, sum0 = 0.f, sum1 = 0.f;

    for (int kt = 0; kt < nkt; ++kt) {
        const int stage = kt & 1;
        if (kt > 0) {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads();  // tile kt landed; everyone is done with the other stage
        }
        if (kt + 1 < nkt) load_kv(kt + 1, stage ^ 1);
        const bf16 *ks_t = k_s + stage * FA_BN * FA_STRIDE, *vs_t = v_s + stage * FA_BN * FA_STRIDE;

        // ---- S = Q K^T : 16 x 64 per warp
        float s[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
            for (int np = 0; np < 4; ++np) {
                uint32_t kb[4];
                const int key = np * 16 + (lane & 7) + ((lane >> 4) & 1) * 8;
                fa_ldsm4(kb, fa_smem(ks_t + key * FA_STRIDE + ks * 16 + ((lane >> 3) & 1) * 8));
                fa_mma(s[2 * np], qa[ks], kb[0], kb[1]);
                fa_mma(s[2 * np + 1], qa[ks], kb[2], kb[3]);
            }
        }
        // ---- scale, mask (diagonal / context-edge / invalid-page tiles only), online softmax
        const int j0 = kt * FA_BN;
        const bool tile_bad = bad[stage] == kt + 1;
        const bool full = j0 + FA_BN <= lim_min && !tile_bad;
        float mx0 = -CUDART_INF_F, mx1 = -CUDART_INF_F;
#pragma unroll
        for (int n = 0; n < 8; ++n) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float a0 = s[n][e] * c2, a1 = s[n][2 + e] * c2;
                if (!full) {
                    const int j = j0 + n * 8 + 2 * t + e;
                    bool okj = true;
                    if (tile_bad) {
                        const int pid = bt[static_cast<size_t>(b) * max_pages + min(j, ctx - 1) / page_size];
                        okj = pid >= 0 && pid < num_pages;
                    }
                    if (j >= lim0 || !okj) a0 = -CUDART_INF_F;
                    if (j >= lim1 || !okj) a1 = -CUDART_INF_F;
                }
                s[n][e] = a0, s[n][2 + e] = a1;
                mx0 = fmaxf(mx0, a0), mx1 = fmaxf(mx1, a1);
            }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float nm0 = fmaxf(m0, mx0), nm1 = fmaxf(m1, mx1);
        const float r0 = nm0 == -CUDART_INF_F ? 0.f : nm0, r1 = nm1 == -CUDART_INF_F ? 0.f : nm1;  // fully masked so far
        const float al0 = fa_exp2(m0 - r0), al1 = fa_exp2(m1 - r1);
        m0 = nm0, m1 = nm1;
        float ps0 = 0.f, ps1 = 0.f;
        uint32_t pa[4][4];  // P as A fragments: 4 k-steps of 16 keys
#pragma unroll
        for (int n = 0; n < 8; ++n) {
            const float p00 = fa_exp2(s[n][0] - r0), p01 = fa_exp2(s[n][1] - r0);
            const float p10 = fa_exp2(s[n][2] - r1), p11 = fa_exp2(s[n][3] - r1);
            ps0 += p00 + p01, ps1 += p10 + p11;
            pa[n >> 1][(n & 1) * 2] = pack2<bf16>(p00, p01);
            pa[n >> 1][(n & 1) * 2 + 1] = pack2<bf16>(p10, p11);
        }
        sum0 = sum0 * al0 + ps0, sum1 = sum1 * al1 + ps1;
#pragma unroll
        for (int n = 0; n < 16; ++n) o[n][0] *= al0, o[n][1] *= al0, o[n][2] *= al1, o[n][3] *= al1;
        // ---- O += P V : 16 x 128 per warp
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int dp = 0; dp < 8; ++dp) {
                uint32_t vb[4];
                const int key = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                fa_ldsm4_t(vb, fa_smem(vs_t + key * FA_STRIDE + dp * 16 + ((lane >> 4) & 1) * 8));
                fa_mma(o[2 * dp], pa[kk], vb[0], vb[1]);
                fa_mma(o[2 * dp + 1], pa[kk], vb[2], vb[3]);
            }
        }
    }
    // ---- finalize: row sums across the 4 lanes of a row, normalise, store
    sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
    sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
    sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
    sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
    const float i0 = sum0 == 0.f ? 0.f : 1.0f / sum0, i1 = sum1 == 0.f ? 0.f : 1.0f / sum1;
    bf16 *o_head = out + static_cast<size_t>(head_row) * L * FA_D;
#pragma unroll
    for (int n = 0; n < 16; ++n) {
        if (l0 < L) *reinterpret_cast<uint32_t *>(o_head + static_cast<size_t>(l0) * FA_D + n * 8 + 2 * t) = pack2<bf16>(o[n][0] * i0, o[n][1] * i0);
        if (l1 < L) *reinterpret_cast<uint32_t *>(o_head + static_cast<size_t>(l1) * FA_D + n * 8 + 2 * t) = pack2<bf16>(o[n][2] * i1, o[n][3] * i1);
    }
}

int launch_paged_prefill_fa(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl, void *out, int rows,
                            int L, int num_pages, int page_size, int max_pages, float scale, int is_causal, int num_kv_heads,
                            int num_heads, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(paged_prefill_fa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(FA_SMEM_BYTES)) != cudaSuccess)
            return fail(TL_ECUDA, "paged_attention: cannot raise shared memory limit");
        configured = true;
    }
    dim3 grid((L + FA_BM - 1) / FA_BM, rows);
    paged_prefill_fa_kernel<<<grid, FA_THREADS, FA_SMEM_BYTES, st>>>(
        static_cast<const bf16 *>(q), static_cast<const bf16 *>(kp), static_cast<const bf16 *>(vp), bt, cl, static_cast<bf16 *>(out), L,
        num_heads, num_kv_heads, page_size, max_pages, num_pages, scale, is_causal);
    TL_LAUNCH_CHECK("paged_prefill_fa");
    return TL_OK;
}

}  // namespace tl
