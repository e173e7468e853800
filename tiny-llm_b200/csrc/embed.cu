// Heads of packed passes over the model's final hidden states.  Sentence embeddings (tl_embed_pool, DESIGN.md section
// 17): one CTA per segment applies the model's final RMSNorm to the rows it pools, pools them (the last row, or the fp32
// mean of the normalised rows), truncates to the first d features and optionally divides by the L2 norm.  Selected-token
// logits (tl_select_logits, section 19): one CTA per listed row normalises it the same way and computes the logits of a
// few token ids from the packed LM head, and their log-softmax.
//
// A row is normalised in rms_norm_kernel's order (elementwise.cu), as moe_gather does (moe.cu): TPR threads per row
// (rms_norm_path: 32 up to 512 elements, else 256), thread `lane` owning the chunks of EPV consecutive elements at
// lane * EPV + n * TPR * EPV (16-byte vectors when rms_norm's VEC path applies, else single elements), its sum of
// squares reduced by the same warp and CTA steps.  So each normalised row is tl_rms_norm's bit for bit.  The pooled
// vector lives in shared memory, each element written only by the thread that owns it, so the mean is summed in row
// order per element and the L2 norm is one fixed-order CTA reduction.
#include <math_constants.h>

#include "common.cuh"
#include "kernels.h"

namespace tl {

template <int TPR>
__device__ __forceinline__ float pool_sum(float v, float *part) {
    v = warp_sum(v);
    if constexpr (TPR > 32) {
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
        __syncthreads();
        v = warp_sum((threadIdx.x & 31) < TPR / 32 ? part[threadIdx.x & 31] : 0.f);
        __syncthreads();  // part is written again by the next reduction
    }
    return v;
}

// 1 / rms of row xr (rms_norm_kernel's visiting order and reductions); the caller multiplies x * inv * w per element.
template <typename T, int TPR, int EPV>
__device__ __forceinline__ float row_rms_inv(const T *xr, int H, float eps, float *part) {
    float ss = 0.f;
    for (int c = threadIdx.x * EPV; c < H; c += TPR * EPV)
#pragma unroll
        for (int q = 0; q < EPV; ++q) {
            const float v = to_f(ld_cg(xr + c + q));
            ss += v * v;
        }
    ss = pool_sum<TPR>(ss, part);
    return rsqrtf(ss / static_cast<float>(H) + eps);
}

template <typename T, int TPR, int EPV>
__global__ void __launch_bounds__(256) embed_pool_kernel(const T *__restrict__ x, const T *__restrict__ w, float eps, const int32_t *__restrict__ seg,
                                                        int rows, int H, int d, int mean, int normalize, float *__restrict__ out) {
    extern __shared__ float acc[];  // [H] the pooled row
    __shared__ float part[TPR / 32];
    griddep_launch();
    griddep_wait();
    const int s = blockIdx.x, lane = threadIdx.x;
    const int r0 = max(ld_cg(seg + s), 0), r1 = min(ld_cg(seg + s + 1), rows);  // an empty segment pools to zeros
    for (int c = lane * EPV; c < H; c += TPR * EPV)
#pragma unroll
        for (int q = 0; q < EPV; ++q) acc[c + q] = 0.f;
    for (int r = r1 <= r0 ? r1 : mean ? r0 : r1 - 1; r < r1; ++r) {
        const T *xr = x + static_cast<size_t>(r) * H;
        const float inv = row_rms_inv<T, TPR, EPV>(xr, H, eps, part);
        for (int c = lane * EPV; c < H; c += TPR * EPV)
#pragma unroll
            for (int q = 0; q < EPV; ++q) acc[c + q] += to_f(from_f<T>(to_f(ld_cg(xr + c + q)) * inv * to_f(w[c + q])));
    }
    const float count = static_cast<float>(mean && r1 > r0 ? r1 - r0 : 1);
    float ss = 0.f;
    for (int c = lane * EPV; c < d; c += TPR * EPV)
#pragma unroll
        for (int q = 0; q < EPV; ++q)
            if (c + q < d) {
                const float v = acc[c + q] / count;
                acc[c + q] = v;
                ss += v * v;
            }
    float nrm = 1.f;
    if (normalize) {
        nrm = sqrtf(pool_sum<TPR>(ss, part));
        if (nrm == 0.f) nrm = 1.f;  // a zero vector stays zero
    }
    float *o = out + static_cast<size_t>(s) * d;
    for (int c = lane * EPV; c < d; c += TPR * EPV)
#pragma unroll
        for (int q = 0; q < EPV; ++q)
            if (c + q < d) o[c + q] = acc[c + q] / nrm;
}

template <typename T>
static cudaError_t embed_pool_t(const void *x, const void *w, float eps, const int32_t *seg, int n, int rows, int H, int d, int mean,
                                int normalize, float *out, int dtype, cudaStream_t st) {
    bool vec = false;
    const int tpr = rms_norm_path(H, dtype, x, w, x, &vec);
    const T *xp = static_cast<const T *>(x), *wp = static_cast<const T *>(w);
    const size_t smem = static_cast<size_t>(H) * sizeof(float);
    constexpr int V = 16 / sizeof(T);
    if (tpr == 32)
        return vec ? launch_chained(embed_pool_kernel<T, 32, V>, dim3(n), dim3(32), smem, st, xp, wp, eps, seg, rows, H, d, mean, normalize, out)
                   : launch_chained(embed_pool_kernel<T, 32, 1>, dim3(n), dim3(32), smem, st, xp, wp, eps, seg, rows, H, d, mean, normalize, out);
    return vec ? launch_chained(embed_pool_kernel<T, 256, V>, dim3(n), dim3(256), smem, st, xp, wp, eps, seg, rows, H, d, mean, normalize, out)
               : launch_chained(embed_pool_kernel<T, 256, 1>, dim3(n), dim3(256), smem, st, xp, wp, eps, seg, rows, H, d, mean, normalize, out);
}

int launch_embed_pool(const void *x, const void *w, float eps, const int32_t *seg, int n, int rows, int H, int d, int mean, int normalize,
                      float *out, int dtype, cudaStream_t st) {
    if (n == 0) return TL_OK;
    const cudaError_t e = dtype == TL_F16 ? embed_pool_t<__half>(x, w, eps, seg, n, rows, H, d, mean, normalize, out, dtype, st)
                                          : embed_pool_t<__nv_bfloat16>(x, w, eps, seg, n, rows, H, d, mean, normalize, out, dtype, st);
    if (e != cudaSuccess) return fail(TL_ECUDA, "embed_pool: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("embed_pool");
    return TL_OK;
}

// ------------------------------------------------------------ selected-token logits --
// CTA s: row r = row_idx[s] of x, RMS-normalised into hs (T-rounded, as tl_rms_norm writes it); then for each id i the
// dot product of hs with the LM-head row of ids[i], each weight T(code * scale + bias) (code * scale is exact in fp32:
// at most 8 + 11 significant bits), summed in fp32 per thread over its words in increasing order, then by pool_sum's
// fixed reduction, and rounded to T as every LM-head route rounds its output.  Lane 0 then takes the fp32 log-softmax
// of the m logits in index order.  A row or id out of range gives NaN for what it touches; nothing is read for it.
template <typename T, int TPR, int EPV, int BITS>
__global__ void __launch_bounds__(256) select_logits_kernel(const T *__restrict__ x, const T *__restrict__ w, float eps,
                                                            const int32_t *__restrict__ row_idx, int rows, int H, const uint32_t *__restrict__ wq,
                                                            const T *__restrict__ scales, const T *__restrict__ biases, int V,
                                                            const int32_t *__restrict__ ids, int m, float *__restrict__ logits,
                                                            float *__restrict__ logprobs) {
    extern __shared__ __align__(16) float hs[];  // [H] the normalised row
    __shared__ float part[TPR / 32];
    __shared__ float lg[TL_SELECT_MAX_IDS];
    griddep_launch();
    griddep_wait();
    constexpr int PER = 32 / BITS;  // codes per word
    const int s = blockIdx.x, lane = threadIdx.x;
    const int r = ld_cg(row_idx + s);
    const bool row_ok = r >= 0 && r < rows;
    if (row_ok) {
        const T *xr = x + static_cast<size_t>(r) * H;
        const float inv = row_rms_inv<T, TPR, EPV>(xr, H, eps, part);
        for (int c = lane * EPV; c < H; c += TPR * EPV)
#pragma unroll
            for (int q = 0; q < EPV; ++q) hs[c + q] = to_f(from_f<T>(to_f(ld_cg(xr + c + q)) * inv * to_f(w[c + q])));
    }
    __syncthreads();
    const int words = H / PER, groups = H / 128;
    for (int i = 0; i < m; ++i) {
        const int id = ld_cg(ids + i);
        const bool ok = row_ok && id >= 0 && id < V;
        float acc = 0.f;
        if (ok) {
            const uint32_t *wrow = wq + static_cast<size_t>(id) * words;
            const T *srow = scales + static_cast<size_t>(id) * groups, *brow = biases + static_cast<size_t>(id) * groups;
            for (int k = lane; k < words; k += TPR) {
                const uint32_t packed = wrow[k];
                const int grp = k * PER / 128;
                const float sc = to_f(srow[grp]), bi = to_f(brow[grp]);
                const float4 *h4 = reinterpret_cast<const float4 *>(hs + k * PER);
#pragma unroll
                for (int v4 = 0; v4 < PER / 4; ++v4) {
                    const float4 h = h4[v4];
                    const float hv[4] = {h.x, h.y, h.z, h.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float code = static_cast<float>((packed >> (BITS * (4 * v4 + e))) & ((1u << BITS) - 1u));
                        acc += to_f(from_f<T>(code * sc + bi)) * hv[e];
                    }
                }
            }
        }
        acc = pool_sum<TPR>(acc, part);
        if (lane == 0) lg[i] = ok ? to_f(from_f<T>(acc)) : CUDART_NAN_F;
    }
    if (lane == 0) {
        float mx = -CUDART_INF_F;
        for (int i = 0; i < m; ++i) mx = fmaxf(mx, lg[i]);
        float sum = 0.f;
        for (int i = 0; i < m; ++i) sum += expf(lg[i] - mx);
        const float lse = mx + logf(sum);
        bool any_nan = false;
        for (int i = 0; i < m; ++i) any_nan |= lg[i] != lg[i];
        for (int i = 0; i < m; ++i) {
            logits[static_cast<size_t>(s) * m + i] = lg[i];
            logprobs[static_cast<size_t>(s) * m + i] = any_nan ? CUDART_NAN_F : lg[i] - lse;
        }
    }
}

template <typename T, int BITS>
static cudaError_t select_logits_t(const void *x, const void *w, float eps, const int32_t *row_idx, int n, int rows, int H, const void *wq,
                                   const void *scales, const void *biases, int V, const int32_t *ids, int m, float *logits, float *logprobs,
                                   int dtype, cudaStream_t st) {
    bool vec = false;
    const int tpr = rms_norm_path(H, dtype, x, w, x, &vec);
    const T *xp = static_cast<const T *>(x), *wp = static_cast<const T *>(w);
    const T *sp = static_cast<const T *>(scales), *bp = static_cast<const T *>(biases);
    const uint32_t *qp = static_cast<const uint32_t *>(wq);
    const size_t smem = static_cast<size_t>(H) * sizeof(float);
    constexpr int VV = 16 / sizeof(T);
    auto go = [&](auto kernel, int threads) {
        static bool configured = false;  // one flag per kernel instantiation (the lambda is instantiated per type)
        if (!configured) {
            const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TL_EMBED_MAX_HIDDEN * sizeof(float));
            if (e != cudaSuccess) return e;
            configured = true;
        }
        return launch_chained(kernel, dim3(n), dim3(threads), smem, st, xp, wp, eps, row_idx, rows, H, qp, sp, bp, V, ids, m, logits, logprobs);
    };
    if (tpr == 32) return vec ? go(select_logits_kernel<T, 32, VV, BITS>, 32) : go(select_logits_kernel<T, 32, 1, BITS>, 32);
    return vec ? go(select_logits_kernel<T, 256, VV, BITS>, 256) : go(select_logits_kernel<T, 256, 1, BITS>, 256);
}

int launch_select_logits(const void *x, const void *w, float eps, const int32_t *row_idx, int n, int rows, int H, const void *wq,
                         const void *scales, const void *biases, int V, int bits, const int32_t *ids, int m, float *logits, float *logprobs,
                         int dtype, cudaStream_t st) {
    if (n == 0) return TL_OK;
    cudaError_t e;
    if (dtype == TL_F16)
        e = bits == 8 ? select_logits_t<__half, 8>(x, w, eps, row_idx, n, rows, H, wq, scales, biases, V, ids, m, logits, logprobs, dtype, st)
                      : select_logits_t<__half, 4>(x, w, eps, row_idx, n, rows, H, wq, scales, biases, V, ids, m, logits, logprobs, dtype, st);
    else
        e = bits == 8 ? select_logits_t<__nv_bfloat16, 8>(x, w, eps, row_idx, n, rows, H, wq, scales, biases, V, ids, m, logits, logprobs, dtype, st)
                      : select_logits_t<__nv_bfloat16, 4>(x, w, eps, row_idx, n, rows, H, wq, scales, biases, V, ids, m, logits, logprobs, dtype, st);
    if (e != cudaSuccess) return fail(TL_ECUDA, "select_logits: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("select_logits");
    return TL_OK;
}

}  // namespace tl
