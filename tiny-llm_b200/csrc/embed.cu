// Sentence embeddings from packed hidden states (tl_embed_pool, DESIGN.md section 17): one CTA per segment applies the
// model's final RMSNorm to the rows it pools, pools them (the last row, or the fp32 mean of the normalised rows),
// truncates to the first d features and optionally divides by the L2 norm.
//
// A row is normalised in rms_norm_kernel's order (elementwise.cu), as moe_gather does (moe.cu): TPR threads per row
// (rms_norm_path: 32 up to 512 elements, else 256), thread `lane` owning the chunks of EPV consecutive elements at
// lane * EPV + n * TPR * EPV (16-byte vectors when rms_norm's VEC path applies, else single elements), its sum of
// squares reduced by the same warp and CTA steps.  So each normalised row is tl_rms_norm's bit for bit.  The pooled
// vector lives in shared memory, each element written only by the thread that owns it, so the mean is summed in row
// order per element and the L2 norm is one fixed-order CTA reduction.
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
        float ss = 0.f;
        for (int c = lane * EPV; c < H; c += TPR * EPV)
#pragma unroll
            for (int q = 0; q < EPV; ++q) {
                const float v = to_f(ld_cg(xr + c + q));
                ss += v * v;
            }
        ss = pool_sum<TPR>(ss, part);
        const float inv = rsqrtf(ss / static_cast<float>(H) + eps);
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

}  // namespace tl
