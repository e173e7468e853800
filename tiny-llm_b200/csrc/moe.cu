// Qwen3-MoE sparse block (reference: moe.py:36-89, qwen3_week3.py:253-272) as capture-safe launches: every output is
// sized by T * k rows and E experts, nothing is synchronised and no count is read back to the host.
//
//   tl_moe_topk     logits [T, E] -> probs = bf16(softmax_fp32), ids / scores of the k largest probs (ties: lower id),
//                   scores optionally renormalised: bf16(score / bf16(sum_fp32 scores)); one warp per token row
//   tl_moe_group    ids [R] -> offsets [E + 1], perm [R] (sorted position -> row, stable within an expert) and the
//                   grouped GEMM's tile table; one CTA, integer only
//   tl_moe_gather   xs[j] = x[perm[j] / rows_per_source], optionally RMSNorm-ed (the rounding point of rms_norm)
//   tl_moe_combine  r = bf16(sum_fp32 over slots j of bf16(y_j * score_j)), x' = bf16(x + r), optionally the next RMSNorm
//   grouped W4A16   the swap-AB wgmma kernel of w4a16_skinny.cu indexed per expert; here its scalar control kernel
#include "common.cuh"
#include "kernels.h"

namespace tl {

__device__ __forceinline__ int ceil_div_dev(int a, int b) { return (a + b - 1) / b; }

// ------------------------------------------------------------------ top-k --
constexpr int MOE_PER_LANE = TL_MOE_MAX_EXPERTS / 32;

template <typename T>
__global__ void __launch_bounds__(256) moe_topk_kernel(const T *__restrict__ logits, T *__restrict__ probs, int32_t *__restrict__ ids,
                                                       T *__restrict__ scores, int rows, int E, int k, int norm) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
    griddep_launch();
    griddep_wait();
    if (row >= rows) return;
    const T *lr = logits + static_cast<size_t>(row) * E;
    float v[MOE_PER_LANE];
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < MOE_PER_LANE; ++i) {
        const int e = lane + 32 * i;
        v[i] = e < E ? to_f(ld_cg(lr + e)) : -INFINITY;
        m = fmaxf(m, v[i]);
    }
    m = warp_max(m);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MOE_PER_LANE; ++i) {
        v[i] = lane + 32 * i < E ? expf(v[i] - m) : 0.f;
        s += v[i];
    }
    s = warp_sum(s);
    // probabilities in the output dtype: selection compares these rounded values, as the reference's argpartition does
#pragma unroll
    for (int i = 0; i < MOE_PER_LANE; ++i) {
        const int e = lane + 32 * i;
        if (e < E) {
            const T p = from_f<T>(v[i] / s);
            probs[static_cast<size_t>(row) * E + e] = p;
            // A NaN softmax (a NaN or +inf logit, or every logit -inf) fails every comparison below; as -0.5 it ranks
            // under every probability and over the picked and padding entries (-1), so the row still names k experts.
            v[i] = isnan(to_f(p)) ? -0.5f : to_f(p);
        } else {
            v[i] = -1.f;
        }
    }
    float picked[TL_MOE_MAX_TOPK];
    int picked_id[TL_MOE_MAX_TOPK];
    float total = 0.f;
    for (int j = 0; j < k; ++j) {
        // largest value, lowest expert id among equals
        float best = -2.f;
        int best_e = 0x7fffffff;
#pragma unroll
        for (int i = 0; i < MOE_PER_LANE; ++i) {
            const int e = lane + 32 * i;
            if (v[i] > best || (v[i] == best && e < best_e)) best = v[i], best_e = e;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oe = __shfl_xor_sync(0xffffffffu, best_e, o);
            if (ob > best || (ob == best && oe < best_e)) best = ob, best_e = oe;
        }
#pragma unroll
        for (int i = 0; i < MOE_PER_LANE; ++i)
            if (lane + 32 * i == best_e) v[i] = -1.f;
        picked[j] = best >= 0.f ? best : __int_as_float(0x7fffffff);  // a NaN row's scores stay NaN
        picked_id[j] = best_e;
        total += best;  // slot order
    }
    if (lane != 0) return;
    const float den = to_f(from_f<T>(total));
    for (int j = 0; j < k; ++j) {
        ids[static_cast<size_t>(row) * k + j] = picked_id[j];
        scores[static_cast<size_t>(row) * k + j] = from_f<T>(norm ? picked[j] / den : picked[j]);
    }
}

int launch_moe_topk(const void *logits, void *probs, int32_t *ids, void *scores, int rows, int E, int k, int norm, int dtype, cudaStream_t st) {
    if (rows == 0) return TL_OK;
    const dim3 grid(ceil_div(rows, 8));
    cudaError_t e;
    if (dtype == TL_BF16)
        e = launch_chained(moe_topk_kernel<__nv_bfloat16>, grid, dim3(256), 0, st, static_cast<const __nv_bfloat16 *>(logits),
                           static_cast<__nv_bfloat16 *>(probs), ids, static_cast<__nv_bfloat16 *>(scores), rows, E, k, norm);
    else if (dtype == TL_F16)
        e = launch_chained(moe_topk_kernel<__half>, grid, dim3(256), 0, st, static_cast<const __half *>(logits), static_cast<__half *>(probs), ids,
                           static_cast<__half *>(scores), rows, E, k, norm);
    else
        e = launch_chained(moe_topk_kernel<float>, grid, dim3(256), 0, st, static_cast<const float *>(logits), static_cast<float *>(probs), ids,
                           static_cast<float *>(scores), rows, E, k, norm);
    if (e != cudaSuccess) return fail(TL_ECUDA, "moe_topk: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("moe_topk");
    return TL_OK;
}

// ------------------------------------------------------------------ group --
// One CTA of MOE_GROUP_WARPS warps; warp w owns the rows [w S, (w + 1) S).  Pass A counts each warp's rows per expert,
// a column scan over the warps turns the counts into each warp's first sorted position per expert, pass B places the
// rows in order.  Within a warp, rows of one expert are ranked with __match_any_sync, so perm is stable.
constexpr int MOE_GROUP_WARPS = 32;

__global__ void __launch_bounds__(MOE_GROUP_WARPS * 32) moe_group_kernel(const int32_t *__restrict__ ids, int R, int E, int nt, int32_t *offsets,
                                                                         int32_t *perm, int32_t *tiles) {
    __shared__ int base[MOE_GROUP_WARPS][TL_MOE_MAX_EXPERTS];
    __shared__ int start[TL_MOE_MAX_EXPERTS + 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    griddep_launch();
    for (int i = threadIdx.x; i < MOE_GROUP_WARPS * TL_MOE_MAX_EXPERTS; i += blockDim.x) (&base[0][0])[i] = 0;
    griddep_wait();
    __syncthreads();
    const int per = ceil_div_dev(R, MOE_GROUP_WARPS);
    const int r0 = min(warp * per, R), r1 = min(r0 + per, R);
    // ids outside [0, E) are a caller error; they are clamped so that every write stays in bounds
    auto expert_of = [&](int r) { return min(max(ld_cg(ids + r), 0), E - 1); };
    for (int c = r0; c < r1; c += 32) {
        const int r = c + lane;
        const bool live = r < r1;
        const int e = live ? expert_of(r) : -1 - lane;
        const unsigned same = __match_any_sync(0xffffffffu, e);
        if (live && (same & lt) == 0) base[warp][e] += __popc(same);
        __syncwarp();
    }
    __syncthreads();
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
        int run = 0;
        for (int w = 0; w < MOE_GROUP_WARPS; ++w) {
            const int n = base[w][e];
            base[w][e] = run;
            run += n;
        }
        start[e] = run;  // count of expert e, for now
    }
    __syncthreads();
    if (warp == 0) {
        // exclusive scan of the counts (and of the tiles per expert) over E <= 256 experts: 8 consecutive per lane
        int cnt[MOE_PER_LANE], sum = 0, tsum = 0;
#pragma unroll
        for (int i = 0; i < MOE_PER_LANE; ++i) {
            const int e = lane * MOE_PER_LANE + i;
            cnt[i] = e < E ? start[e] : 0;
            sum += cnt[i];
            tsum += nt > 0 ? ceil_div_dev(cnt[i], nt) : 0;
        }
        int incl = sum, tincl = tsum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int a = __shfl_up_sync(0xffffffffu, incl, o), b = __shfl_up_sync(0xffffffffu, tincl, o);
            if (lane >= o) incl += a, tincl += b;
        }
        int run = incl - sum, trun = tincl - tsum;
#pragma unroll
        for (int i = 0; i < MOE_PER_LANE; ++i) {
            const int e = lane * MOE_PER_LANE + i;
            if (e < E) {
                start[e] = run;
                offsets[e] = run;
                if (nt > 0)
                    for (int t = 0; t < ceil_div_dev(cnt[i], nt); ++t) {
                        tiles[1 + 2 * (trun + t)] = e;
                        tiles[2 + 2 * (trun + t)] = run + t * nt;
                    }
            }
            run += cnt[i];
            trun += nt > 0 ? ceil_div_dev(cnt[i], nt) : 0;
        }
        if (lane == 31) {
            offsets[E] = run;
            if (nt > 0) tiles[0] = trun;
        }
    }
    __syncthreads();
    for (int c = r0; c < r1; c += 32) {
        const int r = c + lane;
        const bool live = r < r1;
        const int e = live ? expert_of(r) : -1 - lane;
        const unsigned same = __match_any_sync(0xffffffffu, e);
        if (live) perm[start[e] + base[warp][e] + __popc(same & lt)] = r;
        __syncwarp();
        if (live && (same & lt) == 0) base[warp][e] += __popc(same);
        __syncwarp();
    }
}

int launch_moe_group(const int32_t *ids, int R, int E, int nt, int32_t *offsets, int32_t *perm, int32_t *tiles, cudaStream_t st) {
    cudaError_t e = launch_chained(moe_group_kernel, dim3(1), dim3(MOE_GROUP_WARPS * 32), 0, st, ids, R, E, nt, offsets, perm, tiles);
    if (e != cudaSuccess) return fail(TL_ECUDA, "moe_group: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("moe_group");
    return TL_OK;
}

// ------------------------------------------------- rows with an RMSNorm --
// The gather and the combine visit a row's elements in rms_norm_kernel's order (elementwise.cu): TPR threads per row
// (rms_norm_path: 32 up to 512 elements, else 256), thread `lane` taking chunks of EPV consecutive elements (16-byte
// vectors when rms_norm's VEC path applies, else single elements) at lane * EPV + n * TPR * EPV, and its sum of squares
// reduced by the same warp and CTA steps.  So the RMSNorm they apply is bit for bit tl_rms_norm's.
template <int TPR>
__device__ __forceinline__ float moe_row_sum(float ss, float *part) {
    ss = warp_sum(ss);
    if constexpr (TPR > 32) {
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = ss;
        __syncthreads();
        ss = warp_sum((threadIdx.x & 31) < TPR / 32 ? part[threadIdx.x & 31] : 0.f);
    }
    return ss;
}

template <typename T, int TPR, int EPV>
__global__ void __launch_bounds__(256) moe_gather_kernel(const T *__restrict__ x, const int32_t *__restrict__ perm, const T *__restrict__ norm_w,
                                                         float eps, T *__restrict__ xs, int R, int rows_per_source, int H) {
    __shared__ float part[8];
    griddep_launch();
    griddep_wait();
    const int lane = threadIdx.x % TPR;
    const int j = blockIdx.x * (256 / TPR) + threadIdx.x / TPR;
    const bool live = j < R;
    const T *src = x + static_cast<size_t>(live ? ld_cg(perm + j) / rows_per_source : 0) * H;
    T *dst = xs + static_cast<size_t>(live ? j : 0) * H;
    if (norm_w == nullptr) {
        if (live)
            for (int i = lane; i < H; i += TPR) dst[i] = ld_cg(src + i);
        return;
    }
    float ss = 0.f;
    if (live)
        for (int c = lane * EPV; c < H; c += TPR * EPV)
#pragma unroll
            for (int q = 0; q < EPV; ++q) {
                const float v = to_f(ld_cg(src + c + q));
                ss += v * v;
            }
    ss = moe_row_sum<TPR>(ss, part);
    if (!live) return;
    const float inv = rsqrtf(ss / static_cast<float>(H) + eps);
    for (int c = lane * EPV; c < H; c += TPR * EPV)
#pragma unroll
        for (int q = 0; q < EPV; ++q) dst[c + q] = from_f<T>(to_f(ld_cg(src + c + q)) * inv * to_f(norm_w[c + q]));
}

// The layout (threads per row, elements per chunk) of an RMSNorm over rows of H elements at x -> out with weight w.
template <typename T>
static void moe_row_layout(int H, int dtype, const void *x, const void *w, const void *out, int *tpr, int *epv) {
    bool vec = false;
    *tpr = rms_norm_path(H, dtype, x, w != nullptr ? w : x, out, &vec);
    *epv = vec ? 16 / static_cast<int>(sizeof(T)) : 1;
}

template <typename T>
static cudaError_t moe_gather_t(const void *x, const int32_t *perm, const void *norm_w, float eps, void *xs, int R, int rows_per_source, int H,
                                int dtype, cudaStream_t st) {
    int tpr, epv;
    moe_row_layout<T>(H, dtype, x, norm_w, xs, &tpr, &epv);
    const dim3 grid(ceil_div(R, 256 / tpr));
    const T *xp = static_cast<const T *>(x), *wp = static_cast<const T *>(norm_w);
    T *op = static_cast<T *>(xs);
    constexpr int V = 16 / sizeof(T);
    if (tpr == 32)
        return epv == 1 ? launch_chained(moe_gather_kernel<T, 32, 1>, grid, dim3(256), 0, st, xp, perm, wp, eps, op, R, rows_per_source, H)
                        : launch_chained(moe_gather_kernel<T, 32, V>, grid, dim3(256), 0, st, xp, perm, wp, eps, op, R, rows_per_source, H);
    return epv == 1 ? launch_chained(moe_gather_kernel<T, 256, 1>, grid, dim3(256), 0, st, xp, perm, wp, eps, op, R, rows_per_source, H)
                    : launch_chained(moe_gather_kernel<T, 256, V>, grid, dim3(256), 0, st, xp, perm, wp, eps, op, R, rows_per_source, H);
}

int launch_moe_gather(const void *x, const int32_t *perm, const void *norm_w, float eps, void *xs, int R, int rows_per_source, int H, int dtype,
                      cudaStream_t st) {
    if (R == 0) return TL_OK;
    cudaError_t e;
    if (dtype == TL_BF16)
        e = moe_gather_t<__nv_bfloat16>(x, perm, norm_w, eps, xs, R, rows_per_source, H, dtype, st);
    else if (dtype == TL_F16)
        e = moe_gather_t<__half>(x, perm, norm_w, eps, xs, R, rows_per_source, H, dtype, st);
    else
        e = moe_gather_t<float>(x, perm, norm_w, eps, xs, R, rows_per_source, H, dtype, st);
    if (e != cudaSuccess) return fail(TL_ECUDA, "moe_gather: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("moe_gather");
    return TL_OK;
}

// ---------------------------------------------------------------- combine --
template <typename T, int TPR, int EPV>
__global__ void __launch_bounds__(256) moe_combine_kernel(const T *__restrict__ y, const T *__restrict__ scores, const T *__restrict__ residual,
                                                          const T *__restrict__ norm_w, float eps, T *__restrict__ out, T *__restrict__ normed, int T_,
                                                          int k, int H) {
    __shared__ float part[8];
    griddep_launch();
    griddep_wait();
    const int lane = threadIdx.x % TPR;
    const int t = blockIdx.x * (256 / TPR) + threadIdx.x / TPR;
    const bool live = t < T_;
    float ss = 0.f;
    T *orow = out + static_cast<size_t>(live ? t : 0) * H;
    if (live) {
        float sc[TL_MOE_MAX_TOPK];
#pragma unroll
        for (int j = 0; j < TL_MOE_MAX_TOPK; ++j) sc[j] = j < k ? to_f(ld_cg(scores + static_cast<size_t>(t) * k + j)) : 0.f;
        const T *yr = y + static_cast<size_t>(t) * k * H;
        for (int c = lane * EPV; c < H; c += TPR * EPV)
            for (int q = 0; q < EPV; ++q) {
                const int i = c + q;
                float acc = 0.f;
#pragma unroll
                for (int j = 0; j < TL_MOE_MAX_TOPK; ++j)  // slot order; a fixed trip count keeps sc[] in registers
                    // __fmul_rn: the product is rounded before the sum for fp32 too (not contracted into an fma)
                    if (j < k) acc += to_f(from_f<T>(__fmul_rn(to_f(ld_cg(yr + static_cast<size_t>(j) * H + i)), sc[j])));
                T v = from_f<T>(acc);
                if (residual != nullptr) v = from_f<T>(to_f(ld_cg(residual + static_cast<size_t>(t) * H + i)) + to_f(v));
                orow[i] = v;
                const float f = to_f(v);
                ss += f * f;
            }
    }
    if (normed == nullptr) return;
    ss = moe_row_sum<TPR>(ss, part);
    if (!live) return;
    const float inv = rsqrtf(ss / static_cast<float>(H) + eps);
    T *nrow = normed + static_cast<size_t>(t) * H;
    for (int c = lane * EPV; c < H; c += TPR * EPV)  // each thread reads back only the elements it wrote itself
#pragma unroll
        for (int q = 0; q < EPV; ++q) nrow[c + q] = from_f<T>(to_f(orow[c + q]) * inv * to_f(norm_w[c + q]));
}

template <typename T>
static cudaError_t moe_combine_t(const void *y, const void *scores, const void *residual, const void *norm_w, float eps, void *out, void *normed,
                                 int T_, int k, int H, int dtype, cudaStream_t st) {
    int tpr, epv;
    moe_row_layout<T>(H, dtype, out, norm_w, normed != nullptr ? normed : out, &tpr, &epv);
    const dim3 grid(ceil_div(T_, 256 / tpr));
    auto args = [&](auto kernel) {
        return launch_chained(kernel, grid, dim3(256), 0, st, static_cast<const T *>(y), static_cast<const T *>(scores), static_cast<const T *>(residual),
                              static_cast<const T *>(norm_w), eps, static_cast<T *>(out), static_cast<T *>(normed), T_, k, H);
    };
    constexpr int V = 16 / sizeof(T);
    if (tpr == 32) return epv == 1 ? args(moe_combine_kernel<T, 32, 1>) : args(moe_combine_kernel<T, 32, V>);
    return epv == 1 ? args(moe_combine_kernel<T, 256, 1>) : args(moe_combine_kernel<T, 256, V>);
}

int launch_moe_combine(const void *y, const void *scores, const void *residual, const void *norm_w, float eps, void *out, void *normed, int T,
                       int k, int H, int dtype, cudaStream_t st) {
    if (T == 0) return TL_OK;
    cudaError_t e;
    if (dtype == TL_BF16)
        e = moe_combine_t<__nv_bfloat16>(y, scores, residual, norm_w, eps, out, normed, T, k, H, dtype, st);
    else if (dtype == TL_F16)
        e = moe_combine_t<__half>(y, scores, residual, norm_w, eps, out, normed, T, k, H, dtype, st);
    else
        e = moe_combine_t<float>(y, scores, residual, norm_w, eps, out, normed, T, k, H, dtype, st);
    if (e != cudaSuccess) return fail(TL_ECUDA, "moe_combine: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("moe_combine");
    return TL_OK;
}

// ------------------------------------------------- grouped control kernel --
// One thread per (sorted row, output): the arithmetic of w4a16_vanilla_kernel on the rows of the row's expert.  The
// expert is found by a binary search of offsets.  EPI_SWIGLU_PAIRS: output column c reads the interleaved gate row
// 16 (c / 8) + c % 8 and its up row 8 further.
template <typename T>
__device__ __forceinline__ float moe_dot(const T *scales, const T *biases, const uint32_t *b, const T *arow, size_t wrow, int N) {
    const int G = N / 128;
    const uint32_t *brow = b + wrow * (N / 8);
    float sum = 0.f;
    for (int grp = 0; grp < G; ++grp) {
        const float s = to_f(scales[wrow * G + grp]), c = to_f(biases[wrow * G + grp]);
        for (int w = 0; w < 16; ++w) {
            const uint32_t packed = brow[grp * 16 + w];
            const T *av = arow + grp * 128 + w * 8;
#pragma unroll
            for (int q = 0; q < 8; ++q) sum += (static_cast<float>((packed >> (4 * q)) & 0xFu) * s + c) * to_f(av[q]);
        }
    }
    return sum;
}

template <typename T>
__global__ void moe_grouped_vanilla_kernel(const T *__restrict__ scales, const T *__restrict__ biases, const T *__restrict__ a,
                                           const uint32_t *__restrict__ b, T *__restrict__ out, const int32_t *offsets,
                                           const int32_t *out_index, int E, int N, int K, int epilogue) {
    griddep_launch();
    griddep_wait();
    const int j = blockIdx.x;  // rows on grid.x: up to 2^31 - 1 of them
    const int width = epilogue == TL_EPI_SWIGLU_PAIRS ? K / 2 : K;
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= width) return;
    int lo = 0, hi = E - 1;  // last expert whose segment starts at or before j
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (ld_cg(offsets + mid) <= j) lo = mid;
        else hi = mid - 1;
    }
    const T *arow = a + static_cast<size_t>(j) * N;
    const size_t e0 = static_cast<size_t>(lo) * K;
    const int orow = out_index != nullptr ? ld_cg(out_index + j) : j;
    T v;
    if (epilogue == TL_EPI_SWIGLU_PAIRS) {
        const int n_gate = (c >> 3) * 16 + (c & 7);
        const float gate = to_f(from_f<T>(moe_dot(scales, biases, b, arow, e0 + n_gate, N)));
        const float up = to_f(from_f<T>(moe_dot(scales, biases, b, arow, e0 + n_gate + 8, N)));
        v = from_f<T>((gate / (1.0f + expf(-gate))) * up);
    } else {
        v = from_f<T>(moe_dot(scales, biases, b, arow, e0 + c, N));
    }
    out[static_cast<size_t>(orow) * width + c] = v;
}

int launch_moe_grouped_vanilla(const void *scales, const void *biases, const void *a, const void *b, void *out, const int32_t *offsets,
                               const int32_t *out_index, int R, int E, int N, int K, int epilogue, int dtype, cudaStream_t st) {
    if (R == 0 || K == 0) return TL_OK;
    const int width = epilogue == TL_EPI_SWIGLU_PAIRS ? K / 2 : K;
    const dim3 grid(R, ceil_div(width, 128));
    cudaError_t e;
    if (dtype == TL_BF16)
        e = launch_chained(moe_grouped_vanilla_kernel<__nv_bfloat16>, grid, dim3(128), 0, st, static_cast<const __nv_bfloat16 *>(scales),
                           static_cast<const __nv_bfloat16 *>(biases), static_cast<const __nv_bfloat16 *>(a), static_cast<const uint32_t *>(b),
                           static_cast<__nv_bfloat16 *>(out), offsets, out_index, E, N, K, epilogue);
    else if (dtype == TL_F16)
        e = launch_chained(moe_grouped_vanilla_kernel<__half>, grid, dim3(128), 0, st, static_cast<const __half *>(scales),
                           static_cast<const __half *>(biases), static_cast<const __half *>(a), static_cast<const uint32_t *>(b),
                           static_cast<__half *>(out), offsets, out_index, E, N, K, epilogue);
    else
        return fail(TL_EDTYPE, "moe_grouped_matmul: scales must be float16 or bfloat16");
    if (e != cudaSuccess) return fail(TL_ECUDA, "moe_grouped_vanilla: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("moe_grouped_vanilla");
    return TL_OK;
}

}  // namespace tl
