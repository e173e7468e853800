// Memory-bound model kernels: RMSNorm, RoPE, SwiGLU, residual add, W4 embedding
// gather, paged KV writes, greedy argmax.  All are HBM/L2-bound byte movers:
// 128-bit coalesced accesses when alignment allows, fp32 math, one rounding.
//
// Arithmetic follows the reference Metal kernels (paths relative to
// src/extensions_ref/src): week2_kernels.metal:6-117,
// quantized_matmul.metal:58-89, paged_attention.metal:82-106.
#include <float.h>
#include <limits.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace tl {

template <typename T>
struct Vec {
    static constexpr int N = 16 / sizeof(T);  // elements per 128-bit access
};

template <typename T, bool CG = false>
__device__ __forceinline__ void load16(const T *p, float (&v)[Vec<T>::N]) {
    uint4 raw;
    if constexpr (CG)
        raw = ld_cg(reinterpret_cast<const uint4 *>(p));  // written by the previous kernel of a dependent-launch chain
    else
        raw = *reinterpret_cast<const uint4 *>(p);
    if constexpr (sizeof(T) == 4) {
        v[0] = __uint_as_float(raw.x), v[1] = __uint_as_float(raw.y);
        v[2] = __uint_as_float(raw.z), v[3] = __uint_as_float(raw.w);
    } else {
        float2 a = unpack2<T>(raw.x), b = unpack2<T>(raw.y), c = unpack2<T>(raw.z), d = unpack2<T>(raw.w);
        v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y, v[4] = c.x, v[5] = c.y, v[6] = d.x, v[7] = d.y;
    }
}

template <typename T>
__device__ __forceinline__ void store16(T *p, const float (&v)[Vec<T>::N]) {
    uint4 raw;
    if constexpr (sizeof(T) == 4) {
        raw.x = __float_as_uint(v[0]), raw.y = __float_as_uint(v[1]);
        raw.z = __float_as_uint(v[2]), raw.w = __float_as_uint(v[3]);
    } else {
        raw.x = pack2<T>(v[0], v[1]), raw.y = pack2<T>(v[2], v[3]);
        raw.z = pack2<T>(v[4], v[5]), raw.w = pack2<T>(v[6], v[7]);
    }
    *reinterpret_cast<uint4 *>(p) = raw;
}

// ---------------------------------------------------------------- RMSNorm --
// TPR threads cooperate on one row (32: one warp per row for per-head norms of
// width 128; 256: one CTA per row for hidden-size rows).
template <typename T, int TPR, bool VEC>
__global__ void __launch_bounds__(256) rms_norm_kernel(const T *x, const T *__restrict__ w, T *out, int rows, int dim, float eps) {
    griddep_launch();
    griddep_wait();  // x is the previous kernel's output (common.cuh: programmatic dependent launch)
    constexpr int ROWS = 256 / TPR;
    constexpr int EPV = Vec<T>::N;
    const int sub = threadIdx.x / TPR;
    const int lane = threadIdx.x % TPR;
    const int row = blockIdx.x * ROWS + sub;
    const bool live = row < rows;
    const T *xr = x + static_cast<size_t>(live ? row : 0) * dim;
    T *outr = out + static_cast<size_t>(live ? row : 0) * dim;

    float ss = 0.f;
    constexpr int KEEP = 2;  // chunks per thread that stay in registers between the two passes (dim <= 2 * TPR * EPV: one L2 trip)
    float keep[KEEP][EPV];
    if (live) {
        if constexpr (VEC) {
            int it = 0;
            for (int i = lane * EPV; i < dim; i += TPR * EPV, ++it) {
                float v[EPV];
                load16<T, true>(xr + i, v);
#pragma unroll
                for (int j = 0; j < EPV; ++j) ss += v[j] * v[j];
#pragma unroll
                for (int k = 0; k < KEEP; ++k)
                    if (it == k) {
#pragma unroll
                        for (int j = 0; j < EPV; ++j) keep[k][j] = v[j];
                    }
            }
        } else {
            for (int i = lane; i < dim; i += TPR) {
                float v = to_f(ld_cg(xr + i));
                ss += v * v;
            }
        }
    }
    ss = warp_sum(ss);
    if constexpr (TPR > 32) {
        __shared__ float part[TPR / 32];
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = ss;
        __syncthreads();
        float t = (threadIdx.x & 31) < TPR / 32 ? part[threadIdx.x & 31] : 0.f;
        ss = warp_sum(t);
    }
    if (!live) return;
    const float inv = rsqrtf(ss / static_cast<float>(dim) + eps);
    if constexpr (VEC) {
        int it = 0;
        for (int i = lane * EPV; i < dim; i += TPR * EPV, ++it) {
            float v[EPV], g[EPV];
            if (it >= KEEP) load16<T, true>(xr + i, v);
#pragma unroll
            for (int k = 0; k < KEEP; ++k)
                if (it == k) {
#pragma unroll
                    for (int j = 0; j < EPV; ++j) v[j] = keep[k][j];
                }
            load16<T>(w + i, g);
#pragma unroll
            for (int j = 0; j < EPV; ++j) v[j] = v[j] * inv * g[j];
            store16<T>(outr + i, v);
        }
    } else {
        for (int i = lane; i < dim; i += TPR) outr[i] = from_f<T>(to_f(ld_cg(xr + i)) * inv * to_f(w[i]));
    }
}

// Threads per row (32 up to 512 elements, else 256) and whether every access can be a 16-byte vector.
int rms_norm_path(int dim, int dtype, const void *x, const void *w, const void *out, bool *vec) {
    const int epv = 16 / (dtype == TL_F32 ? 4 : 2);
    *vec = dim % epv == 0 && aligned16(x) && aligned16(w) && aligned16(out);
    return dim <= 512 ? 32 : 256;
}

template <typename T>
static int rms_norm_t(const void *x, const void *w, void *out, int rows, int dim, float eps, int dtype, cudaStream_t st) {
    bool vec;
    const int tpr = rms_norm_path(dim, dtype, x, w, out, &vec);
    const T *xp = static_cast<const T *>(x);
    const T *wp = static_cast<const T *>(w);
    T *op = static_cast<T *>(out);
    if (tpr == 32) {
        dim3 grid(ceil_div(rows, 8));
        if (vec)
            launch_chained(rms_norm_kernel<T, 32, true>, grid, dim3(256), 0, st, xp, wp, op, rows, dim, eps);
        else
            launch_chained(rms_norm_kernel<T, 32, false>, grid, dim3(256), 0, st, xp, wp, op, rows, dim, eps);
    } else {
        dim3 grid(rows);
        if (vec)
            launch_chained(rms_norm_kernel<T, 256, true>, grid, dim3(256), 0, st, xp, wp, op, rows, dim, eps);
        else
            launch_chained(rms_norm_kernel<T, 256, false>, grid, dim3(256), 0, st, xp, wp, op, rows, dim, eps);
    }
    TL_LAUNCH_CHECK("rms_norm");
    return TL_OK;
}

int launch_rms_norm(const void *x, const void *w, void *out, int rows, int dim, float eps, int dtype,
                    cudaStream_t st) {
    if (rows == 0) return TL_OK;
    switch (dtype) {
        case TL_F32: return rms_norm_t<float>(x, w, out, rows, dim, eps, dtype, st);
        case TL_F16: return rms_norm_t<__half>(x, w, out, rows, dim, eps, dtype, st);
        case TL_BF16: return rms_norm_t<__nv_bfloat16>(x, w, out, rows, dim, eps, dtype, st);
    }
    return fail(TL_EDTYPE, "rms_norm: expected float32, float16, or bfloat16");
}

// ------------------------------------------------------------------- RoPE --
// One thread per (b, l, h, item): item < dims/2 rotates one pair, the remaining
// items copy the un-rotated tail [dims, D).  Consecutive threads touch
// consecutive elements, so each warp access is one contiguous segment.
template <typename T>
__global__ void rope_kernel(const T *__restrict__ x, const int32_t *__restrict__ offsets, T *__restrict__ out, int B,
                            int L, int H, int D, int dims, float base, int traditional) {
    const int half_dim = dims / 2;
    const int items = half_dim + (D - dims);
    const long long total = static_cast<long long>(B) * L * H * items;
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int item = static_cast<int>(idx % items);
    const int h = static_cast<int>((idx / items) % H);
    const int l = static_cast<int>((idx / (static_cast<long long>(items) * H)) % L);
    const int b = static_cast<int>(idx / (static_cast<long long>(items) * H * L));
    const size_t head_base = ((static_cast<size_t>(b) * L + l) * H + h) * D;
    if (item >= half_dim) {
        const int d = dims + item - half_dim;
        out[head_base + d] = x[head_base + d];
        return;
    }
    // angle = position * base^(-pair/half) (week2_kernels.metal:86-92).  The frequency is
    // formed in double so that long contexts (position ~32K) do not inherit the ~1e-7
    // relative error of an fp32 exp2/pow; the product and sincosf stay fp32.
    const double inv_freq = exp2(-static_cast<double>(item) / static_cast<double>(half_dim) * log2(static_cast<double>(base)));
    const float angle = static_cast<float>(static_cast<double>(offsets[b] + l) * inv_freq);
    float s, c;
    sincosf(angle, &s, &c);
    const size_t re_i = traditional ? head_base + 2 * item : head_base + item;
    const size_t im_i = traditional ? re_i + 1 : re_i + half_dim;
    const float re = to_f(x[re_i]);
    const float im = to_f(x[im_i]);
    out[re_i] = from_f<T>(re * c - im * s);
    out[im_i] = from_f<T>(im * c + re * s);
}

// Prefill-sized inputs, full rotation (dims == D): one thread per (b, l, pair) forms the frequency
// (double exp2/log2) and sincosf ONCE and walks the H heads - the per-element kernel above recomputes
// them once per head.
template <typename T>
__global__ void rope_heads_kernel(const T *__restrict__ x, const int32_t *__restrict__ offsets, T *__restrict__ out, int B, int L,
                                  int H, int D, float base, int traditional) {
    const int half_dim = D / 2;
    const long long total = static_cast<long long>(B) * L * half_dim;
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int item = static_cast<int>(idx % half_dim);
    const int l = static_cast<int>((idx / half_dim) % L);
    const int b = static_cast<int>(idx / (static_cast<long long>(half_dim) * L));
    const double inv_freq = exp2(-static_cast<double>(item) / static_cast<double>(half_dim) * log2(static_cast<double>(base)));
    const float angle = static_cast<float>(static_cast<double>(offsets[b] + l) * inv_freq);
    float s, c;
    sincosf(angle, &s, &c);
    size_t re_i = (static_cast<size_t>(b) * L + l) * H * D + (traditional ? 2 * item : item);
    const int im_off = traditional ? 1 : half_dim;
    for (int h = 0; h < H; ++h, re_i += D) {
        const float re = to_f(x[re_i]), im = to_f(x[re_i + im_off]);
        out[re_i] = from_f<T>(re * c - im * s);
        out[re_i + im_off] = from_f<T>(im * c + re * s);
    }
}

// The per-(token, pair) kernel pays off once there are several heads to walk and enough tokens to fill the GPU.
bool rope_heads_path(int B, int L, int H, int D, int dims) { return dims == D && H > 1 && static_cast<long long>(B) * L >= 64; }

template <typename T>
static int rope_t(const void *x, const int32_t *off, void *out, int B, int L, int H, int D, int dims, float base,
                  int traditional, cudaStream_t st) {
    const long long total = static_cast<long long>(B) * L * H * (dims / 2 + D - dims);
    if (total == 0) return TL_OK;
    if (rope_heads_path(B, L, H, D, dims)) {
        const long long work = static_cast<long long>(B) * L * (D / 2);
        const long long nb = ceil_div_ll(work, 128);
        if (nb > INT_MAX) return fail(TL_EINVAL, "rope: tensor too large");
        rope_heads_kernel<T><<<static_cast<unsigned>(nb), 128, 0, st>>>(static_cast<const T *>(x), off, static_cast<T *>(out), B, L, H, D, base,
                                                                      traditional);
        TL_LAUNCH_CHECK("rope");
        return TL_OK;
    }
    const int threads = 256;
    const long long blocks = ceil_div_ll(total, threads);
    if (blocks > INT_MAX) return fail(TL_EINVAL, "rope: tensor too large");
    rope_kernel<T><<<static_cast<unsigned>(blocks), threads, 0, st>>>(static_cast<const T *>(x), off,
                                                                       static_cast<T *>(out), B, L, H, D, dims, base,
                                                                       traditional);
    TL_LAUNCH_CHECK("rope");
    return TL_OK;
}

int launch_rope(const void *x, const int32_t *off, void *out, int B, int L, int H, int D, int dims, float base,
                int traditional, int dtype, cudaStream_t st) {
    switch (dtype) {
        case TL_F32: return rope_t<float>(x, off, out, B, L, H, D, dims, base, traditional, st);
        case TL_F16: return rope_t<__half>(x, off, out, B, L, H, D, dims, base, traditional, st);
        case TL_BF16: return rope_t<__nv_bfloat16>(x, off, out, B, L, H, D, dims, base, traditional, st);
    }
    return fail(TL_EDTYPE, "rope: expected float32, float16, or bfloat16");
}

// ------------------------------------------------------ SwiGLU / residual --
enum class Ew { SWIGLU, ADD };

template <typename T, Ew OP, bool VEC>
__global__ void binary_kernel(const T *__restrict__ a, const T *__restrict__ b, T *__restrict__ out, long long n) {
    constexpr int EPV = Vec<T>::N;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    auto f = [](float p, float q) -> float {
        if constexpr (OP == Ew::SWIGLU)
            return (p / (1.0f + expf(-p))) * q;  // week2_kernels.metal:115-116
        else
            return p + q;
    };
    if constexpr (VEC) {
        const long long nv = n / EPV;
        for (; i < nv; i += stride) {
            float p[EPV], q[EPV];
            load16<T>(a + i * EPV, p);
            load16<T>(b + i * EPV, q);
#pragma unroll
            for (int j = 0; j < EPV; ++j) p[j] = f(p[j], q[j]);
            store16<T>(out + i * EPV, p);
        }
    } else {
        for (; i < n; i += stride) out[i] = from_f<T>(f(to_f(a[i]), to_f(b[i])));
    }
}

template <typename T, Ew OP>
static int binary_t(const void *a, const void *b, void *out, long long n, cudaStream_t st, const char *name) {
    if (n == 0) return TL_OK;
    constexpr int EPV = Vec<T>::N;
    const bool vec = n % EPV == 0 && aligned16(a) && aligned16(b) && aligned16(out);
    const long long work = vec ? n / EPV : n;
    const int threads = 256;
    const long long want = ceil_div_ll(work, threads);
    const unsigned blocks = static_cast<unsigned>(want < 148LL * 16 ? want : 148LL * 16);
    if (vec)
        binary_kernel<T, OP, true><<<blocks, threads, 0, st>>>(static_cast<const T *>(a), static_cast<const T *>(b),
                                                                static_cast<T *>(out), n);
    else
        binary_kernel<T, OP, false><<<blocks, threads, 0, st>>>(static_cast<const T *>(a), static_cast<const T *>(b),
                                                                 static_cast<T *>(out), n);
    TL_LAUNCH_CHECK(name);
    return TL_OK;
}

int launch_swiglu(const void *gate, const void *up, void *out, long long n, int dtype, cudaStream_t st) {
    switch (dtype) {
        case TL_F32: return binary_t<float, Ew::SWIGLU>(gate, up, out, n, st, "swiglu");
        case TL_F16: return binary_t<__half, Ew::SWIGLU>(gate, up, out, n, st, "swiglu");
        case TL_BF16: return binary_t<__nv_bfloat16, Ew::SWIGLU>(gate, up, out, n, st, "swiglu");
    }
    return fail(TL_EDTYPE, "swiglu: expected float32, float16, or bfloat16");
}

int launch_add(const void *a, const void *b, void *out, long long n, int dtype, cudaStream_t st) {
    switch (dtype) {
        case TL_F32: return binary_t<float, Ew::ADD>(a, b, out, n, st, "add");
        case TL_F16: return binary_t<__half, Ew::ADD>(a, b, out, n, st, "add");
        case TL_BF16: return binary_t<__nv_bfloat16, Ew::ADD>(a, b, out, n, st, "add");
    }
    return fail(TL_EDTYPE, "add: expected float32, float16, or bfloat16");
}

// ------------------------------------------------------ W4 embedding rows --
// One thread per packed word: 8 codes -> 8 outputs (one 128-bit store).
// value = float(code) * scale + bias, rounded once (quantized_matmul.metal:83-88).
template <typename T>
__global__ void quantized_embedding_kernel(const int32_t *__restrict__ indices, const T *__restrict__ scales,
                                           const T *__restrict__ biases, const uint32_t *__restrict__ weight,
                                           T *__restrict__ out, int tokens, int vocab, int dim, bool vec_store) {
    const int words = dim / 8;
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= static_cast<long long>(tokens) * words) return;
    const int token = static_cast<int>(idx / words);
    const int wcol = static_cast<int>(idx % words);
    const int row = indices[token];
    float v[8];
    if (row < 0 || row >= vocab) {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
    } else {
        const uint32_t packed = weight[static_cast<size_t>(row) * words + wcol];
        const size_t g = static_cast<size_t>(row) * (dim / 128) + wcol / 16;
        const float s = to_f(scales[g]);
        const float b = to_f(biases[g]);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = static_cast<float>((packed >> (4 * j)) & 0xFu) * s + b;
    }
    T *dst = out + static_cast<size_t>(token) * dim + wcol * 8;
    if (vec_store) {
        uint4 raw;
        raw.x = pack2<T>(v[0], v[1]), raw.y = pack2<T>(v[2], v[3]);
        raw.z = pack2<T>(v[4], v[5]), raw.w = pack2<T>(v[6], v[7]);
        *reinterpret_cast<uint4 *>(dst) = raw;
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[j] = from_f<T>(v[j]);
    }
}

template <typename T>
static int embedding_t(const void *indices, const void *scales, const void *biases, const void *weight, void *out,
                       int tokens, int vocab, int dim, cudaStream_t st) {
    const long long total = static_cast<long long>(tokens) * (dim / 8);
    if (total == 0) return TL_OK;
    const int threads = 256;
    quantized_embedding_kernel<T><<<static_cast<unsigned>(ceil_div_ll(total, threads)), threads, 0, st>>>(
        static_cast<const int32_t *>(indices), static_cast<const T *>(scales), static_cast<const T *>(biases),
        static_cast<const uint32_t *>(weight), static_cast<T *>(out), tokens, vocab, dim, aligned16(out));
    TL_LAUNCH_CHECK("quantized_embedding");
    return TL_OK;
}

int launch_quantized_embedding(const void *indices, const void *scales, const void *biases, const void *weight,
                               void *out, int tokens, int vocab, int dim, int dtype, cudaStream_t st) {
    switch (dtype) {
        case TL_F16: return embedding_t<__half>(indices, scales, biases, weight, out, tokens, vocab, dim, st);
        case TL_BF16: return embedding_t<__nv_bfloat16>(indices, scales, biases, weight, out, tokens, vocab, dim, st);
    }
    return fail(TL_EDTYPE, "quantized_embedding: scales and biases must have the same 16-bit dtype");
}

// ------------------------------------------------------ paged KV writes ----
// pages [P, H, page, D]; values [1, H, length, D]  (paged_attention.metal:82-106)
template <typename V>
__global__ void paged_cache_update_kernel(const V *__restrict__ values, V *__restrict__ pages, int heads, int length,
                                          int dvec, int page_size, int page_id, int start) {
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(heads) * length * dvec;
    if (idx >= total) return;
    const int d = static_cast<int>(idx % dvec);
    const int t = static_cast<int>((idx / dvec) % length);
    const int h = static_cast<int>(idx / (static_cast<long long>(dvec) * length));
    const size_t dst = ((static_cast<size_t>(page_id) * heads + h) * page_size + start + t) * dvec + d;
    pages[dst] = values[idx];
}

int launch_paged_cache_update(void *pages, const void *values, int heads, int page_size, int head_dim, int length,
                              int page_id, int start, int dtype, cudaStream_t st) {
    const int esize = dtype == TL_F32 ? 4 : 2;
    const long long elems = static_cast<long long>(heads) * length * head_dim;
    if (elems == 0) return TL_OK;
    const int threads = 256;
    const bool vec = (head_dim * esize) % 16 == 0 && aligned16(pages) && aligned16(values);
    if (vec) {
        const int dvec = head_dim * esize / 16;
        const long long total = static_cast<long long>(heads) * length * dvec;
        paged_cache_update_kernel<uint4><<<static_cast<unsigned>(ceil_div_ll(total, threads)), threads, 0, st>>>(
            static_cast<const uint4 *>(values), static_cast<uint4 *>(pages), heads, length, dvec, page_size, page_id,
            start);
    } else if (esize == 4) {
        paged_cache_update_kernel<uint32_t><<<static_cast<unsigned>(ceil_div_ll(elems, threads)), threads, 0, st>>>(
            static_cast<const uint32_t *>(values), static_cast<uint32_t *>(pages), heads, length, head_dim, page_size,
            page_id, start);
    } else {
        paged_cache_update_kernel<uint16_t><<<static_cast<unsigned>(ceil_div_ll(elems, threads)), threads, 0, st>>>(
            static_cast<const uint16_t *>(values), static_cast<uint16_t *>(pages), heads, length, head_dim, page_size,
            page_id, start);
    }
    TL_LAUNCH_CHECK("paged_cache_update");
    return TL_OK;
}

// Chunk append: up to TL_PAGE_SPANS (page, first row, rows, first source token) spans of ONE
// request written in one launch, K and V together, straight from strided [1, H, L, D] sources
// (the per-page paged_cache_update sequence of paged_kv_cache.py:271-312 cost 64 launches plus
// 64 slice copies per layer for a 4096-token chunk).
template <typename V>
__global__ void paged_cache_append_chunk_kernel(V *__restrict__ key_pages, V *__restrict__ value_pages, const V *__restrict__ keys,
                                                const V *__restrict__ values, const tl_page_span_list spans, int heads, int page_size,
                                                int dvec, long long src_head_stride, long long src_token_stride) {
    const int span = blockIdx.y;
    const int pid = spans.page_id[span], start = spans.start[span], count = spans.count[span], src0 = spans.src[span];
    const long long total = static_cast<long long>(heads) * count * dvec;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int d = static_cast<int>(idx % dvec);
        const int t = static_cast<int>((idx / dvec) % count);
        const int h = static_cast<int>(idx / (static_cast<long long>(dvec) * count));
        const size_t dst = ((static_cast<size_t>(pid) * heads + h) * page_size + start + t) * dvec + d;
        const size_t src = static_cast<size_t>(h) * src_head_stride + static_cast<size_t>(src0 + t) * src_token_stride + d;
        key_pages[dst] = keys[src];
        value_pages[dst] = values[src];
    }
}

int launch_paged_cache_append_chunk(void *key_pages, void *value_pages, const void *keys, const void *values,
                                    const tl_page_span_list &spans, int heads, int page_size, int head_dim, long long src_head_stride,
                                    long long src_token_stride, int dtype, cudaStream_t st) {
    const int esize = dtype == TL_F32 ? 4 : 2;
    if (spans.n == 0) return TL_OK;
    int longest = 0;
    for (int i = 0; i < spans.n; ++i) longest = spans.count[i] > longest ? spans.count[i] : longest;
    const bool vec = (head_dim * esize) % 16 == 0 && aligned16(key_pages) && aligned16(value_pages) && aligned16(keys) && aligned16(values) &&
                     (src_head_stride * esize) % 16 == 0 && (src_token_stride * esize) % 16 == 0;
    const int threads = 256;
    if (vec) {
        const int per = 16 / esize, dvec = head_dim / per;
        const long long work = static_cast<long long>(heads) * longest * dvec;
        dim3 grid(static_cast<unsigned>(std::min<long long>(ceil_div_ll(work, threads), 64)), spans.n);
        paged_cache_append_chunk_kernel<uint4><<<grid, threads, 0, st>>>(static_cast<uint4 *>(key_pages), static_cast<uint4 *>(value_pages),
                                                                       static_cast<const uint4 *>(keys), static_cast<const uint4 *>(values),
                                                                       spans, heads, page_size, dvec, src_head_stride / per, src_token_stride / per);
    } else {
        const long long work = static_cast<long long>(heads) * longest * head_dim;
        dim3 grid(static_cast<unsigned>(std::min<long long>(ceil_div_ll(work, threads), 64)), spans.n);
        if (esize == 4)
            paged_cache_append_chunk_kernel<uint32_t><<<grid, threads, 0, st>>>(
                static_cast<uint32_t *>(key_pages), static_cast<uint32_t *>(value_pages), static_cast<const uint32_t *>(keys),
                static_cast<const uint32_t *>(values), spans, heads, page_size, head_dim, src_head_stride, src_token_stride);
        else
            paged_cache_append_chunk_kernel<uint16_t><<<grid, threads, 0, st>>>(
                static_cast<uint16_t *>(key_pages), static_cast<uint16_t *>(value_pages), static_cast<const uint16_t *>(keys),
                static_cast<const uint16_t *>(values), spans, heads, page_size, head_dim, src_head_stride, src_token_stride);
    }
    TL_LAUNCH_CHECK("paged_cache_append_chunk");
    return TL_OK;
}

// Decode-batch append: row b owns token ctx[b]-1; page id and slot are read
// from device memory (graph-replayable).  keys/values [B, H, 1, D].
template <typename V>
__global__ void paged_cache_append_decode_kernel(V *__restrict__ key_pages, V *__restrict__ value_pages,
                                                 const V *__restrict__ keys, const V *__restrict__ values,
                                                 const int32_t *__restrict__ block_table,
                                                 const int32_t *__restrict__ context_lens, int batch, int num_pages,
                                                 int heads, int page_size, int dvec, int max_pages) {
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(batch) * heads * dvec;
    if (idx >= total) return;
    const int d = static_cast<int>(idx % dvec);
    const int h = static_cast<int>((idx / dvec) % heads);
    const int b = static_cast<int>(idx / (static_cast<long long>(dvec) * heads));
    const int ctx = context_lens[b];
    if (ctx <= 0) return;
    const int tok = ctx - 1;
    const int lp = tok / page_size;
    if (lp >= max_pages) return;
    const int pid = block_table[static_cast<size_t>(b) * max_pages + lp];
    if (pid < 0 || pid >= num_pages) return;
    const size_t dst = ((static_cast<size_t>(pid) * heads + h) * page_size + (tok - lp * page_size)) * dvec + d;
    key_pages[dst] = keys[idx];
    value_pages[dst] = values[idx];
}

int launch_paged_cache_append_decode(void *key_pages, void *value_pages, const void *keys, const void *values,
                                     const int32_t *block_table, const int32_t *context_lens, int batch,
                                     int num_pages, int heads, int page_size, int head_dim, int max_pages, int dtype,
                                     cudaStream_t st) {
    const int esize = dtype == TL_F32 ? 4 : 2;
    const long long elems = static_cast<long long>(batch) * heads * head_dim;
    if (elems == 0) return TL_OK;
    const int threads = 256;
    const bool vec = (head_dim * esize) % 16 == 0 && aligned16(key_pages) && aligned16(value_pages) &&
                     aligned16(keys) && aligned16(values);
#define TL_APPEND(V, DV)                                                                                         \
    paged_cache_append_decode_kernel<V>                                                                          \
        <<<static_cast<unsigned>(ceil_div_ll(static_cast<long long>(batch) * heads * (DV), threads)), threads, 0, \
           st>>>(static_cast<V *>(key_pages), static_cast<V *>(value_pages), static_cast<const V *>(keys),      \
                 static_cast<const V *>(values), block_table, context_lens, batch, num_pages, heads, page_size,  \
                 (DV), max_pages)
    if (vec) {
        TL_APPEND(uint4, head_dim * esize / 16);
    } else if (esize == 4) {
        TL_APPEND(uint32_t, head_dim);
    } else {
        TL_APPEND(uint16_t, head_dim);
    }
#undef TL_APPEND
    TL_LAUNCH_CHECK("paged_cache_append_decode");
    return TL_OK;
}

// ---------------------------------------------------------- greedy argmax --
struct Best {
    float v;
    int i;
};
__device__ __forceinline__ Best better(Best a, Best b) {
    return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;  // first maximum wins
}
__device__ __forceinline__ Best block_best(Best mine) {
    __shared__ float sv[32];
    __shared__ int si[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Best other{__shfl_xor_sync(0xffffffffu, mine.v, o), __shfl_xor_sync(0xffffffffu, mine.i, o)};
        mine = better(mine, other);
    }
    if ((threadIdx.x & 31) == 0) sv[threadIdx.x >> 5] = mine.v, si[threadIdx.x >> 5] = mine.i;
    __syncthreads();
    const int nw = (blockDim.x + 31) / 32;
    Best r{(threadIdx.x & 31) < nw ? sv[threadIdx.x & 31] : -INFINITY, (threadIdx.x & 31) < nw ? si[threadIdx.x & 31] : INT_MAX};
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Best other{__shfl_xor_sync(0xffffffffu, r.v, o), __shfl_xor_sync(0xffffffffu, r.i, o)};
        r = better(r, other);
    }
    return r;
}

template <typename T>
__global__ void argmax_partial_kernel(const T *__restrict__ logits, float *__restrict__ pv, int *__restrict__ pi,
                                      int vocab, int chunk, int vec) {
    const int row = blockIdx.y;
    const int begin = blockIdx.x * chunk;
    const int end = min(vocab, begin + chunk);
    const T *src = logits + static_cast<size_t>(row) * vocab;
    Best mine{-INFINITY, INT_MAX};
    if constexpr (sizeof(T) == 2) {
        if (vec) {  // chunk, vocab and the row pitch are multiples of 8 elements: 128-bit loads
            for (int i = begin + threadIdx.x * 8; i < end; i += blockDim.x * 8) {
                const uint4 raw = *reinterpret_cast<const uint4 *>(src + i);
                const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = unpack2<T>(w[j]);
                    mine = better(mine, Best{f.x, i + 2 * j});
                    mine = better(mine, Best{f.y, i + 2 * j + 1});
                }
            }
            mine = block_best(mine);
            if (threadIdx.x == 0) pv[row * gridDim.x + blockIdx.x] = mine.v, pi[row * gridDim.x + blockIdx.x] = mine.i;
            return;
        }
    }
    for (int i = begin + threadIdx.x; i < end; i += blockDim.x) mine = better(mine, Best{to_f(src[i]), i});
    mine = block_best(mine);
    if (threadIdx.x == 0) pv[row * gridDim.x + blockIdx.x] = mine.v, pi[row * gridDim.x + blockIdx.x] = mine.i;
}

__global__ void argmax_final_kernel(const float *__restrict__ pv, const int *__restrict__ pi, int32_t *__restrict__ out,
                                    int parts) {
    const int row = blockIdx.x;
    Best mine{-INFINITY, INT_MAX};
    for (int i = threadIdx.x; i < parts; i += blockDim.x) mine = better(mine, Best{pv[row * parts + i], pi[row * parts + i]});
    mine = block_best(mine);
    if (threadIdx.x == 0) out[row] = mine.i == INT_MAX ? 0 : mine.i;
}

static int argmax_parts(int vocab) { return vocab <= 4096 ? 1 : (ceil_div(vocab, 4096) < 64 ? ceil_div(vocab, 4096) : 64); }

size_t argmax_workspace(int rows, int vocab) { return static_cast<size_t>(rows) * argmax_parts(vocab) * 8; }

int launch_argmax(const void *logits, int32_t *out, int rows, int vocab, int dtype, void *ws, size_t ws_bytes,
                  cudaStream_t st) {
    if (rows == 0) return TL_OK;
    const int parts = argmax_parts(vocab);
    if (ws == nullptr || ws_bytes < argmax_workspace(rows, vocab)) return fail(TL_EWORKSPACE, "argmax: workspace too small");
    float *pv = static_cast<float *>(ws);
    int *pi = reinterpret_cast<int *>(pv + static_cast<size_t>(rows) * parts);
    const int chunk = ceil_div(ceil_div(vocab, parts), 8) * 8;
    const int vec = (vocab % 8 == 0 && aligned16(logits)) ? 1 : 0;
    dim3 grid(parts, rows);
    switch (dtype) {
        case TL_F32: argmax_partial_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(logits), pv, pi, vocab, chunk, vec); break;
        case TL_F16: argmax_partial_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half *>(logits), pv, pi, vocab, chunk, vec); break;
        case TL_BF16:
            argmax_partial_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(static_cast<const __nv_bfloat16 *>(logits), pv, pi, vocab, chunk, vec);
            break;
        default: return fail(TL_EDTYPE, "argmax: expected float32, float16, or bfloat16");
    }
    TL_LAUNCH_CHECK("argmax_partial");
    argmax_final_kernel<<<rows, 64, 0, st>>>(pv, pi, out, parts);
    TL_LAUNCH_CHECK("argmax_final");
    return TL_OK;
}

// -------------------------------------- fused q/k norm + RoPE + KV append ----
// Decode step (L == 1).  qkv [B, (Hq + 2*Hkv) * D] holds the q heads, then the k
// heads, then the v heads of each request.  One CTA per (head, request), D/2
// threads, thread i owns the non-traditional RoPE pair (i, i + D/2):
//   q/k heads: n = T(x * rsqrt(mean(x^2)+eps) * w)   -- rounded, as rms_norm stores it
//              y = T(rope(n))                        -- as rope stores it
//   q -> q_out [B, Hq, D];  k, v -> page slot of token context_lens[b]-1.
// Same arithmetic and rounding points as rms_norm -> rope -> paged_cache_update
// (qwen3_week3.py:69-96), in one launch instead of six.
template <typename T>
__global__ void decode_qk_norm_rope_append_kernel(const T *qkv, const T *__restrict__ qw,
                                                  const T *__restrict__ kw, const int32_t *__restrict__ offsets,
                                                  const int32_t *__restrict__ bt, const int32_t *__restrict__ cl,
                                                  T *__restrict__ q_out, T *__restrict__ kp, T *__restrict__ vp, int Hq,
                                                  int Hkv, int D, float base, float eps, int num_pages, int page_size,
                                                  int max_pages, int bt_stride, long long q_row_stride, long long q_head_stride) {
    // bt_stride: block-table elements between rows (max_pages: one request per row; 0: every row is a token of ONE
    // request - a prefill chunk).  q_out element (row b, head h) starts at b * q_row_stride + h * q_head_stride.
    __shared__ float warp_part[8];
    griddep_launch();
    griddep_wait();  // qkv is the previous kernel's output: read through L2 (common.cuh: programmatic dependent launch)
    const int head = blockIdx.x;  // 0..Hq-1 q | Hq..Hq+Hkv-1 k | rest v
    const int b = blockIdx.y;
    const int half = D / 2;
    const int i = threadIdx.x;
    const T *src = qkv + (static_cast<size_t>(b) * (Hq + 2 * Hkv) + head) * D;
    const bool is_q = head < Hq;
    const bool is_k = !is_q && head < Hq + Hkv;
    const int kvh = is_q ? 0 : (is_k ? head - Hq : head - Hq - Hkv);

    float re = 0.f, im = 0.f;
    if (i < half) re = to_f(ld_cg(src + i)), im = to_f(ld_cg(src + i + half));
    T out_re, out_im;
    if (is_q || is_k) {
        float ss = warp_sum(re * re + im * im);
        if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = ss;
        __syncthreads();
        const int nw = (blockDim.x + 31) / 32;
        float tot = (threadIdx.x & 31) < nw ? warp_part[threadIdx.x & 31] : 0.f;
        tot = warp_sum(tot);
        const float inv = rsqrtf(tot / static_cast<float>(D) + eps);
        const T *w = is_q ? qw : kw;
        float nre = 0.f, nim = 0.f;
        if (i < half) {
            nre = to_f(from_f<T>(re * inv * to_f(w[i])));
            nim = to_f(from_f<T>(im * inv * to_f(w[i + half])));
        }
        const double inv_freq = exp2(-static_cast<double>(i) / static_cast<double>(half) * log2(static_cast<double>(base)));
        const float angle = static_cast<float>(static_cast<double>(offsets[b]) * inv_freq);
        float s, c;
        sincosf(angle, &s, &c);
        out_re = from_f<T>(nre * c - nim * s);
        out_im = from_f<T>(nim * c + nre * s);
    } else {
        out_re = from_f<T>(re);
        out_im = from_f<T>(im);
    }
    if (i >= half) return;
    if (is_q) {
        T *dst = q_out + static_cast<size_t>(b) * q_row_stride + static_cast<size_t>(head) * q_head_stride;
        dst[i] = out_re, dst[i + half] = out_im;
        return;
    }
    const int ctx = cl[b];
    if (ctx <= 0) return;
    const int tok = ctx - 1;
    const int lp = tok / page_size;
    if (lp >= max_pages) return;
    const int pid = bt[static_cast<size_t>(b) * bt_stride + lp];
    if (pid < 0 || pid >= num_pages) return;
    T *dst = (is_k ? kp : vp) + ((static_cast<size_t>(pid) * Hkv + kvh) * page_size + (tok - lp * page_size)) * D;
    dst[i] = out_re, dst[i + half] = out_im;
}

// The same for D == 128 (every Qwen3): one CTA per ROW (request or chunk token), sixteen warps, warp w takes heads w,
// w + 16, ...; lane l owns the RoPE pairs (l, l + 64) and (l + 32, l + 96), so the angle arithmetic (a double-precision
// exp2 and a sincosf per pair) is done once per lane instead of once per head, and the sum of squares is two warp
// reductions.  All of a warp's loads are issued before the first is used (one L2
// round trip; a first version that walked its heads one after the other was slower than the one-CTA-per-head form).
// A dependent-latency chain either way (load -> trig -> norm -> store); the gain is the chunk's 6144 tiny CTAs.  Bit-identical to the per-head kernel: the squares are added in the same tree (pairs
// 0..31 and 32..63 reduced separately, then summed).
constexpr int QKN_WARPS = 16, QKN_MAXH = 4;  // up to 64 heads (q + k + v) per row
// PLANES: qkv does not exist in memory - its rows are still the fp32 partial planes of the q|k|v projection's split
// reduction (w4a16_skinny.cu); this kernel adds them (split order, as the reduction launch would) and rounds to T first.
template <typename T, bool PLANES>
__global__ void __launch_bounds__(QKN_WARPS * 32) decode_qk_norm_rope_append_d128_kernel(
    const T *qkv, const float *part, int splits, long long plane, const T *__restrict__ qw, const T *__restrict__ kw, const int32_t *__restrict__ offsets, const int32_t *__restrict__ bt,
    const int32_t *__restrict__ cl, T *q_out, T *kp, T *vp, int Hq, int Hkv, float base, float eps, int num_pages, int page_size, int max_pages,
    int bt_stride, long long q_row_stride, long long q_head_stride) {
    constexpr int D = 128, half = 64;
    griddep_launch();
    griddep_wait();  // qkv is the previous kernel's output: read through L2 (common.cuh: programmatic dependent launch)
    const int b = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int heads = Hq + 2 * Hkv;
    float re[QKN_MAXH][2], im[QKN_MAXH][2];
    if constexpr (PLANES) {
        const float *prow = part + static_cast<size_t>(b) * heads * D;
#pragma unroll
        for (int hh = 0; hh < QKN_MAXH; ++hh)
#pragma unroll
            for (int j = 0; j < 2; ++j) re[hh][j] = im[hh][j] = 0.f;
        for (int sp0 = 0; sp0 < splits; sp0 += 4) {  // four planes per round trip, added in split order
            float v[QKN_MAXH][4][4];
#pragma unroll
            for (int hh = 0; hh < QKN_MAXH; ++hh) {
                const int head = warp + QKN_WARPS * hh;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const bool live = head < heads && sp0 + q < splits;
                    const float *src = prow + (sp0 + q) * plane + head * D + lane;
#pragma unroll
                    for (int e = 0; e < 4; ++e) v[hh][q][e] = live ? ld_cg(src + 32 * e) : 0.f;  // e: pairs (l, l+64), (l+32, l+96) -> offsets 0, 32, 64, 96
                }
            }
#pragma unroll
            for (int hh = 0; hh < QKN_MAXH; ++hh)
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (sp0 + q < splits) re[hh][0] += v[hh][q][0], re[hh][1] += v[hh][q][1], im[hh][0] += v[hh][q][2], im[hh][1] += v[hh][q][3];
        }
#pragma unroll
        for (int hh = 0; hh < QKN_MAXH; ++hh)
#pragma unroll
            for (int j = 0; j < 2; ++j) re[hh][j] = to_f(from_f<T>(re[hh][j])), im[hh][j] = to_f(from_f<T>(im[hh][j]));  // the projection's rounding
    } else {
        const T *row = qkv + static_cast<size_t>(b) * heads * D;
#pragma unroll
        for (int hh = 0; hh < QKN_MAXH; ++hh) {
            const int head = warp + QKN_WARPS * hh;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                re[hh][j] = head < heads ? to_f(ld_cg(row + head * D + lane + 32 * j)) : 0.f;
                im[hh][j] = head < heads ? to_f(ld_cg(row + head * D + lane + 32 * j + half)) : 0.f;
            }
        }
    }
    // the 64 (sin, cos) pairs of this row's position: computed ONCE per CTA by its first two warps (one pair index per
    // thread: a double-precision exp2 and a large-argument sincosf each) and shared; every lane doing its own kept the
    // FP64 / slow-path trig pipes busy 16x over
    __shared__ float sn_s[half], cs_s[half];
    if (threadIdx.x < half) {
        const int i = threadIdx.x;
        const double inv_freq = exp2(-static_cast<double>(i) / static_cast<double>(half) * log2(static_cast<double>(base)));
        const float angle = static_cast<float>(static_cast<double>(offsets[b]) * inv_freq);
        sincosf(angle, &sn_s[i], &cs_s[i]);
    }
    __syncthreads();
    float sn[2], cs[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) sn[j] = sn_s[lane + 32 * j], cs[j] = cs_s[lane + 32 * j];
    // page slot of this row's token (k / v heads)
    const int ctx = cl[b];
    T *k_dst = nullptr, *v_dst = nullptr;
    if (ctx > 0) {
        const int tok = ctx - 1, lp = tok / page_size;
        if (lp < max_pages) {
            const int pid = bt[static_cast<size_t>(b) * bt_stride + lp];
            if (pid >= 0 && pid < num_pages) {
                const size_t slot = (static_cast<size_t>(pid) * Hkv * page_size + (tok - lp * page_size)) * D;
                k_dst = kp + slot, v_dst = vp + slot;
            }
        }
    }
#pragma unroll
    for (int hh = 0; hh < QKN_MAXH; ++hh) {
        const int head = warp + QKN_WARPS * hh;
        if (head >= heads) break;  // warp-uniform
        const bool is_q = head < Hq, is_k = !is_q && head < Hq + Hkv;
        T o_re[2], o_im[2];
        if (is_q || is_k) {
            const float tot = warp_sum(re[hh][0] * re[hh][0] + im[hh][0] * im[hh][0]) + warp_sum(re[hh][1] * re[hh][1] + im[hh][1] * im[hh][1]);
            const float inv = rsqrtf(tot / static_cast<float>(D) + eps);
            const T *w = is_q ? qw : kw;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int i = lane + 32 * j;
                const float nre = to_f(from_f<T>(re[hh][j] * inv * to_f(w[i])));
                const float nim = to_f(from_f<T>(im[hh][j] * inv * to_f(w[i + half])));
                o_re[j] = from_f<T>(nre * cs[j] - nim * sn[j]);
                o_im[j] = from_f<T>(nim * cs[j] + nre * sn[j]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 2; ++j) o_re[j] = from_f<T>(re[hh][j]), o_im[j] = from_f<T>(im[hh][j]);
        }
        T *dst;
        if (is_q) {
            dst = q_out + static_cast<size_t>(b) * q_row_stride + static_cast<size_t>(head) * q_head_stride;
        } else {
            T *base_dst = is_k ? k_dst : v_dst;
            if (base_dst == nullptr) continue;  // warp-uniform
            const int kvh = is_k ? head - Hq : head - Hq - Hkv;
            dst = base_dst + static_cast<size_t>(kvh) * page_size * D;
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) dst[lane + 32 * j] = o_re[j], dst[lane + 32 * j + half] = o_im[j];
    }
}

int launch_decode_qk_norm_rope_append(const void *qkv, const void *q_norm_w, const void *k_norm_w, const int32_t *offsets,
                                      const int32_t *block_table, const int32_t *context_lens, void *q_out, void *key_pages,
                                      void *value_pages, int batch, int Hq, int Hkv, int D, float base, float eps,
                                      int num_pages, int page_size, int max_pages, int dtype, cudaStream_t st, bool chunk) {
    if (batch == 0) return TL_OK;
    // chunk: the rows are the tokens of one request (shared block-table row); q_out is [Hq, rows, D], the layout
    // paged_attention takes; otherwise one request per row and q_out [rows, Hq, D]
    const int bt_stride = chunk ? 0 : max_pages;
    const long long q_row_stride = chunk ? D : static_cast<long long>(Hq) * D;
    const long long q_head_stride = chunk ? static_cast<long long>(batch) * D : D;
    const int threads = ((D / 2 + 31) / 32) * 32;
    dim3 grid(Hq + 2 * Hkv, batch);
    if (qkv_planes_rope_supported(Hq, Hkv, D, dtype)) {  // one CTA per row (see the kernel's comment)
        using T = __nv_bfloat16;
        launch_chained(decode_qk_norm_rope_append_d128_kernel<T, false>, dim3(batch), dim3(QKN_WARPS * 32), 0, st, static_cast<const T *>(qkv),
                       static_cast<const float *>(nullptr), 0, 0LL, static_cast<const T *>(q_norm_w), static_cast<const T *>(k_norm_w), offsets, block_table, context_lens, static_cast<T *>(q_out),
                       static_cast<T *>(key_pages), static_cast<T *>(value_pages), Hq, Hkv, base, eps, num_pages, page_size, max_pages, bt_stride,
                       q_row_stride, q_head_stride);
        TL_LAUNCH_CHECK("decode_qk_norm_rope_append");
        return TL_OK;
    }
#define TL_QKN(T)                                                                                                      \
    launch_chained(decode_qk_norm_rope_append_kernel<T>, grid, dim3(threads), 0, st,                                  \
        static_cast<const T *>(qkv), static_cast<const T *>(q_norm_w), static_cast<const T *>(k_norm_w), offsets,     \
        block_table, context_lens, static_cast<T *>(q_out), static_cast<T *>(key_pages), static_cast<T *>(value_pages), \
        Hq, Hkv, D, base, eps, num_pages, page_size, max_pages, bt_stride, q_row_stride, q_head_stride)
    if (dtype == TL_BF16)
        TL_QKN(__nv_bfloat16);
    else if (dtype == TL_F32)
        TL_QKN(float);
    else
        return fail(TL_EDTYPE, "decode_qk_norm_rope_append: bfloat16 or float32 required");
#undef TL_QKN
    TL_LAUNCH_CHECK("decode_qk_norm_rope_append");
    return TL_OK;
}

// The row kernel's shapes (bf16, D == 128, <= 64 heads): it runs the standalone forms there, and only it can take the
// split-reduction planes of the q|k|v projection; everything else runs the per-head kernel
bool qkv_planes_rope_supported(int Hq, int Hkv, int D, int dtype) { return D == 128 && dtype == TL_BF16 && Hq + 2 * Hkv <= QKN_WARPS * QKN_MAXH; }
int launch_qkv_planes_rope_append(const float *part, int splits, const void *q_norm_w, const void *k_norm_w, const int32_t *offsets,
                                  const int32_t *block_table, const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int batch,
                                  int Hq, int Hkv, float base, float eps, int num_pages, int page_size, int max_pages, cudaStream_t st, bool chunk) {
    using T = __nv_bfloat16;
    constexpr int D = 128;
    const int bt_stride = chunk ? 0 : max_pages;
    const long long q_row_stride = chunk ? D : static_cast<long long>(Hq) * D;
    const long long q_head_stride = chunk ? static_cast<long long>(batch) * D : D;
    const long long plane = static_cast<long long>(batch) * (Hq + 2 * Hkv) * D;
    launch_chained(decode_qk_norm_rope_append_d128_kernel<T, true>, dim3(batch), dim3(QKN_WARPS * 32), 0, st, static_cast<const T *>(nullptr), part, splits,
                   plane, static_cast<const T *>(q_norm_w), static_cast<const T *>(k_norm_w), offsets, block_table, context_lens, static_cast<T *>(q_out),
                   static_cast<T *>(key_pages), static_cast<T *>(value_pages), Hq, Hkv, base, eps, num_pages, page_size, max_pages, bt_stride,
                   q_row_stride, q_head_stride);
    TL_LAUNCH_CHECK("qkv_planes_rope_append");
    return TL_OK;
}

// ------------------------------------------------ decode-loop bookkeeping --
__global__ void decode_advance_kernel(int32_t *tokens, const int32_t *next_tokens, int32_t *offsets,
                                      int32_t *context_lens, int32_t *out_log, int32_t *step_counter, int batch,
                                      int log_capacity) {
    const int step = *step_counter;
    for (int b = threadIdx.x; b < batch; b += blockDim.x) {
        const bool active = context_lens[b] > 0;
        const int32_t tok = next_tokens[b];
        if (active) {
            tokens[b] = tok;
            offsets[b] += 1;
            context_lens[b] += 1;
        }
        if (step < log_capacity) out_log[static_cast<size_t>(step) * batch + b] = active ? tok : -1;
    }
    __syncthreads();
    if (threadIdx.x == 0) *step_counter = step + 1;
}

int launch_decode_advance(int32_t *tokens, const int32_t *next_tokens, int32_t *offsets, int32_t *context_lens,
                          int32_t *out_log, int32_t *step_counter, int batch, int log_capacity, cudaStream_t st) {
    decode_advance_kernel<<<1, 128, 0, st>>>(tokens, next_tokens, offsets, context_lens, out_log, step_counter, batch,
                                             log_capacity);
    TL_LAUNCH_CHECK("decode_advance");
    return TL_OK;
}

}  // namespace tl
