// Qwen3-MoE router projection for routers stored as MLX affine 8-bit codes at group 64 (tl_moe_router; the layout
// mlx_lm gives `mlp.gate` when it converts qwen3_moe), which the group-128 projection kernels cannot take:
//
//   logits[t, e] = T( sum_k fp32 (scale[e, g] * code[e, k] + bias[e, g]) * a[t, k] ),  g = k / 64
//
// computed per group as scale * (sum_k code_k a_k) + bias * (sum_k a_k) in fp32.  Both sums are tensor-core products
// with fp32 accumulation from zero at each group: a code (0..255) is exact in bf16 and fp16, so is every product, and
// the row sum of a comes from the same MMA against a column of ones.  With the RMSNorm prologue, a = T(x * rsqrt(mean(x^2)
// + eps) * w), the row visited in rms_norm_kernel's order (elementwise.cu, as moe_gather does), so a is tl_rms_norm's
// output bit for bit.
//
// Every output element goes through the same arithmetic whatever T and the tile shape: the K_SLICES warps of a CTA take
// the groups g = s, s + K_SLICES, ... in increasing order (slice s), fold them into an fp32 partial, and the CTA adds
// the K_SLICES partials in slice order.  So a row's logits depend only on that row, and the decode-sized and
// prefill-sized tiles give the same bits.
#include "common.cuh"
#include "kernels.h"

namespace tl {

namespace {

constexpr int K_SLICES = 8;  // warps per CTA, one slice of the groups each
constexpr int RG = 64;       // inputs per quantisation group

template <typename T>
struct RouterMma;
template <>
struct RouterMma<__nv_bfloat16> {
    static constexpr uint32_t ONES = 0x3F803F80u;
    // 2 codes (bytes b0, b1 of w, selected by `sel`) -> bf16x2, exact: via fp32 2^23 + code
    static __device__ __forceinline__ uint32_t codes2(uint32_t w, int lo) {
        const float f0 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440u | lo)) - 8388608.f;
        const float f1 = __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440u | (lo + 1))) - 8388608.f;
        return pack2<__nv_bfloat16>(f0, f1);
    }
    static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
};
template <>
struct RouterMma<__half> {
    static constexpr uint32_t ONES = 0x3C003C00u;
    // 2 codes -> fp16x2, exact: 1024 + code (0x64XX) minus 1024
    static __device__ __forceinline__ uint32_t codes2(uint32_t w, int lo) {
        const uint32_t sel = 0x4040u | static_cast<uint32_t>(lo) | (static_cast<uint32_t>(lo + 1) << 8);
        const uint32_t biased = __byte_perm(w, 0x64646464u, sel);
        __half2 h = *reinterpret_cast<const __half2 *>(&biased);
        const uint32_t k1024 = 0x64006400u;
        h = __hsub2(h, *reinterpret_cast<const __half2 *>(&k1024));
        return *reinterpret_cast<uint32_t *>(&h);
    }
    static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
};

// 1 / rms of row xr, visited as rms_norm_kernel<T, TPR, EPV == 8> visits it: thread `lane` of TPR sums the squares of its
// chunks at lane * EPV + n * TPR * EPV in order, then the warp and (TPR = 256) CTA reductions.
template <typename T, int TPR, int EPV>
__device__ __forceinline__ float router_row_inv(const T *xr, int H, float eps, int lane, float *part) {
    float ss = 0.f;
    for (int c = lane * EPV; c < H; c += TPR * EPV)
#pragma unroll
        for (int q = 0; q < EPV; ++q) {
            const float v = to_f(ld_cg(xr + c + q));
            ss += v * v;
        }
    ss = warp_sum(ss);
    if constexpr (TPR > 32) {
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = ss;
        __syncthreads();
        ss = warp_sum((threadIdx.x & 31) < TPR / 32 ? part[threadIdx.x & 31] : 0.f);
        __syncthreads();  // part is written again by the next row
    }
    return rsqrtf(ss / static_cast<float>(H) + eps);
}

// Eight consecutive inputs of one row as four packed pairs; with the prologue they are normalised and rounded to T.
template <typename T, bool NORM>
__device__ __forceinline__ uint4 load_a8(const T *row, const T *__restrict__ nw, int k, float inv) {
    const uint4 raw = ld_cg(reinterpret_cast<const uint4 *>(row + k));
    if constexpr (!NORM) {
        return raw;
    } else {
        const uint4 g = *reinterpret_cast<const uint4 *>(nw + k);
        const uint32_t rv[4] = {raw.x, raw.y, raw.z, raw.w}, gv[4] = {g.x, g.y, g.z, g.w};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 v = unpack2<T>(rv[i]), w = unpack2<T>(gv[i]);
            o[i] = pack2<T>(v.x * inv * w.x, v.y * inv * w.y);
        }
        return make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// CTA: MI m16 row tiles x NT n8 expert tiles, K_SLICES warps.  Inside a k32 chunk, thread (g = lane / 4, c = lane % 4)
// owns inputs 8c .. 8c + 7: MMA step 0 takes 8c + 0..3 as the fragment's k = 2c, 2c + 1, 2c + 8, 2c + 9, step 1 takes
// 8c + 4..7, for both operands alike, so every input of the chunk is multiplied exactly once.
template <typename T, int MI, int NT, bool NORM, int TPR>
__global__ void __launch_bounds__(K_SLICES * 32) moe_router_kernel(const T *__restrict__ x, const T *__restrict__ nw, float eps,
                                                                 const uint32_t *__restrict__ wq, const T *__restrict__ scales,
                                                                 const T *__restrict__ biases, T *__restrict__ out, int rows, int E, int H) {
    constexpr int MT = 16 * MI, NE = 8 * NT;
    __shared__ float red[K_SLICES][MT][NE + 1];
    __shared__ float inv_s[NORM ? MT : 1];
    __shared__ float part[K_SLICES];
    griddep_launch();
    griddep_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g8 = lane >> 2, c4 = lane & 3;
    const int r0 = blockIdx.y * MT, e0 = blockIdx.x * NE;
    const int G = H / RG, words = H / 4;

    if constexpr (NORM) {
        if constexpr (TPR == 32) {
            for (int r = warp; r < MT; r += K_SLICES) {
                const float inv = r0 + r < rows ? router_row_inv<T, 32, 8>(x + static_cast<size_t>(r0 + r) * H, H, eps, lane, part) : 0.f;
                if (lane == 0) inv_s[r] = inv;
            }
        } else {
            for (int r = 0; r < MT && r0 + r < rows; ++r) {
                const float inv = router_row_inv<T, 256, 8>(x + static_cast<size_t>(r0 + r) * H, H, eps, threadIdx.x, part);
                if (threadIdx.x == 0) inv_s[r] = inv;
            }
        }
        __syncthreads();
    }

    // this thread's rows (g8, g8 + 8 of each m16 tile) and experts (g8 of each n8 tile for the codes; 2 c4, 2 c4 + 1 for
    // the outputs)
    const T *arow[MI][2];
    bool alive[MI][2];
    float ainv[MI][2];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = r0 + 16 * i + 8 * h + g8;
            alive[i][h] = r < rows;
            arow[i][h] = x + static_cast<size_t>(alive[i][h] ? r : 0) * H;
            ainv[i][h] = NORM ? inv_s[16 * i + 8 * h + g8] : 0.f;
        }
    const uint32_t *wrow[NT];
    bool elive[NT];
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        const int e = e0 + 8 * j + g8;
        elive[j] = e < E;
        wrow[j] = wq + static_cast<size_t>(elive[j] ? e : 0) * words;
    }
    bool m_any[MI];
#pragma unroll
    for (int i = 0; i < MI; ++i) m_any[i] = r0 + 16 * i < rows;

    float acc[MI][NT][4];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

    for (int grp = warp; grp < G; grp += K_SLICES) {
        float dot[MI][NT][4], asum[MI][4];
#pragma unroll
        for (int i = 0; i < MI; ++i) {
#pragma unroll
            for (int q = 0; q < 4; ++q) asum[i][q] = 0.f;
#pragma unroll
            for (int j = 0; j < NT; ++j)
#pragma unroll
                for (int q = 0; q < 4; ++q) dot[i][j][q] = 0.f;
        }
#pragma unroll
        for (int ch = 0; ch < RG / 32; ++ch) {
            const int k = grp * RG + ch * 32 + 8 * c4;
            uint4 av[MI][2];
            uint2 bv[NT];
#pragma unroll
            for (int j = 0; j < NT; ++j) bv[j] = elive[j] ? *reinterpret_cast<const uint2 *>(wrow[j] + k / 4) : make_uint2(0u, 0u);
#pragma unroll
            for (int i = 0; i < MI; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h) av[i][h] = alive[i][h] ? load_a8<T, NORM>(arow[i][h], nw, k, ainv[i][h]) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int step = 0; step < 2; ++step) {
                uint32_t b0[NT], b1[NT];
#pragma unroll
                for (int j = 0; j < NT; ++j) {
                    const uint32_t w = step == 0 ? bv[j].x : bv[j].y;
                    b0[j] = RouterMma<T>::codes2(w, 0);
                    b1[j] = RouterMma<T>::codes2(w, 2);
                }
#pragma unroll
                for (int i = 0; i < MI; ++i) {
                    if (!m_any[i]) continue;
                    const uint32_t a[4] = {step == 0 ? av[i][0].x : av[i][0].z, step == 0 ? av[i][1].x : av[i][1].z,
                                           step == 0 ? av[i][0].y : av[i][0].w, step == 0 ? av[i][1].y : av[i][1].w};
                    RouterMma<T>::mma(asum[i], a, RouterMma<T>::ONES, RouterMma<T>::ONES);
#pragma unroll
                    for (int j = 0; j < NT; ++j) RouterMma<T>::mma(dot[i][j], a, b0[j], b1[j]);
                }
            }
        }
        // fold the group: acc += scale * dot + bias * asum (fp32)
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            float sc[2], bi[2];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const int e = e0 + 8 * j + 2 * c4 + q;
                sc[q] = e < E ? to_f(scales[static_cast<size_t>(e) * G + grp]) : 0.f;
                bi[q] = e < E ? to_f(biases[static_cast<size_t>(e) * G + grp]) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < MI; ++i)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[i][j][q] = fmaf(bi[q & 1], asum[i][q & 2], fmaf(sc[q & 1], dot[i][j][q], acc[i][j][q]));
        }
    }

    // the slices' partials, added in slice order
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) red[warp][16 * i + 8 * (q >> 1) + g8][8 * j + 2 * c4 + (q & 1)] = acc[i][j][q];
    __syncthreads();
    for (int idx = threadIdx.x; idx < MT * NE; idx += K_SLICES * 32) {
        const int r = idx / NE, n = idx % NE;
        if (r0 + r >= rows || e0 + n >= E) continue;
        float s = red[0][r][n];
#pragma unroll
        for (int w = 1; w < K_SLICES; ++w) s += red[w][r][n];
        out[static_cast<size_t>(r0 + r) * E + e0 + n] = from_f<T>(s);
    }
}

template <typename T, int MI, int NT>
cudaError_t router_launch(const void *x, const void *nw, float eps, const void *w, const void *scales, const void *biases, void *out, int T_,
                          int E, int H, int dtype, cudaStream_t st) {
    const dim3 grid(ceil_div(E, 8 * NT), ceil_div(T_, 16 * MI)), block(K_SLICES * 32);
    const T *xp = static_cast<const T *>(x), *np = static_cast<const T *>(nw);
    const uint32_t *wp = static_cast<const uint32_t *>(w);
    const T *sp = static_cast<const T *>(scales), *bp = static_cast<const T *>(biases);
    T *op = static_cast<T *>(out);
    if (nw == nullptr) return launch_chained(moe_router_kernel<T, MI, NT, false, 32>, grid, block, 0, st, xp, np, eps, wp, sp, bp, op, T_, E, H);
    bool vec = false;
    const int tpr = rms_norm_path(H, dtype, x, nw, x, &vec);  // vec holds: H % 64 == 0 and both are 16-byte aligned
    if (tpr == 32) return launch_chained(moe_router_kernel<T, MI, NT, true, 32>, grid, block, 0, st, xp, np, eps, wp, sp, bp, op, T_, E, H);
    return launch_chained(moe_router_kernel<T, MI, NT, true, 256>, grid, block, 0, st, xp, np, eps, wp, sp, bp, op, T_, E, H);
}

// Wide tiles once the pass is long enough to fill the GPU with them (T = 1024 at 128 experts).
bool moe_router_wide_tiles(int T, int E) { return static_cast<long long>(T) * E >= 128 * 1024; }

template <typename T>
cudaError_t router_t(const void *x, const void *nw, float eps, const void *w, const void *scales, const void *biases, void *out, int T_, int E,
                     int H, int dtype, cudaStream_t st) {
    // decode- and chunk-sized row counts: one m16 x n8 tile per CTA, so a few rows still spread over E / 8 CTAs;
    // long prefill passes: 32 x 32 tiles, which read each activation row E / 32 times instead of E / 8
    if (moe_router_wide_tiles(T_, E))
        return router_launch<T, 2, 4>(x, nw, eps, w, scales, biases, out, T_, E, H, dtype, st);
    return router_launch<T, 1, 1>(x, nw, eps, w, scales, biases, out, T_, E, H, dtype, st);
}

}  // namespace

int launch_moe_router(const void *x, const void *norm_weight, float eps, const void *w, const void *scales, const void *biases, void *out, int T,
                      int E, int H, int dtype, cudaStream_t st) {
    if (T == 0) return TL_OK;
    const cudaError_t e = dtype == TL_F16 ? router_t<__half>(x, norm_weight, eps, w, scales, biases, out, T, E, H, dtype, st)
                                          : router_t<__nv_bfloat16>(x, norm_weight, eps, w, scales, biases, out, T, E, H, dtype, st);
    if (e != cudaSuccess) return fail(TL_ECUDA, "moe_router: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("moe_router");
    return TL_OK;
}

}  // namespace tl
