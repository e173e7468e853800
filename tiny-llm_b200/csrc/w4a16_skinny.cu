// W4A16 GEMM on the Hopper tensor cores, swap-AB: the dequantised WEIGHTS are the 64-row A operand of wgmma, the
// activation rows (tokens) the N operand.  Two uses:
//
//   * "skinny" (9 <= M <= 128 activation rows: batched decode steps, 128-token prefill chunks): one token tile of
//     NT = 16 / 32 / 64 / 128 columns, the reduction split over `splits` CTAs per feature tile so that EVERY SM
//     streams weights; partial sums go to a workspace in fp32 and a small second launch adds the planes in split
//     order (deterministic) and runs the epilogue (plain / + residual / SwiGLU of interleaved gate|up rows);
//   * prefill (any M, launch_w4a16_tiles): 128-token tiles along grid.y, no split, the epilogue in the kernel.
//
//   out[m, n] = sum_k a[m, k] * T(code[n, k] * scale[n, k/128] + bias[n, k/128])       (m = token, n = feature)
//
// Reference's answer on its hardware: quantized_matmul_splitk (quantized_matmul.metal:251-293, policy
// quantized_matmul.cpp:136-150).  One CTA = 128 output features x NT tokens, 384 threads:
//
//   warp 0             TMA producer of the packed weights: one 128-row x 128-byte box = two quantisation groups of
//                      128 reduction elements per copy, PSTAGES boxes in flight;
//   warp 1             TMA producer of the activations: two [NT x 64] tiles per 128-wide group block (tokens beyond
//                      M zero-filled by the TMA unit), BSTAGES blocks in flight;
//   warpgroups 1, 2    consumers, 64 feature rows each: thread (row, half) turns 64 codes of its row into T (LOP3
//                      magic -> exact code -> one HFMA2, the rounding point of the reference's tiled kernel,
//                      quantized_matmul.metal:183-194) and stores them in the K-major 128-byte-swizzled layout
//                      wgmma reads; then the warpgroup issues eight wgmma m64nNTk16 (fp32 accumulators in
//                      registers) and dequantises the next block while they run (two A stages per warpgroup).
//
// 8-bit codes (BITS = 8, b [K, N/4], code i of a word = (w >> 8i) & 255): a 128-byte box row holds ONE group, so a box
// is one group block and is released after it.  Thread (row, half) reads 64 bytes = 64 codes.  The dequantiser keeps the
// W4 rounding point, T(code * scale + bias) rounded once by one HFMA2 from the exact code:
//   fp16: PRMT (0x64, q) -> 1024 + q, exact for every byte; HSUB2 -> q;
//   bf16: 128 + q is exact only below q = 128, so PRMT (0x4B0000, q) -> fp32 2^23 + q, FADD -> q in fp32; q has at most
//         8 significant bits, so the high halves of two such floats (one PRMT) are the bf16 codes, exactly.
// Instruction budget per 64 codes (one thread, one block): fp16 32 PRMT + 32 HSUB2 + 32 HFMA2 (96); bf16 96 PRMT + 64 FADD
// + 32 HFMA2 (192), against W4's 32 LOP3 + 24 SHF + 32 HSUB2 + 32 HFMA2 + 16 PRMT (136).  Per byte of weights that is
// 1.5 (fp16) and 3.0 (bf16) instructions at 8 bits against 4.25 at 4 bits; per MMA, 0.7x and 1.4x of W4.
#include <type_traits>

#include "common.cuh"
#include "kernels.h"
#include "trace.cuh"
#include "wgmma.cuh"

namespace tl {

constexpr int SK_FEAT = 128;      // features per CTA tile (two warpgroups x 64 wgmma rows)
constexpr int SK_KB = 64;         // reduction elements per activation tile / MMA descriptor (one 128-byte swizzle atom)
constexpr int SK_GB = 128;        // reduction elements per pipeline step: one quantisation group, two activation tiles, 8 MMAs
constexpr int SK_PG = 2;          // group blocks per packed-weight TMA box: 128 rows x 128 B
constexpr int SK_PACKED_BYTES = SK_PG * SK_FEAT * SK_GB / 2;  // 16 KiB per box, 128-byte swizzle
constexpr int SK_CONSUMERS = 2;   // consumer warpgroups
constexpr int SK_THREADS = 128 * (1 + SK_CONSUMERS);
constexpr int SK_A_BYTES = 64 * SK_GB * 2;  // one warpgroup's dequantised block: two [64 rows x 128 B] halves, 16 KiB
constexpr int SK_ASTAGES = 2;
enum { SK_EPI_NONE = 0, SK_EPI_RESIDUAL = 1, SK_EPI_SWIGLU_PAIRS = 2 };

// Shared memory: dequantised weight blocks (SK_ASTAGES per consumer warpgroup) + activation ring (BSTAGES group blocks
// of two [NT x 64] tiles) + packed-weight ring (PSTAGES boxes) + barriers.  One CTA per SM.
template <int NT>
struct SkSmem {
    static constexpr int B_BYTES = NT * SK_KB * 2;                            // one [NT x 64] activation tile
    static constexpr int BSTAGES = NT >= 128 ? 2 : (NT >= 64 ? 3 : 4);        // group blocks in flight
    static constexpr int PSTAGES = 4;                                         // packed boxes in flight (two group blocks each)
    static constexpr int A_OFF = 0;
    static constexpr int B_OFF = A_OFF + SK_CONSUMERS * SK_ASTAGES * SK_A_BYTES;
    static constexpr int P_OFF = B_OFF + BSTAGES * 2 * B_BYTES;
    static constexpr int BAR_OFF = P_OFF + PSTAGES * SK_PACKED_BYTES;
    static constexpr int BYTES = BAR_OFF + 256;
    static_assert(BYTES <= 227 * 1024, "budget");
};

struct SkArgs {
    const void *scales, *biases, *residual;
    void *out;
    float *partials;   // [splits][M][K] fp32 (splits > 1)
    int M, N, K;       // tokens, reduction, features
    int splits, gb_per_split;  // reduction split in units of 128-wide group blocks
    int epilogue;
    // grouped (MoE) form: tile table [count, (expert, first sorted row) x count], expert segments offsets [E + 1], and
    // optionally the destination row of each sorted row
    const int32_t *tiles, *offsets, *out_index;
};

template <typename T>
struct SkNum;
template <>
struct SkNum<__nv_bfloat16> {
    using V2 = __nv_bfloat162;
    static constexpr uint32_t MAGIC = 0x43004300u;
};
template <>
struct SkNum<__half> {
    using V2 = __half2;
    static constexpr uint32_t MAGIC = 0x64006400u;
};

// GROUPED (MoE experts): the activation rows are sorted by expert; CTA row blockIdx.y is entry blockIdx.y of the tile
// table (expert e, first sorted row), its weights are rows e K + tile * 128 of the stacked [E K, N / 8] experts, rows
// past the expert's segment are computed and not stored, and CTAs past the table's count exit.  splits == 1.
template <typename T, int NT, bool GROUPED = false, int BITS = 4>
__global__ void __launch_bounds__(SK_THREADS, 1)
w4a16_skinny_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w, const SkArgs args) {
    static_assert(BITS == 4 || (BITS == 8 && !GROUPED), "8-bit codes: dense projections only");
    constexpr int PG = BITS == 4 ? SK_PG : 1;  // group blocks per packed box
    using Smem = SkSmem<NT>;
    constexpr int PSTAGES = Smem::PSTAGES;
    constexpr int BSTAGES = Smem::BSTAGES;
    extern __shared__ __align__(1024) unsigned char ssm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg_idx = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x) >> 7, 0);  // warpgroup, provably warp-uniform
    const int tile = blockIdx.x / args.splits, split = blockIdx.x - tile * args.splits;
    int m0 = blockIdx.y * NT;  // first token of this CTA
    const int G = args.N / SK_GB;  // group blocks of the whole reduction = quantisation groups per row
    const int gb0 = min(split * args.gb_per_split, G), gb1 = min(gb0 + args.gb_per_split, G);
    const int n_gb = gb1 - gb0;
    TL_TRACE_STAMP(30);
    // Programmatic dependent launch: the next kernel of the stream may become resident now (its own prologue and weight
    // pipeline do not depend on this grid).  Of THIS kernel only the activation loads and the epilogue depend on the
    // predecessor: barrier init, the packed-weight TMA ring and the dequantisers run ahead of griddep_wait(), i.e. under
    // the predecessor's tail.
    griddep_launch();
    int m_end = args.M, wrow0 = tile * SK_FEAT;  // rows stored below m_end; first packed-weight row of the tile
    if constexpr (GROUPED) {
        griddep_wait();  // the tile table is the predecessor's output, and it names the weights
        if (static_cast<int>(blockIdx.y) >= ld_cg(args.tiles)) return;
        const int e = ld_cg(args.tiles + 1 + 2 * blockIdx.y);
        m0 = ld_cg(args.tiles + 2 + 2 * blockIdx.y);
        m_end = ld_cg(args.offsets + e + 1);
        wrow0 = e * args.K + tile * SK_FEAT;
    }

    const uint32_t a_base = g_smem_u32(ssm + Smem::A_OFF), b_base = g_smem_u32(ssm + Smem::B_OFF), p_base = g_smem_u32(ssm + Smem::P_OFF);
    const uint32_t bar = g_smem_u32(ssm + Smem::BAR_OFF);
    const uint32_t p_full = bar, p_empty = p_full + 8 * PSTAGES, full_b = p_empty + 8 * PSTAGES, b_empty = full_b + 8 * BSTAGES;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < BSTAGES; ++i) {
            g_mbar_init(full_b + 8 * i, 1);
            g_mbar_init(b_empty + 8 * i, SK_CONSUMERS);  // one arrival per consumer warpgroup
        }
        for (int i = 0; i < PSTAGES; ++i) {
            g_mbar_init(p_full + 8 * i, 1);
            g_mbar_init(p_empty + 8 * i, SK_CONSUMERS * 4);  // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    TL_TRACE_STAMP(31);

    if (warp == 0) {
        // ------------------------------------------------ TMA producer: packed weights, one 128-row x 128-byte box per two group blocks
        const int n_box = (n_gb + PG - 1) / PG;
        int ps = 0;
        uint32_t ph = 1;  // producer side: the first pass through the ring does not wait
        for (int i = 0; i < n_box; ++i) {
            g_mbar_wait(p_empty + 8 * ps, ph);
            if (g_elect_one()) {
                g_mbar_expect_tx(p_full + 8 * ps, SK_PACKED_BYTES);  // columns past the row end are zero-filled and still counted
                g_tma_load_2d(p_base + ps * SK_PACKED_BYTES, &tmap_w, (gb0 + i * PG) * (SK_GB * BITS / 8), wrow0, p_full + 8 * ps);
            }
            __syncwarp();
            if (++ps == PSTAGES) ps = 0, ph ^= 1u;
        }
    } else if (warp == 1) {
        // ------------------------------------------------ TMA producer: activations, two [NT x 64] tiles per group block
        griddep_wait();  // the activations are the predecessor's output (every lane: whichever one is elected below has waited)
        int bs = 0;
        uint32_t ph = 1;
        for (int i = 0; i < n_gb; ++i) {
            g_mbar_wait(b_empty + 8 * bs, ph);
            if (g_elect_one()) {
                g_mbar_expect_tx(full_b + 8 * bs, 2 * Smem::B_BYTES);
                g_tma_load_2d(b_base + (2 * bs) * Smem::B_BYTES, &tmap_a, (gb0 + i) * SK_GB, m0, full_b + 8 * bs);
                g_tma_load_2d(b_base + (2 * bs + 1) * Smem::B_BYTES, &tmap_a, (gb0 + i) * SK_GB + SK_KB, m0, full_b + 8 * bs);
            }
            __syncwarp();
            if (++bs == BSTAGES) bs = 0, ph ^= 1u;
        }
    } else if (wg_idx >= 1) {
        // ------------------------------------------------ consumers: dequantise, MMA, epilogue
        const int wg = wg_idx - 1;           // 0 or 1: feature rows [64 wg, 64 wg + 64) of the tile
        const int t = threadIdx.x & 127;
        const int row = t >> 1, half = t & 1;     // row of this warpgroup's block, 64-wide half of the 128 reduction elements
        const int frow = wg * 64 + row;           // feature row of the tile = row of the packed box
        using V2 = typename SkNum<T>::V2;
        const uint32_t magic = SkNum<T>::MAGIC;
        const V2 offset2 = *reinterpret_cast<const V2 *>(&magic);
        const size_t srow = static_cast<size_t>(GROUPED ? wrow0 + frow : min(tile * SK_FEAT + frow, args.K - 1)) * G;
        const unsigned short *sc = reinterpret_cast<const unsigned short *>(args.scales) + srow + gb0;
        const unsigned short *bi = reinterpret_cast<const unsigned short *>(args.biases) + srow + gb0;
        const uint32_t swz = static_cast<uint32_t>(row & 7);  // == frow & 7
        const unsigned char *p_row = ssm + Smem::P_OFF + frow * 128;
        unsigned char *a_row = ssm + Smem::A_OFF + wg * SK_ASTAGES * SK_A_BYTES + half * (SK_A_BYTES / 2) + row * 128;
        const uint32_t a_wg = a_base + wg * SK_ASTAGES * SK_A_BYTES;
        float acc[NT / 2];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
        unsigned short s_next = 0, b_next = 0;
        if (n_gb > 0) s_next = __ldg(sc), b_next = __ldg(bi);
        int ps = 0, bs = 0, prev_bs = 0;
        uint32_t php = 0, phb = 0;
        for (int i = 0; i < n_gb; ++i) {
            const int s = i & 1;  // A stage
            const unsigned short s16 = s_next, b16 = b_next;
            const int nxt = min(i + 1, n_gb - 1);  // unconditional (branch-free) prefetch of the next block's pair
            s_next = __ldg(sc + nxt), b_next = __ldg(bi + nxt);
            g_mbar_wait(p_full + 8 * ps, php);
            V2 s2, b2;
            s2.x = s2.y = *reinterpret_cast<const T *>(&s16);
            b2.x = b2.y = *reinterpret_cast<const T *>(&b16);
            // row `frow` of the box: 128 bytes = 8 chunks of 16 B, chunk c stored at (c ^ (row & 7)) by the TMA swizzle;
            // group block i is bytes [64 (i % 2), + 64), this thread's half of it 32 bytes = 64 codes
            const unsigned char *src = p_row + ps * SK_PACKED_BYTES;
            uint32_t outw[32];
            if constexpr (BITS == 8) {
                // this thread's half of the group: chunks 4 half .. 4 half + 3 of the row, codes in byte order
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const uint4 v4 = *reinterpret_cast<const uint4 *>(src + (((static_cast<uint32_t>(4 * half + c)) ^ swz) << 4));
                    const uint32_t wv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        if constexpr (std::is_same<T, __half>::value) {
#pragma unroll
                            for (int q = 0; q < 2; ++q) {
                                uint32_t bits = __byte_perm(wv[j], 0x64646464u, q == 0 ? 0x4140 : 0x4342);  // (1024 + c_2q, 1024 + c_2q+1)
                                V2 code = __hsub2(*reinterpret_cast<V2 *>(&bits), offset2);
                                V2 v = __hfma2(code, s2, b2);
                                outw[8 * c + 2 * j + q] = *reinterpret_cast<uint32_t *>(&v);
                            }
                        } else {
                            uint32_t f[4];
#pragma unroll
                            for (int q = 0; q < 4; ++q) f[q] = __float_as_uint(__uint_as_float(__byte_perm(wv[j], 0x4B000000u, 0x7440 | q)) - 8388608.f);
#pragma unroll
                            for (int q = 0; q < 2; ++q) {
                                uint32_t bits = __byte_perm(f[2 * q], f[2 * q + 1], 0x7632);  // (c_2q, c_2q+1) in bf16
                                V2 v = __hfma2(*reinterpret_cast<V2 *>(&bits), s2, b2);
                                outw[8 * c + 2 * j + q] = *reinterpret_cast<uint32_t *>(&v);
                            }
                        }
                    }
                }
            } else {
                const uint32_t c0 = static_cast<uint32_t>(4 * (i & 1) + 2 * half);
                const uint4 lo = *reinterpret_cast<const uint4 *>(src + ((c0 ^ swz) << 4));
                const uint4 hi = *reinterpret_cast<const uint4 *>(src + (((c0 + 1) ^ swz) << 4));
                const uint32_t wv[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    uint32_t p[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        uint32_t bits;  // (128 + code_q, 128 + code_{q+4}) in one LOP3: ((w >> 4q) & 0x000F000F) | magic
                        asm("lop3.b32 %0, %1, 0x000F000F, %2, 0xEA;" : "=r"(bits) : "r"(wv[j] >> (4 * q)), "r"(magic));
                        V2 code = __hsub2(*reinterpret_cast<V2 *>(&bits), offset2);
                        V2 v = __hfma2(code, s2, b2);                                   // code * scale + bias, one rounding
                        p[q] = *reinterpret_cast<uint32_t *>(&v);
                    }
                    outw[4 * j + 0] = __byte_perm(p[0], p[1], 0x5410);  // (e0, e1)
                    outw[4 * j + 1] = __byte_perm(p[2], p[3], 0x5410);  // (e2, e3)
                    outw[4 * j + 2] = __byte_perm(p[0], p[1], 0x7632);  // (e4, e5)
                    outw[4 * j + 3] = __byte_perm(p[2], p[3], 0x7632);  // (e6, e7)
                }
            }
            // The box is released only now: the arithmetic above consumed the loaded words, so this warp's
            // shared-memory reads of the box have completed (mbarrier operations are not ordered behind loads).
            __syncwarp();
            g_mbar_arrive_if(p_empty + 8 * ps, lane == 0 && (PG == 1 || (i & 1) || i + 1 == n_gb));
            // A stage s was last read by the MMAs of block i - 2, complete since wgmma_wait<1> of block i - 1
            unsigned char *dst = a_row + s * SK_A_BYTES;
#pragma unroll
            for (int c = 0; c < 8; ++c)
                *reinterpret_cast<uint4 *>(dst + ((static_cast<uint32_t>(c) ^ swz) << 4)) =
                    make_uint4(outw[4 * c], outw[4 * c + 1], outw[4 * c + 2], outw[4 * c + 3]);
            g_fence_proxy_async();        // generic-proxy stores -> visible to the tensor core's async proxy
            g_named_sync(1 + wg, 128);    // the whole 64-row block is written
            g_mbar_wait(full_b + 8 * bs, phb);
            wgmma_reg_fence(acc);
            wgmma_fence();
            {
                const uint32_t ab = a_wg + s * SK_A_BYTES, bb = b_base + (2 * bs) * Smem::B_BYTES;
#pragma unroll
                for (int k = 0; k < SK_GB / 16; ++k)
                    Wgmma<T, NT>::ss(acc, g_wgmma_desc(ab + (k >> 2) * (SK_A_BYTES / 2) + 32 * (k & 3), 16, 1024),
                                     g_wgmma_desc(bb + (k >> 2) * Smem::B_BYTES + 32 * (k & 3), 16, 1024), 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the MMAs of block i - 1 have completed: their activation stage goes back to the producer
            wgmma_reg_fence(acc);
            g_mbar_arrive_if(b_empty + 8 * prev_bs, i > 0 && t == 0);
            prev_bs = bs;
            if (PG == 1 || (i & 1) || i + 1 == n_gb)
                if (++ps == PSTAGES) ps = 0, php ^= 1u;
            if (++bs == BSTAGES) bs = 0, phb ^= 1u;
        }
        wgmma_wait<0>();
        wgmma_reg_fence(acc);
        TL_TRACE_STAMP_T(34, 128);  // accumulators complete
        // the epilogue reads the residual and overwrites buffers (output, partial planes) that the predecessor - the
        // reduction kernel of the previous projection - may still be reading
        griddep_wait();
        // ---- epilogue: acc[4 j + 2 r + c] = D[feature f0 + 8 r, token 8 j + 2 (t % 4) + c]
        const int f0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int n0 = tile * SK_FEAT + f0;
        const int mq = m0 + 2 * (lane & 3);
        const size_t plane = static_cast<size_t>(args.M) * args.K;
        if (args.splits > 1) {
            // park the fp32 partial tile; w4a16_skinny_reduce_kernel adds the planes in split order
            float *part = args.partials + split * plane;
#pragma unroll
            for (int i = 0; i < NT / 2; ++i) {
                const int m = mq + 8 * (i >> 2) + (i & 1), n = n0 + 8 * ((i >> 1) & 1);
                if (m < args.M && n < args.K) part[static_cast<size_t>(m) * args.K + n] = acc[i];
            }
        } else if (args.epilogue == SK_EPI_SWIGLU_PAIRS) {
            // rows 16j + r (gate) and 16j + 8 + r (up) of the interleaved weight -> activation 8j + r: f0 is a gate row
            // (f0 % 16 < 8) and this thread also holds its up row f0 + 8
            T *out = static_cast<T *>(args.out);
            const int feat = (n0 >> 4) * 8 + (n0 & 7);
#pragma unroll
            for (int i = 0; i < NT / 2; i += 4)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int m = mq + 8 * (i >> 2) + c;
                    const float gate = to_f(from_f<T>(acc[i + c])), up = to_f(from_f<T>(acc[i + 2 + c]));
                    if (m < m_end && n0 < args.K) {
                        const int orow = GROUPED && args.out_index != nullptr ? ld_cg(args.out_index + m) : m;
                        out[static_cast<size_t>(orow) * (args.K / 2) + feat] = from_f<T>((gate / (1.0f + expf(-gate))) * up);
                    }
                }
        } else {
            T *out = static_cast<T *>(args.out);
            const T *res = static_cast<const T *>(args.residual);
#pragma unroll
            for (int i = 0; i < NT / 2; ++i) {
                const int m = mq + 8 * (i >> 2) + (i & 1), n = n0 + 8 * ((i >> 1) & 1);
                if (m < m_end && n < args.K) {
                    T vb = from_f<T>(acc[i]);
                    if (args.epilogue == SK_EPI_RESIDUAL) vb = from_f<T>(to_f(ld_cg(res + static_cast<size_t>(m) * args.K + n)) + to_f(vb));
                    const int orow = GROUPED && args.out_index != nullptr ? ld_cg(args.out_index + m) : m;
                    out[static_cast<size_t>(orow) * args.K + n] = vb;
                }
            }
        }
    }
    TL_TRACE_STAMP(36);
}

#if TL_TRACE
void trace_bind_skinny(unsigned long long *buf, unsigned int *n, unsigned int cap) { trace_bind(buf, n, cap); }
#endif

// Adds the fp32 partial planes of a split reduction in split order (deterministic: same bits on every run and for
// every CTA schedule) and applies the epilogue; one thread per output.  All `splits` loads of a thread are independent
// and in flight together (letting the last CTA of a tile do this costs a chain of dependent round trips).
template <typename T>
__global__ void __launch_bounds__(256) w4a16_skinny_reduce_kernel(const float *part, const T *res, T *out, int M, int K, int splits, int epilogue) {
    const size_t plane = static_cast<size_t>(M) * K;
    griddep_launch();
    griddep_wait();  // the planes are the GEMM's output; they are rewritten by every projection, so read them through L2
    // four planes per round trip, added in split order
    auto plane_sum = [&](size_t at) {
        float sum = 0.f;
        for (int sp0 = 0; sp0 < splits; sp0 += 4) {
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = sp0 + j < splits ? ld_cg(part + (sp0 + j) * plane + at) : 0.f;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (sp0 + j < splits) sum += v[j];
        }
        return sum;
    };
    if (epilogue == SK_EPI_SWIGLU_PAIRS) {
        const int half = K / 2;
        const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
        if (idx >= static_cast<size_t>(M) * half) return;
        const int m = static_cast<int>(idx / half), feat = static_cast<int>(idx - static_cast<size_t>(m) * half);
        const int n_gate = (feat >> 3) * 16 + (feat & 7);  // rows 16j + r (gate) and 16j + 8 + r (up) -> activation 8j + r
        const float g = plane_sum(static_cast<size_t>(m) * K + n_gate), u = plane_sum(static_cast<size_t>(m) * K + n_gate + 8);
        const float gate = to_f(from_f<T>(g)), up = to_f(from_f<T>(u));
        out[idx] = from_f<T>((gate / (1.0f + expf(-gate))) * up);
        return;
    }
    const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= plane) return;
    T vb = from_f<T>(plane_sum(idx));
    if (epilogue == SK_EPI_RESIDUAL) vb = from_f<T>(to_f(ld_cg(res + idx)) + to_f(vb));
    out[idx] = vb;
}

// The same reduction for the residual epilogue when the RMSNorm of the NEXT projection follows (o -> post-attention norm,
// down -> next layer's input norm): one CTA per token row adds the planes, adds the residual, writes the residual
// stream and - the row being complete in its registers - the normalised row too (week2_kernels.metal:41-47 arithmetic:
// T(x * rsqrt(mean(x^2) + eps) * w) on the ROUNDED residual sum).  Saves the rms_norm launch and its read of the row.
constexpr int SK_NORM_PER = 16;  // elements per thread: K <= 4096
template <typename T>
__global__ void __launch_bounds__(256) w4a16_skinny_reduce_norm_kernel(const float *part, const T *res, const T *__restrict__ norm_w, T *out, T *normed,
                                                                       int M, int K, int splits, float eps) {
    __shared__ float warp_part[8];
    griddep_launch();
    griddep_wait();
    const size_t plane = static_cast<size_t>(M) * K, row = static_cast<size_t>(blockIdx.x) * K;
    // all loads of a round (four planes x the thread's elements, then the residual) are issued before the first is used:
    // ld_cg is a volatile asm, so a load-then-add loop per element would pay one L2 round trip per batch
    float xs[SK_NORM_PER];
#pragma unroll
    for (int j = 0; j < SK_NORM_PER; ++j) xs[j] = 0.f;
    for (int sp0 = 0; sp0 < splits; sp0 += 4) {
        float v[SK_NORM_PER][4];
#pragma unroll
        for (int j = 0; j < SK_NORM_PER; ++j) {
            const int n = threadIdx.x + j * 256;
#pragma unroll
            for (int q = 0; q < 4; ++q) v[j][q] = (n < K && sp0 + q < splits) ? ld_cg(part + (sp0 + q) * plane + row + n) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < SK_NORM_PER; ++j) {
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (sp0 + q < splits) xs[j] += v[j][q];  // split order
        }
    }
    T rs[SK_NORM_PER];
#pragma unroll
    for (int j = 0; j < SK_NORM_PER; ++j) {
        const int n = threadIdx.x + j * 256;
        rs[j] = n < K ? ld_cg(res + row + n) : from_f<T>(0.f);
    }
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < SK_NORM_PER; ++j) {
        const int n = threadIdx.x + j * 256;
        if (n < K) {
            const T vb = from_f<T>(to_f(rs[j]) + to_f(from_f<T>(xs[j])));
            out[row + n] = vb;
            xs[j] = to_f(vb);
            ss += xs[j] * xs[j];
        }
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = ss;
    __syncthreads();
    ss = warp_sum((threadIdx.x & 31) < 8 ? warp_part[threadIdx.x & 31] : 0.f);
    const float inv = rsqrtf(ss / static_cast<float>(K) + eps);
#pragma unroll
    for (int j = 0; j < SK_NORM_PER; ++j) {
        const int n = threadIdx.x + j * 256;
        if (n < K) normed[row + n] = from_f<T>(xs[j] * inv * to_f(norm_w[n]));
    }
}

// ---------------------------------------------------------------- host side --
// Split policy (ours; the reference's constants are M4-Pro tuning, quantized_matmul.cpp:138-150): the split count that
// minimises waves x (group blocks per CTA + fixed cost) + reduce launch, with `slots` CTAs resident at once (one per
// SM), a fixed cost per CTA worth ~10 group blocks (barrier set-up, first TMA round trips, epilogue) and ~8 for the
// extra reduce launch.
static int skinny_slots(int) { return sm_count(); }
int w4a16_skinny_splits(int M, int N, int K, int *gb_per_split) {
    const int tiles = (K + SK_FEAT - 1) / SK_FEAT;
    const int num_gb = N / SK_GB;
    const int slots = skinny_slots(M);
    int best = 1;
    long long best_cost = -1;
    for (int s = 1; s <= 16 && s <= num_gb / 2 + (num_gb < 2); ++s) {
        const int gbps = (num_gb + s - 1) / s;
        const int real = (num_gb + gbps - 1) / gbps;  // splits that actually get blocks
        const long long waves = (static_cast<long long>(tiles) * real + slots - 1) / slots;
        const long long cost = waves * (gbps + 10) + (real > 1 ? 8 : 0);  // in units of one group block
        if (best_cost < 0 || cost < best_cost) best_cost = cost, best = real;
    }
    if (gb_per_split != nullptr) *gb_per_split = (num_gb + best - 1) / best;
    return best;
}

size_t w4a16_skinny_workspace(int M, int N, int K) {
    const int splits = w4a16_skinny_splits(M, N, K);
    return splits > 1 ? static_cast<size_t>(splits) * M * K * sizeof(float) : 0;
}

// Tensor maps of the activations a [M, N] (16-bit, [nt tokens x 64] boxes) and of the packed weights b [K, N * bits / 8]
// (bytes, 128 rows x 128-byte boxes), both with the 128-byte swizzle wgmma reads.
template <typename T>
static int sk_maps(CUtensorMap *ma, CUtensorMap *mw, const void *a, const void *b, int M, int N, int K, int nt, int bits = 4) {
    const CUtensorMapDataType dt = std::is_same<T, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const cuuint64_t a_dims[2] = {static_cast<cuuint64_t>(N), static_cast<cuuint64_t>(M)};
    const cuuint32_t a_box[2] = {SK_KB, static_cast<cuuint32_t>(nt)};
    const cuuint64_t w_dims[2] = {static_cast<cuuint64_t>(N) * bits / 8, static_cast<cuuint64_t>(K)};
    const cuuint32_t w_box[2] = {SK_PG * SK_GB / 2, SK_FEAT};
    if (int e = cached_tensor_map(ma, a, dt, 2, a_dims, a_box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, "quantized_matmul"))
        return e;
    return cached_tensor_map(mw, b, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, w_dims, w_box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                             "quantized_matmul");
}

template <typename T, int NT, bool GROUPED = false, int BITS = 4>
static int skinny_launch(const CUtensorMap &ma, const CUtensorMap &mw, const SkArgs &args, dim3 grid, cudaStream_t st) {
    constexpr size_t smem = SkSmem<NT>::BYTES;
    auto *kernel = w4a16_skinny_kernel<T, NT, GROUPED, BITS>;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) != cudaSuccess ||
            cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess)
            return fail(TL_ECUDA, "quantized_matmul: cannot raise shared memory limit");
        configured = true;
    }
    cudaError_t e = launch_chained(kernel, grid, dim3(SK_THREADS), smem, st, ma, mw, args);
    if (e != cudaSuccess) return fail(TL_ECUDA, "w4a16_skinny: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("w4a16_skinny");
    return TL_OK;
}

template <typename T>
static int skinny_t(const void *scales, const void *biases, const void *a, const void *b, void *out, const void *residual, int M, int N, int K,
                    int epilogue, void *ws, size_t ws_bytes, const void *norm_w, float norm_eps, void *normed, bool *norm_done, cudaStream_t st,
                    int *planes_out, int bits) {
    if (!aligned16(a) || !aligned16(b)) return fail(TL_EINVAL, "quantized_matmul: a and b must be 16-byte aligned");
    const int NT = M <= 16 ? 16 : (M <= 32 ? 32 : (M <= 64 ? 64 : 128));
    const int tiles = (K + SK_FEAT - 1) / SK_FEAT;
    SkArgs args{};
    args.scales = scales, args.biases = biases, args.residual = residual, args.out = out;
    args.M = M, args.N = N, args.K = K, args.epilogue = epilogue;
    args.splits = w4a16_skinny_splits(M, N, K, &args.gb_per_split);
    if (args.splits > 1 && (ws == nullptr || ws_bytes < w4a16_skinny_workspace(M, N, K)))
        return fail(TL_EWORKSPACE, "quantized_matmul: workspace too small (%zu < %zu)", ws_bytes, w4a16_skinny_workspace(M, N, K));
    args.partials = static_cast<float *>(ws);
    CUtensorMap ma, mw;
    if (int e = sk_maps<T>(&ma, &mw, a, b, M, N, K, NT, bits)) return e;
    const dim3 grid(tiles * args.splits);
    int rc;
    if (bits == 8) {
        switch (NT) {
            case 16: rc = skinny_launch<T, 16, false, 8>(ma, mw, args, grid, st); break;
            case 32: rc = skinny_launch<T, 32, false, 8>(ma, mw, args, grid, st); break;
            case 64: rc = skinny_launch<T, 64, false, 8>(ma, mw, args, grid, st); break;
            default: rc = skinny_launch<T, 128, false, 8>(ma, mw, args, grid, st); break;
        }
    } else {
        switch (NT) {
            case 16: rc = skinny_launch<T, 16>(ma, mw, args, grid, st); break;
            case 32: rc = skinny_launch<T, 32>(ma, mw, args, grid, st); break;
            case 64: rc = skinny_launch<T, 64>(ma, mw, args, grid, st); break;
            default: rc = skinny_launch<T, 128>(ma, mw, args, grid, st); break;
        }
    }
    if (planes_out != nullptr) {  // the caller adds the planes itself (fused consumer); 1 = `out` holds the finished result
        *planes_out = args.splits;
        if (args.splits > 1) return rc;
    }
    if (rc != TL_OK || args.splits == 1) return rc;
    if (normed != nullptr && epilogue == SK_EPI_RESIDUAL && K <= 256 * SK_NORM_PER) {
        cudaError_t e = launch_chained(w4a16_skinny_reduce_norm_kernel<T>, dim3(M), dim3(256), 0, st, static_cast<const float *>(args.partials),
                                       static_cast<const T *>(residual), static_cast<const T *>(norm_w), static_cast<T *>(out), static_cast<T *>(normed),
                                       M, K, args.splits, norm_eps);
        if (e != cudaSuccess) return fail(TL_ECUDA, "w4a16_skinny_reduce_norm: launch failed: %s", cudaGetErrorString(e));
        TL_LAUNCH_CHECK("w4a16_skinny_reduce_norm");
        *norm_done = true;
        return TL_OK;
    }
    const size_t outputs = static_cast<size_t>(M) * (epilogue == SK_EPI_SWIGLU_PAIRS ? K / 2 : K);
    cudaError_t e = launch_chained(w4a16_skinny_reduce_kernel<T>, dim3(static_cast<unsigned>((outputs + 255) / 256)), dim3(256), 0, st,
                                   static_cast<const float *>(args.partials), static_cast<const T *>(residual), static_cast<T *>(out), M, K,
                                   args.splits, epilogue);
    if (e != cudaSuccess) return fail(TL_ECUDA, "w4a16_skinny_reduce: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("w4a16_skinny_reduce");
    return TL_OK;
}

int launch_w4a16_skinny(const void *scales, const void *biases, const void *a, const void *b, void *out, const void *residual, int M, int N,
                        int K, int epilogue, int dtype, void *ws, size_t ws_bytes, cudaStream_t st, const void *norm_w, float norm_eps, void *normed,
                        bool *norm_done, int *planes_out, int bits) {
    bool unused = false;
    if (norm_done == nullptr) norm_done = &unused;
    *norm_done = false;
    if (M == 0 || K == 0) return TL_OK;
    if (epilogue == SK_EPI_SWIGLU_PAIRS && K % 16 != 0) return fail(TL_EINVAL, "quantized_matmul: interleaved gate|up rows need K %% 16 == 0");
    if (dtype == TL_BF16)
        return skinny_t<__nv_bfloat16>(scales, biases, a, b, out, residual, M, N, K, epilogue, ws, ws_bytes, norm_w, norm_eps, normed, norm_done, st,
                                       planes_out, bits);
    if (dtype == TL_F16)
        return skinny_t<__half>(scales, biases, a, b, out, residual, M, N, K, epilogue, ws, ws_bytes, norm_w, norm_eps, normed, norm_done, st, planes_out,
                                bits);
    return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
}

// Prefill GEMM (any M): 128-token tiles along grid.y, the whole reduction per CTA, the epilogue in the kernel.
template <typename T>
static int tiles_t(const void *scales, const void *biases, const void *a, const void *b, void *out, int M, int N, int K, cudaStream_t st, int bits) {
    if (!aligned16(a) || !aligned16(b)) return fail(TL_EINVAL, "quantized_matmul: a and b must be 16-byte aligned");
    SkArgs args{};
    args.scales = scales, args.biases = biases, args.out = out;
    args.M = M, args.N = N, args.K = K, args.epilogue = SK_EPI_NONE;
    args.splits = 1, args.gb_per_split = N / SK_GB;
    CUtensorMap ma, mw;
    if (int e = sk_maps<T>(&ma, &mw, a, b, M, N, K, 128, bits)) return e;
    const dim3 grid((K + SK_FEAT - 1) / SK_FEAT, (M + 127) / 128);
    if (grid.y > 65535) return fail(TL_EINVAL, "quantized_matmul: too many rows for one launch");
    return bits == 8 ? skinny_launch<T, 128, false, 8>(ma, mw, args, grid, st) : skinny_launch<T, 128>(ma, mw, args, grid, st);
}

int launch_w4a16_tiles(const void *scales, const void *biases, const void *a, const void *b, void *out, int M, int N, int K, int dtype,
                       cudaStream_t st, int bits) {
    if (M == 0 || K == 0) return TL_OK;
    if (dtype == TL_BF16) return tiles_t<__nv_bfloat16>(scales, biases, a, b, out, M, N, K, st, bits);
    if (dtype == TL_F16) return tiles_t<__half>(scales, biases, a, b, out, M, N, K, st, bits);
    return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
}

// Grouped expert GEMM (MoE): R expert-sorted rows of a [R, N], E experts of K output features stacked in b [E K, N / 8],
// NT-row tiles listed by tl_moe_group, max_tiles CTA rows of which the table's count run.
template <typename T>
static int grouped_t(const void *scales, const void *biases, const void *a, const void *b, void *out, const int32_t *offsets, const int32_t *tiles,
                     const int32_t *out_index, int R, int E, int N, int K, int epilogue, int nt, int max_tiles, cudaStream_t st) {
    SkArgs args{};
    args.scales = scales, args.biases = biases, args.out = out;
    args.M = R, args.N = N, args.K = K, args.epilogue = epilogue;
    args.splits = 1, args.gb_per_split = N / SK_GB;
    args.tiles = tiles, args.offsets = offsets, args.out_index = out_index;
    CUtensorMap ma, mw;
    if (int e = sk_maps<T>(&ma, &mw, a, b, R, N, E * K, nt)) return e;
    const dim3 grid(K / SK_FEAT, max_tiles);
    switch (nt) {
        case 16: return skinny_launch<T, 16, true>(ma, mw, args, grid, st);
        case 32: return skinny_launch<T, 32, true>(ma, mw, args, grid, st);
        case 64: return skinny_launch<T, 64, true>(ma, mw, args, grid, st);
        default: return skinny_launch<T, 128, true>(ma, mw, args, grid, st);
    }
}

int launch_w4a16_grouped(const void *scales, const void *biases, const void *a, const void *b, void *out, const int32_t *offsets, const int32_t *tiles,
                         const int32_t *out_index, int R, int E, int N, int K, int epilogue, int nt, int max_tiles, int dtype, cudaStream_t st) {
    if (R == 0 || K == 0) return TL_OK;
    if (dtype == TL_BF16)
        return grouped_t<__nv_bfloat16>(scales, biases, a, b, out, offsets, tiles, out_index, R, E, N, K, epilogue, nt, max_tiles, st);
    if (dtype == TL_F16) return grouped_t<__half>(scales, biases, a, b, out, offsets, tiles, out_index, R, E, N, K, epilogue, nt, max_tiles, st);
    return fail(TL_EDTYPE, "moe_grouped_matmul: scales must be float16 or bfloat16");
}

}  // namespace tl
