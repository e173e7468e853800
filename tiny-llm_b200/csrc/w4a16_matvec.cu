// W4A16 (4-bit codes, group 128, affine) weight-streaming kernels.
//
//   out[m, k] = sum_n a[m, n] * (code[k, n] * scale[k, n/128] + bias[k, n/128])
//
// a [M, N] (bf16|f16), b [K, N/8] packed u32 (code i of a word = (w >> 4i) & 15,
// src/tiny_llm_ref/quantize.py:113-115), scales/biases [K, N/128].
//
// w4a16_stream5_kernel is the decode kernel (reference: quantized_matvec_x4_fast,
// src/extensions_ref/src/quantized_matmul.metal:441-538): every packed
// weight byte is read exactly once with 128-bit loads that bypass L1; activations (tiny,
// shared by every CTA) are staged once per CTA in shared memory.  The per-weight ALU work
// would exceed the HBM time on CUDA cores (~3 ops/weight), so the 16 x 128 code tile of
// each warp is fed to the tensor cores as an exact small-integer bf16 operand (details and
// the instruction budget: w4a16_item.cuh), with the Metal kernel's "scale * qdot +
// bias * asum" factorisation (:515-521) applied once per 128-wide group in fp32.
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"
#include "w4a16_item.cuh"
#include "trace.cuh"

namespace tl {

// ---------------------------------------------------------------------------
// v5: register-pipelined streaming, contiguous rows per CTA (see w4a16_item.cuh for the
// instruction budget of the inner loop).
//
// Earlier forms - register prefetch, a producer warp with a cp.async.bulk ring, per-warp cp.async rings - were
// instruction-issue bound; fixed-size 16-row tiles dealt to warp teams left a tail of teams working twice as long.
// v5 gives CTA c the contiguous rows of chunks [C*c/grid, C*(c+1)/grid) (C = K/16 chunks, all
// CTAs within one chunk of each other) and deals the CTA's (chunk, unit) pairs to its warps as
// equal contiguous ranges.  A warp accumulates a chunk in registers and parks the partial sums in
// shared-memory entry (chunk + warp); after ONE block barrier the entries of every chunk are summed
// in warp order (deterministic), the residual (prefetched before the stream starts) is added and
// the outputs are stored.
//
// Weights never depend on the previous kernel: each warp requests its first units BEFORE
// griddepcontrol.wait, so with programmatic dependent launch the HBM stream of kernel n+1
// starts while kernel n drains.
//
// Optional fusions that keep every rounding point of the unfused call sequence
// (so results match rms_norm -> matvec, swiglu -> matvec, matvec -> add):
//   prologue RMSNORM : a = T(x * rsqrt(mean(x^2)+eps) * w)   (week2_kernels.metal:41-47)
//   prologue SWIGLU  : a = T(g / (1 + exp(-g)) * u)          (week2_kernels.metal:115-116)
//   epilogue RESIDUAL: out = T(float(res) + float(T(acc)))   (qwen3_week3.py:204-206)
//   epilogue SWIGLU_PAIRS: rows 16c+r / 16c+8+r hold gate / up feature 8c+r;
//                     out[m, 8c+r] = T(silu(T(acc_gate)) * T(acc_up))  (week2_kernels.metal:115-116)
// Experiments that did not pay and were removed again:
//   * 8-warp CTAs, two per SM, one from each of two consecutive launches (so that launch n+1 prefetches while launch n
//     consumes): the consume phase is issue-bound, and half the warps per launch made it slower;
//   * a device-flag hand-off between dependent launches instead of griddepcontrol.wait (the CTAs of the consumer
//     cannot start before the producer's CTAs exit anyway, the flag traffic only adds);
//   * forcing the largest shared-memory carveout: the register pipeline keeps up to 128 KiB of weight loads in flight per
//     SM and those loads are staged in L1 lines even with L1::no_allocate - with ~1 KiB of L1 left every projection
//     slowed down.  No carveout preference is set here;
//   * moving the weight stream from registers to per-warp TMA rings in shared memory (512-thread CTAs at 64 registers,
//     two per SM): correct, but the consume phase pays a shared-memory read per weight word and twice the CTAs hand
//     over more slowly;
//   * asking the CTA's whole weight slice into L2 (cp.async.bulk.prefetch.L2) before griddepcontrol.wait: the prefetch
//     traffic competes with the activation round trip of the staging step;
//   * a lookahead: each CTA, once its own units were requested, asking L2 (cp.async.bulk.prefetch.L2 for the weight
//     rows, prefetch.global.L2 for scales and biases) for the slice the same CTA index of the NEXT projection streams.
//     Decode lost 5-9 % at every placement and cap tried (DESIGN.md section 4): q|k|v, o and down already have
//     (almost) all of their units in flight before the dependency wait, so the extra requests only lengthen the
//     consume phase, and the next launch's griddepcontrol.wait waits for this grid to complete.
constexpr int S5_WARPS = 16;
// Units per warp in flight for up to 8 rows.  3 (96 KiB per SM) keeps the kernel free of register spills; 4 spilled
// 24-48 bytes per thread and 4, 5, 6 were each slower on H100 (DESIGN.md section 4).
#ifndef S5_DEPTH_SMALL
#define S5_DEPTH_SMALL 3
#endif
enum { PRO_NONE = W4_PRO_NONE, PRO_RMSNORM = W4_PRO_RMSNORM, PRO_SWIGLU = W4_PRO_SWIGLU };
enum { EPI_NONE = 0, EPI_RESIDUAL = 1, EPI_SWIGLU_PAIRS = 2 };

struct StreamArgs {
    const void *scales, *biases;
    const uint32_t *b;
    void *out;
    const void *p0, *p1, *residual;
    int M, N, K, lda;
    int prologue, epilogue;
    float eps;
    int rows_per_pass;
};


// MP: activation rows per pass padded to a power of two (template: shared-memory offsets of the
// B fragments become immediates).  U: 128-column groups per unit (2 when N % 256 == 0).
template <typename T, int MP, int U>
__global__ void __launch_bounds__(S5_WARPS * 32, 1) w4a16_stream5_kernel(const StreamArgs args) {
    constexpr int NW = S5_WARPS;
    constexpr int NT = NW * 32;
    constexpr int MT = (MP + 7) / 8;
    constexpr int MPA = w4_mpa(MP);
    constexpr int DEPTH = (MP <= 8 ? S5_DEPTH_SMALL : (MP == 16 ? 3 : 2));  // units per warp in the register pipeline
    constexpr int ENTRY = 16 * 8 * MT;                                      // floats per (chunk, warp) partial sum
    extern __shared__ __align__(128) unsigned char smem5_raw[];
    __shared__ int warp_begin[NW + 1];
    const int N = args.N, K = args.K;
    const int pass = blockIdx.y;
    const int Mp = min(args.rows_per_pass, args.M - pass * args.rows_per_pass);
    const int words = N / 8;
    const int G = N / 128;
    const int P = G / U;  // units per chunk
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;

    // shared layout: act [words*MP] x 16 B | asum [G*MPA] | entries [(chunks + warps)][16][8*MT]
    // (the head of `entries` doubles as the sum-of-squares scratch of the staging step)
    uint4 *act = reinterpret_cast<uint4 *>(smem5_raw);
    float *asum = reinterpret_cast<float *>(smem5_raw + static_cast<size_t>(words) * MP * 16);
    float *entries = asum + G * MPA;

    griddep_launch();
    TL_TRACE_STAMP(10);

    // ---- rows of this CTA (whole 16-row chunks) and units of this warp
    const unsigned all = static_cast<unsigned>(K + 15) >> 4;  // all * gridDim.x < 2^31 (K < 2^24 rows)
    const int c0 = static_cast<int>(all * blockIdx.x / gridDim.x), c1 = static_cast<int>(all * (blockIdx.x + 1) / gridDim.x);
    const int chunks = c1 - c0;
    const int r0 = c0 * 16, r1 = min(K, c1 * 16);
    const unsigned units = static_cast<unsigned>(chunks) * P;
    const int begin = static_cast<int>(units * warp / NW), end = static_cast<int>(units * (warp + 1) / NW);
    if (threadIdx.x <= NW) warp_begin[threadIdx.x] = static_cast<int>(units * threadIdx.x / NW);

    // ---- load cursor (runs DEPTH units ahead of the consumer)
    const unsigned char *bbytes = reinterpret_cast<const unsigned char *>(args.b);
    const unsigned char *sbtable = reinterpret_cast<const unsigned char *>(lane < 16 ? args.scales : args.biases);
    const size_t row_bytes = static_cast<size_t>(N) / 2;
    const unsigned char *l_p0, *l_p8, *l_sb;
    int l_i = begin, l_chunk = begin / P;
    int l_u = begin - l_chunk * P;
    auto chunk_ptrs = [&]() {  // rows past K are clamped: loaded, multiplied, never stored
        const int base = r0 + l_chunk * 16;
        const int q0 = min(base + g, K - 1), q8 = min(base + g + 8, K - 1), qs = min(base + (lane & 15), K - 1);
        l_p0 = bbytes + q0 * row_bytes + l_u * (U * 64) + t * 16;
        l_p8 = bbytes + q8 * row_bytes + l_u * (U * 64) + t * 16;
        l_sb = sbtable + (static_cast<size_t>(qs) * G + l_u * U) * 2;
    };
    chunk_ptrs();
    auto load_next = [&](W4Unit<U> &un) {
        if (l_i < end) {
            w4_load<U>(un, l_p0, l_p8, l_sb);
            l_i += 1;
            if (++l_u == P) {
                l_u = 0;
                l_chunk += 1;
                chunk_ptrs();
            } else {
                l_p0 += U * 64;
                l_p8 += U * 64;
                l_sb += U * 2;
            }
        }
    };
    W4Unit<U> buf[DEPTH];
#pragma unroll
    for (int k = 0; k < DEPTH; ++k) load_next(buf[k]);  // in flight before the activations exist
    TL_TRACE_STAMP(11);

    griddep_wait();  // activations (and the residual) come from the previous kernel
    TL_TRACE_STAMP(12);
    const T *p0 = static_cast<const T *>(args.p0) + static_cast<size_t>(pass) * args.rows_per_pass * args.lda;
    const T *p1 = args.prologue == PRO_SWIGLU
                      ? static_cast<const T *>(args.p1) + static_cast<size_t>(pass) * args.rows_per_pass * args.lda
                      : static_cast<const T *>(args.p1);
    T *out = static_cast<T *>(args.out) + static_cast<size_t>(pass) * args.rows_per_pass * (args.epilogue == EPI_SWIGLU_PAIRS ? K / 2 : K);
    const T *res = args.epilogue == EPI_RESIDUAL ? static_cast<const T *>(args.residual) + static_cast<size_t>(pass) * args.rows_per_pass * K
                                                 : nullptr;
    // the residual of this thread's first output: requested now, needed after the stream
    const int outs = chunks * 16 * Mp;
    float res_first = 0.f;
    if (res != nullptr && static_cast<int>(threadIdx.x) < outs) {
        const int m = threadIdx.x / (chunks * 16), rr = threadIdx.x - m * (chunks * 16);
        if (r0 + rr < r1) res_first = to_f(res[static_cast<size_t>(m) * K + r0 + rr]);
    }
    w4_stage<T, MP, NT>(p0, args.lda, p1, args.prologue, N, Mp, args.eps, act, asum, entries);
    TL_TRACE_STAMP(13);

    const uint4 *act0 = w4_act_lane<MP>(act, g, t);
    const float *asum0 = w4_asum_lane<MP>(asum, t);
    int chunk = begin / P;
    int u = begin - chunk * P;
    const uint4 *actp = act0 + u * U * w4_act_group_stride<MP>();
    const float *asump = asum0 + u * U * w4_asum_group_stride<MP>();
    float acc[MT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) acc[mt][0] = acc[mt][1] = acc[mt][2] = acc[mt][3] = 0.f;
    auto flush = [&]() {  // park this warp's partial sums of `chunk` in entry (chunk + warp)
        float *e = entries + static_cast<size_t>(chunk + warp) * ENTRY;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
            e[g * 8 * MT + mt * 8 + 2 * t] = acc[mt][0];
            e[g * 8 * MT + mt * 8 + 2 * t + 1] = acc[mt][1];
            e[(g + 8) * 8 * MT + mt * 8 + 2 * t] = acc[mt][2];
            e[(g + 8) * 8 * MT + mt * 8 + 2 * t + 1] = acc[mt][3];
            acc[mt][0] = acc[mt][1] = acc[mt][2] = acc[mt][3] = 0.f;
        }
    };
    for (int i = begin; i < end; i += DEPTH) {
#pragma unroll
        for (int k = 0; k < DEPTH; ++k) {
            if (i + k < end) {  // warp-uniform; k is a compile-time register index
                w4_consume<T, MP, U>(buf[k], actp, asump, g, acc);
                load_next(buf[k]);
                actp += U * w4_act_group_stride<MP>();
                asump += U * w4_asum_group_stride<MP>();
                if (++u == P) {
                    flush();
                    u = 0;
                    chunk += 1;
                    actp = act0;
                    asump = asum0;
                }
            }
        }
    }
    if (u != 0) flush();
    TL_TRACE_STAMP(14);
    __syncthreads();
    TL_TRACE_STAMP(16);

    auto chunk_sum = [&](int ch, int row, int m) {  // entries of one output in warp order
        float v = 0.f;
        const int lo = ch * P, hi = lo + P;
#pragma unroll
        for (int w = 0; w < NW; ++w)
            if (warp_begin[w] < hi && warp_begin[w + 1] > lo && warp_begin[w] < warp_begin[w + 1])
                v += entries[static_cast<size_t>(ch + w) * ENTRY + row * 8 * MT + m];
        return v;
    };
    if (args.epilogue == EPI_SWIGLU_PAIRS) {  // gate rows 0-7 and up rows 8-15 of every chunk -> 8 activations
        for (int o = threadIdx.x; o < chunks * 8 * Mp; o += NT) {
            const int m = o / (chunks * 8);
            const int rr = o - m * (chunks * 8);
            const int ch = rr >> 3, row = rr & 7;
            const float gate = to_f(from_f<T>(chunk_sum(ch, row, m))), up = to_f(from_f<T>(chunk_sum(ch, row + 8, m)));
            out[static_cast<size_t>(m) * (K / 2) + c0 * 8 + rr] = from_f<T>((gate / (1.0f + expf(-gate))) * up);
        }
        TL_TRACE_STAMP(15);
        return;
    }
    // ---- sum the entries of each chunk in warp order, add the residual, store
    for (int o = threadIdx.x; o < outs; o += NT) {
        const int m = o / (chunks * 16);  // request-major: consecutive threads store consecutive features
        const int rr = o - m * (chunks * 16);
        const int ch = rr >> 4, row = rr & 15;
        const int k = r0 + rr;
        if (k < r1) {
            T vb = from_f<T>(chunk_sum(ch, row, m));
            if (res != nullptr) {
                const float rv = o == static_cast<int>(threadIdx.x) ? res_first : to_f(res[static_cast<size_t>(m) * K + k]);
                vb = from_f<T>(rv + to_f(vb));
            }
            out[static_cast<size_t>(m) * K + k] = vb;
        }
    }
    TL_TRACE_STAMP(15);
}

#if TL_TRACE
void trace_bind_matvec(unsigned long long *buf, unsigned int *n, unsigned int cap) { trace_bind(buf, n, cap); }
#endif

// Programmatic dependent launch is on by default (tl_set_pdl(0) or TL_PDL=0 turns it off): every
// kernel that carries the attribute reads its predecessor's output only after griddepcontrol.wait,
// so stream order semantics are unchanged.
static bool pdl_default() {
    const char *e = getenv("TL_PDL");
    return !(e != nullptr && e[0] == '0');
}
static bool g_use_pdl = pdl_default();
void set_use_pdl(bool on) { g_use_pdl = on; }
bool use_pdl() { return g_use_pdl; }

constexpr size_t S5_SMEM_MAX = 226 * 1024;
static size_t stream5_smem_bytes(int N, int K, int MP, int grid) {
    const int nw = S5_WARPS;
    const int MT = (MP + 7) / 8, MPA = MP < 8 ? 8 : MP;
    const int all = (K + 15) / 16;
    const int chunks = (all + grid - 1) / grid;
    size_t bytes = static_cast<size_t>(N / 8) * MP * 16;
    bytes += static_cast<size_t>(N / 128) * MPA * 4;
    const size_t entries = static_cast<size_t>(chunks + nw) * 16 * 8 * MT * 4;
    const size_t sq = static_cast<size_t>(N / 128) * MP * 4;
    bytes += entries > sq ? entries : sq;
    return bytes;
}

// ---- launch geometry
// One CTA per SM minus S5_RESERVED_SMS: the few CTAs of the kernel behind it (the 8-CTA attention launch, the first CTAs
// of the next projection) then start early under programmatic dependent launch and issue their independent loads while
// this one is still running.
constexpr int S5_RESERVED_SMS = 8;
static int stream5_grid(int K) {
    const int all = (K + 15) / 16;
    int sms = sm_count() - S5_RESERVED_SMS;
    if (sms < 1) sms = 1;
    return all < sms ? all : sms;
}

// Launch plan of the streaming kernel: rows of `a` per pass (a power of two <= TL_MATVEC_MAX_ROWS, as many as fit in
// shared memory) and 128-column groups per unit (2 when N % 256 == 0, the scale/bias rows are 4-byte aligned and at
// most 16 rows are streamed: 32 rows x pairs would spill).  The launch and tl_quantized_matmul_route both use it.
int w4a16_stream_plan(int M, int N, int K, int lda, const void *p0, const void *p1, const void *b, const void *scales, const void *biases,
                      int *rows_per_pass, int *units) {
    if (!aligned16(p0) || !aligned16(b) || (p1 && !aligned16(p1)) || (lda % 8) != 0)
        return fail(TL_EINVAL, "quantized_matmul: operands must be 16-byte aligned");
    if (K >= (1 << 24)) return fail(TL_EINVAL, "quantized_matmul: more than 2^24 output features");
    const bool pairs = (N % 256) == 0 && (reinterpret_cast<uintptr_t>(scales) & 3u) == 0 && (reinterpret_cast<uintptr_t>(biases) & 3u) == 0;
    int rpp = w4_pad_cols(M < TL_MATVEC_MAX_ROWS ? M : TL_MATVEC_MAX_ROWS);
    const int grid_x = stream5_grid(K);
    while (rpp > 1 && stream5_smem_bytes(N, K, rpp, grid_x) > S5_SMEM_MAX) rpp /= 2;
    if (stream5_smem_bytes(N, K, rpp, grid_x) > S5_SMEM_MAX)
        return fail(TL_EINVAL, "quantized_matmul: activations do not fit in shared memory (N=%d, K=%d, rows=%d)", N, K, rpp);
    *rows_per_pass = rpp;
    *units = pairs && M <= 16 ? 2 : 1;
    return TL_OK;
}

template <typename T, int MP, int U>
static int stream5_launch(StreamArgs args, cudaStream_t st) {
    const int grid_x = stream5_grid(args.K);
    const size_t smem = stream5_smem_bytes(args.N, args.K, MP, grid_x);
    const size_t limit = S5_SMEM_MAX;
    static bool configured = false;  // per process: one device per process (DESIGN.md section 5)
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(w4a16_stream5_kernel<T, MP, U>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(limit));
        if (e != cudaSuccess) return fail(TL_ECUDA, "quantized_matmul: cannot raise shared memory limit: %s", cudaGetErrorString(e));
        configured = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid_x, ceil_div(args.M, args.rows_per_pass));
    cfg.blockDim = dim3(S5_WARPS * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = g_use_pdl ? 1 : 0;
    cudaError_t e = cudaLaunchKernelEx(&cfg, w4a16_stream5_kernel<T, MP, U>, args);
    if (e != cudaSuccess) return fail(TL_ECUDA, "w4a16_stream5: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("w4a16_stream5");
    return TL_OK;
}

template <typename T, int U>
static int stream5_u(StreamArgs args, cudaStream_t st) {
    switch (args.rows_per_pass) {
        case 1: return stream5_launch<T, 1, U>(args, st);
        case 2: return stream5_launch<T, 2, U>(args, st);
        case 4: return stream5_launch<T, 4, U>(args, st);
        case 8: return stream5_launch<T, 8, U>(args, st);
        case 16: return stream5_launch<T, 16, U>(args, st);
        default: return stream5_launch<T, 32, U>(args, st);
    }
}

template <typename T>
static int stream5_t(StreamArgs args, cudaStream_t st) {
    int units = 1;
    if (int e = w4a16_stream_plan(args.M, args.N, args.K, args.lda, args.p0, args.p1, args.b, args.scales, args.biases, &args.rows_per_pass,
                                  &units))
        return e;
    return units == 2 ? stream5_u<T, 2>(args, st) : stream5_u<T, 1>(args, st);
}

int launch_w4a16_fused(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *p1,
                       const void *residual, int M, int N, int K, int lda, int prologue, int epilogue, float eps, int dtype,
                       cudaStream_t st) {
    if (M == 0 || K == 0) return TL_OK;
    StreamArgs args{};
    args.scales = scales, args.biases = biases, args.b = static_cast<const uint32_t *>(b), args.out = out;
    args.p0 = p0, args.p1 = p1, args.residual = residual;
    args.M = M, args.N = N, args.K = K, args.lda = lda;
    args.prologue = prologue, args.epilogue = epilogue, args.eps = eps;
    switch (dtype) {
        case TL_F16: return stream5_t<__half>(args, st);
        case TL_BF16: return stream5_t<__nv_bfloat16>(args, st);
    }
    return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
}

// ---------------------------------------------------------------------------
// Scalar control kernel: one thread per output, the literal arithmetic of
// quantized_matmul_vanilla_w4a16_g128 (quantized_matmul.metal:8-56):
//   sum += (float(code) * scale + bias) * float(a), codes in nibble order.
template <typename T>
__global__ void w4a16_vanilla_kernel(const T *__restrict__ scales, const T *__restrict__ biases,
                                     const T *__restrict__ a, const uint32_t *__restrict__ b, T *__restrict__ out,
                                     int M, int N, int K) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = blockIdx.y;
    if (k >= K || i >= M) return;
    const int words = N / 8;
    const int G = N / 128;
    const uint32_t *brow = b + static_cast<size_t>(k) * words;
    const T *arow = a + static_cast<size_t>(i) * N;
    float sum = 0.f;
    for (int grp = 0; grp < G; ++grp) {
        const float s = to_f(scales[static_cast<size_t>(k) * G + grp]);
        const float c = to_f(biases[static_cast<size_t>(k) * G + grp]);
        for (int w = 0; w < 16; ++w) {
            const uint32_t packed = brow[grp * 16 + w];
            const T *av = arow + grp * 128 + w * 8;
#pragma unroll
            for (int j = 0; j < 8; ++j)
                sum += (static_cast<float>((packed >> (4 * j)) & 0xFu) * s + c) * to_f(av[j]);
        }
    }
    out[static_cast<size_t>(i) * K + k] = from_f<T>(sum);
}

int launch_w4a16_vanilla(const void *scales, const void *biases, const void *a, const void *b, void *out, int M,
                         int N, int K, int dtype, cudaStream_t st) {
    if (M == 0 || K == 0) return TL_OK;
    dim3 grid(ceil_div(K, 128), M);
    if (dtype == TL_BF16)
        w4a16_vanilla_kernel<__nv_bfloat16><<<grid, 128, 0, st>>>(
            static_cast<const __nv_bfloat16 *>(scales), static_cast<const __nv_bfloat16 *>(biases),
            static_cast<const __nv_bfloat16 *>(a), static_cast<const uint32_t *>(b), static_cast<__nv_bfloat16 *>(out),
            M, N, K);
    else if (dtype == TL_F16)
        w4a16_vanilla_kernel<__half><<<grid, 128, 0, st>>>(static_cast<const __half *>(scales),
                                                            static_cast<const __half *>(biases),
                                                            static_cast<const __half *>(a),
                                                            static_cast<const uint32_t *>(b),
                                                            static_cast<__half *>(out), M, N, K);
    else
        return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
    TL_LAUNCH_CHECK("w4a16_vanilla");
    return TL_OK;
}

}  // namespace tl
