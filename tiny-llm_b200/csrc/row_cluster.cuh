// Building blocks of the kernels that reduce one logits row per thread-block cluster: tl_sample (sampling.cu) and
// tl_logprobs (logprobs.cu).  A row of V entries is split over C = ceil(V / SAMPLE_SLICE_MIN) CTAs (at most
// SAMPLE_MAX_CLUSTER; sample_plan() in sampling.cu is the rule), each CTA stages its slice once in shared memory as
// fp32, and the CTAs merge integers and first-maximum-wins candidates over distributed shared memory.
#pragma once

#include <cstdint>

#include "common.cuh"

namespace tl {

namespace {

constexpr int SAMPLE_THREADS = 512;
constexpr int SAMPLE_WARPS = SAMPLE_THREADS / 32;
constexpr int SAMPLE_MAX_CLUSTER = 8;
constexpr int SAMPLE_SLICE_MIN = 4096;      // vocabulary entries per CTA before the cluster grows
constexpr int SAMPLE_MAX_SMEM = 200 << 10;  // staged slice: fp32, 51,200 entries per CTA
constexpr int BINS = 256;
constexpr float MASS_SCALE = 1099511627776.f;  // 2^40: e_i <= 1, so a row of < 2^23 entries sums below 2^63

struct Best {
    float v;
    int i;
};
__device__ __forceinline__ Best better(Best a, Best b) {
    return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;  // first maximum wins; NaN never does
}
__device__ __forceinline__ Best warp_best(Best m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = better(m, Best{__shfl_xor_sync(0xffffffffu, m.v, o), __shfl_xor_sync(0xffffffffu, m.i, o)});
    return m;
}

// Order-preserving key of a non-NaN float (-0 is folded onto +0 first, so equal values have equal keys).
__device__ __forceinline__ uint32_t order_key(float x) {
    const uint32_t b = __float_as_uint(x == 0.f ? 0.f : x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

template <typename T>
__device__ __forceinline__ void stage_slice(const T *__restrict__ src, float *xs, int n, bool vec) {
    if (vec) {  // the slice start and the row pitch are 16-byte aligned, n a multiple of 16 / sizeof(T)
        constexpr int PER = 16 / sizeof(T);
        for (int i = threadIdx.x * PER; i < n; i += SAMPLE_THREADS * PER) {
            const uint4 raw = *reinterpret_cast<const uint4 *>(src + i);
            if constexpr (sizeof(T) == 4) {
                *reinterpret_cast<float4 *>(xs + i) = make_float4(__uint_as_float(raw.x), __uint_as_float(raw.y), __uint_as_float(raw.z),
                                                                  __uint_as_float(raw.w));
            } else {
                const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = unpack2<T>(w[j]);
                    xs[i + 2 * j] = f.x;
                    xs[i + 2 * j + 1] = f.y;
                }
            }
        }
    } else {
        for (int i = threadIdx.x; i < n; i += SAMPLE_THREADS) xs[i] = to_f(src[i]);
    }
}

// One 32-bit broadcast per warp-uniform loop step: the lanes of `peers` share a bin; the lowest of them adds their
// count and mass to it.
__device__ __forceinline__ void bin_add(unsigned int *count, unsigned long long *mass, int bin, unsigned long long e, bool with_mass) {
    const unsigned active = __ballot_sync(0xffffffffu, bin >= 0);
    if (!active) return;
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    const int lane = threadIdx.x & 31;
    unsigned long long sum = 0;
    if (with_mass) {
#pragma unroll 8
        for (int j = 0; j < 32; ++j) {
            const unsigned long long v = __shfl_sync(0xffffffffu, e, j);
            if ((peers >> j) & 1u) sum += v;
        }
    }
    if (bin >= 0 && lane == __ffs(peers) - 1) {
        atomicAdd(&count[bin], static_cast<unsigned>(__popc(peers)));
        if (with_mass) atomicAdd(&mass[bin], sum);
    }
}

}  // namespace

}  // namespace tl
