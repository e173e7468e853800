// Shared device/host helpers for the sm_90a kernels of tiny-llm_b200.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tiny_llm_b200.h"

namespace tl {

// ---- host side: error reporting and launch bookkeeping -------------------
int fail(int code, const char *fmt, ...);  // records tl_last_error(), returns code
int check_launch(const char *what);        // cudaPeekAtLastError -> TL_ECUDA
void count_launch(int n = 1);
int sm_count();

static inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// ---- device side -----------------------------------------------------------
template <typename T>
struct Num;
template <>
struct Num<float> {
    static __device__ __forceinline__ float to_f(float v) { return v; }
    static __device__ __forceinline__ float from_f(float v) { return v; }
};
template <>
struct Num<__half> {
    static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <>
struct Num<__nv_bfloat16> {
    static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

template <typename T>
__device__ __forceinline__ float to_f(T v) {
    return Num<T>::to_f(v);
}
template <typename T>
__device__ __forceinline__ T from_f(float v) {
    return Num<T>::from_f(v);
}

// Two packed 16-bit values <-> two floats.
template <typename T>
__device__ __forceinline__ float2 unpack2(uint32_t u);
template <>
__device__ __forceinline__ float2 unpack2<__nv_bfloat16>(uint32_t u) {
    return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
template <>
__device__ __forceinline__ float2 unpack2<__half>(uint32_t u) {
    __half2 h = *reinterpret_cast<__half2 *>(&u);
    return __half22float2(h);
}
template <typename T>
__device__ __forceinline__ uint32_t pack2(float lo, float hi);
template <>
__device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&v);
}
template <>
__device__ __forceinline__ uint32_t pack2<__half>(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t *>(&v);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Streaming (read-once) 128-bit global load that does not allocate in L1.
__device__ __forceinline__ uint4 ldg_stream(const void *p) {
    uint4 r;
    // .L2::128B: a miss on one 64-byte half of a weight row's 128-byte line fetches the whole line; the same warp's
    // next load reads the other half (decode +1-2 % on H100, DESIGN.md section 4)
    asm volatile("ld.global.nc.L1::no_allocate.L2::128B.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// L2 (ld.global.cg) loads of data another CTA or the previous kernel has just written.  They are
// VOLATILE asm with a memory clobber on purpose: the CUDA header versions (__ldcg) are plain asm
// without a clobber, which the compiler may hoist above griddepcontrol.wait / a grid barrier -
// observed: q rows read before the projection that produces them had finished.
__device__ __forceinline__ uint4 ld_cg(const uint4 *p) {
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ float ld_cg(const float *p) {
    float r;
    asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ int ld_cg(const int *p) {
    int r;
    asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ __nv_bfloat16 ld_cg(const __nv_bfloat16 *p) {
    unsigned short r;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(r) : "l"(p) : "memory");
    return __ushort_as_bfloat16(r);
}
__device__ __forceinline__ __half ld_cg(const __half *p) {
    unsigned short r;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(r) : "l"(p) : "memory");
    return __ushort_as_half(r);
}

// ---- programmatic dependent launch ------------------------------------------
// A kernel launched through launch_chained() may become resident while its predecessor on the stream is still
// running (the predecessor lets it in with griddep_launch(), or implicitly by exiting).  It must execute
// griddep_wait() before it reads anything the predecessor wrote and before it writes anything the predecessor may
// still read; the wait returns once the predecessor grid has COMPLETED and its writes are visible.  Everything a
// kernel does before the wait (barrier init, tensor-map prefetch, weight prefetch) overlaps the
// predecessor's tail.  Data written by an earlier kernel of such a chain is read through L2 (ld_cg / TMA), never
// through a possibly stale L1 line.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool use_pdl();  // kernels.h; TL_PDL=0 turns the attribute off (griddepcontrol.wait then returns at once)

template <typename... P, typename... A>
static inline cudaError_t launch_chained(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A &&...a) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<P>(a)...);
}

}  // namespace tl

#define TL_LAUNCH_CHECK(name)                    \
    do {                                         \
        ::tl::count_launch();                    \
        int _e = ::tl::check_launch(name);       \
        if (_e != TL_OK) return _e;              \
    } while (0)
