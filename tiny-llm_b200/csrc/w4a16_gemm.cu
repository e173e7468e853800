// W4A16 prefill GEMM on the Hopper tensor cores: dispatch onto the swap-AB wgmma kernel of w4a16_skinny.cu with
// 128-token tiles (launch_w4a16_tiles), plus the tensor-map encoder shared by the TMA kernels.
//
//   out[m, n] = sum_k a[m, k] * T(code[n, k] * scale[n, k/128] + bias[n, k/128])
//
// (reference naming: a [M, N_red], b [K_out, N_red/8]; here m = token, n = output feature, k = reduction index).
// Replaces quantized_matmul_simdgroup_w4a16_g128 (src/extensions_ref/src/quantized_matmul.metal:96-249):
// like that kernel the weight is rounded to the activation dtype when it is dequantised into shared memory (:183-194)
// and the accumulation is fp32.
#include <cuda.h>
#include <stdlib.h>
#include <cudaTypedefs.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace tl {

// ---------------------------------------------------------------- host side --
PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
    return fn;
}

// TL_NO_TC_GEMM=1: M > 128 projections on the streaming kernel instead (A/B control).
static bool tc_gemm_disabled() {
    static const bool off = [] { const char *e = getenv("TL_NO_TC_GEMM"); return e != nullptr && e[0] == '1'; }();
    return off;
}

bool w4a16_gemm_supported(int M, int N, int K, int dtype) {
    if (tc_gemm_disabled()) return false;
    return (dtype == TL_BF16 || dtype == TL_F16) && M > 0 && K > 0 && N % 128 == 0;
}

// The schedule never splits the reduction: a 128 x 128 tile already runs N/128 group blocks back to back, and
// small-M problems go to the streaming or split-reduction kernels.  A split-K request therefore runs the very same
// kernel (bit-identical results, tests_refsol/test_week_2_day_7.py:80-109).
int w4a16_gemm_split(int, int, int, int) { return 1; }
size_t w4a16_gemm_workspace(int, int, int, int, int) { return 0; }

int launch_w4a16_gemm(const void *scales, const void *biases, const void *a, const void *b, void *out, int M, int N, int K,
                      int dtype, int /*use_split_k*/, void * /*ws*/, size_t /*ws_bytes*/, cudaStream_t st) {
    if (dtype != TL_BF16 && dtype != TL_F16) return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
    return launch_w4a16_tiles(scales, biases, a, b, out, M, N, K, dtype, st);
}

}  // namespace tl
