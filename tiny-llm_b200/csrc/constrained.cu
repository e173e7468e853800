// Token masks of a regex constraint (DESIGN.md section 8c): the byte DFA of the pattern lifted to the tokens of a
// vocabulary.  One thread per token walks the token's bytes through the DFA table from every state in turn; a warp
// covers 32 consecutive tokens and writes the state's mask word with one ballot.  The table sits in shared memory
// when it fits (at most MASK_SMEM_STATES states), and is read through the L1 from global memory otherwise.
#include "common.cuh"
#include "kernels.h"

namespace tl {

namespace {

constexpr int MASK_THREADS = 256;
constexpr int MASK_SMEM_STATES = 192;  // 192 KiB of int32 [S, 256]

template <bool SMEM>
__global__ void __launch_bounds__(MASK_THREADS)
    token_masks_kernel(const int32_t *__restrict__ dfa, const uint8_t *__restrict__ accept, int S, const int32_t *__restrict__ offsets,
                       const uint8_t *__restrict__ bytes, int V, const int32_t *__restrict__ eos, int n_eos, uint32_t *__restrict__ masks,
                       uint32_t *__restrict__ reach) {
    extern __shared__ int4 table_dyn[];
    const int32_t *table = dfa;
    if constexpr (SMEM) {
        int4 *dst = table_dyn;
        const int4 *src = reinterpret_cast<const int4 *>(dfa);
        for (int i = threadIdx.x; i < S * 64; i += MASK_THREADS) dst[i] = __ldg(src + i);
        __syncthreads();
        table = reinterpret_cast<const int32_t *>(table_dyn);
    }
    const int t = blockIdx.x * MASK_THREADS + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const int word = t >> 5;  // the same for the 32 lanes of a warp
    const int W = (V + 31) >> 5, RW = (S + 31) >> 5;
    const bool in = t < V;
    int b0 = 0, b1 = 0;
    bool is_eos = false;
    if (in) {
        b0 = __ldg(offsets + t);
        b1 = __ldg(offsets + t + 1);
        for (int j = 0; j < n_eos; ++j) is_eos |= __ldg(eos + j) == t;
    }
    if (is_eos) b1 = b0;  // an EOS id never walks bytes
    for (int s = 0; s < S; ++s) {
        int e = -1;
        if (b1 > b0) {
            e = s;
            for (int j = b0; j < b1 && e >= 0; ++j) e = table[e * 256 + __ldg(bytes + j)];
        }
        const bool ok = e >= 0 || (is_eos && __ldg(accept + s) != 0);
        const unsigned bits = __ballot_sync(0xffffffffu, ok);
        if (lane == 0 && word < W) masks[static_cast<size_t>(s) * W + word] = bits;
        const unsigned peers = __match_any_sync(0xffffffffu, e);  // lanes that end in the same state add one bit
        if (e >= 0 && lane == __ffs(peers) - 1) atomicOr(reach + static_cast<size_t>(s) * RW + (e >> 5), 1u << (e & 31));
    }
    const unsigned terminal = __ballot_sync(0xffffffffu, is_eos);  // state S, after EOS: only EOS
    if (lane == 0 && word < W) masks[static_cast<size_t>(S) * W + word] = terminal;
}

}  // namespace

int launch_constraint_token_masks(const int32_t *dfa, const uint8_t *accept, int num_states, const int32_t *token_offsets,
                                  const uint8_t *token_bytes, int vocab, const int32_t *eos_ids, int num_eos, uint32_t *masks,
                                  uint32_t *reach, cudaStream_t st) {
    const dim3 grid(ceil_div(vocab, MASK_THREADS));
    if (num_states <= MASK_SMEM_STATES && aligned16(dfa)) {
        const size_t smem = static_cast<size_t>(num_states) * 256 * sizeof(int32_t);
        static bool configured = false;
        if (!configured) {
            if (cudaFuncSetAttribute(token_masks_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     MASK_SMEM_STATES * 256 * static_cast<int>(sizeof(int32_t))) != cudaSuccess)
                return fail(TL_ECUDA, "constraint_token_masks: cannot raise shared memory limit");
            configured = true;
        }
        token_masks_kernel<true><<<grid, MASK_THREADS, smem, st>>>(dfa, accept, num_states, token_offsets, token_bytes, vocab, eos_ids,
                                                                   num_eos, masks, reach);
    } else {
        token_masks_kernel<false><<<grid, MASK_THREADS, 0, st>>>(dfa, accept, num_states, token_offsets, token_bytes, vocab, eos_ids,
                                                                 num_eos, masks, reach);
    }
    TL_LAUNCH_CHECK("constraint_token_masks");
    return TL_OK;
}

}  // namespace tl
