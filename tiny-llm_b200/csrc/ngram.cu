// Prompt-lookup proposals (DESIGN.md section 14): the tokens that followed the latest, longest earlier occurrence of
// the history's last n tokens, in one launch that first appends the tokens emitted since the previous call.
//
// The history s[0..L) lives in a caller-owned device buffer; the call's `appended` ids (at most 8, by value in the
// kernel's parameters) are s[length..L).  Candidate ends e in [0, L-2] are dealt out in tiles of NG_TILE; CTA b takes
// tiles b, b + grid, ...  Each tile is staged in shared memory with the NG_HALO tokens before it, and thread j of the
// tile counts c(e), the number of tokens s[e - t] == s[L - 1 - t] matching from t = 0, capped at min(n_max, e + 1).
// Keys (c << 32) | e with c >= n_min are reduced by max: within the CTA by shuffles, across CTAs by one atomicMax on
// the state's 64-bit word.  Max is order-independent, so the chosen (c, e) does not depend on the grid.  The last CTA
// to arrive (a counter in the state, after a fence) writes the outputs: c, e and the k continuation tokens of s
// followed by themselves, then the one-hot rows, then zeroes the key and the counter for the next call.  No host
// synchronisation and no allocation: the call captures into a CUDA graph.
#include "common.cuh"
#include "kernels.h"

namespace tl {

namespace {

constexpr int NG_THREADS = 256;
constexpr int NG_TILE = TL_NGRAM_TILE;
constexpr int NG_HALO = TL_NGRAM_MAX_N - 1;
constexpr int NG_MAX_APPEND = TL_NGRAM_MAX_APPEND;

struct Appended {
    int32_t ids[NG_MAX_APPEND];
};

// state words: [0, 2) the 64-bit max key, [2] the arrival counter, [3] the one-hot rows written last, [4, 11) their ids
constexpr int ST_COUNT = 2, ST_PREV_K = 3, ST_PREV = 4;

__device__ __forceinline__ void put_bits(void *buf, long long at, int esize, uint32_t bits) {
    if (esize == 4)
        static_cast<uint32_t *>(buf)[at] = bits;
    else
        static_cast<uint16_t *>(buf)[at] = static_cast<uint16_t>(bits);
}

__global__ void __launch_bounds__(NG_THREADS) ngram_propose_kernel(int32_t *__restrict__ hist, int length, Appended app, int n_app, int k,
                                                                   int n_min, int n_max, int32_t *__restrict__ out,
                                                                   int32_t *__restrict__ state, void *__restrict__ onehot, int vocab,
                                                                   int esize, uint32_t ninf_bits) {
    __shared__ int32_t tile[NG_HALO + NG_TILE];
    __shared__ int32_t s_app[NG_MAX_APPEND], s_suffix[TL_NGRAM_MAX_N];
    __shared__ unsigned long long w_best[NG_THREADS / 32];
    __shared__ bool s_last;
    const int L = length + n_app;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

#pragma unroll
    for (int j = 0; j < NG_MAX_APPEND; ++j)  // static indices: the parameter array stays in the constant bank
        if (threadIdx.x == j && j < n_app) {
            s_app[j] = app.ids[j];
            if (blockIdx.x == 0) hist[length + j] = app.ids[j];  // other CTAs read s[length..L) from s_app
        }
    __syncthreads();
    if (threadIdx.x < n_max && static_cast<int>(threadIdx.x) < L) {
        const int i = L - 1 - threadIdx.x;
        s_suffix[threadIdx.x] = i < length ? hist[i] : s_app[i - length];
    }

    unsigned long long best = 0;
    const int ends = L - 1;  // candidates e in [0, L - 2]
    for (int base = blockIdx.x * NG_TILE; base < ends; base += gridDim.x * NG_TILE) {
        __syncthreads();  // the previous tile is consumed (and, the first time, s_suffix is written)
        for (int j = threadIdx.x; j < NG_HALO + NG_TILE; j += NG_THREADS) {
            const int i = base - NG_HALO + j;
            tile[j] = (i >= 0 && i < L) ? (i < length ? hist[i] : s_app[i - length]) : 0;
        }
        __syncthreads();
        for (int j = threadIdx.x; j < NG_TILE && base + j < ends; j += NG_THREADS) {
            const int e = base + j;
            const int cap = min(n_max, e + 1);  // never reads before s[0]
            int c = 0;
            while (c < cap && tile[NG_HALO + j - c] == s_suffix[c]) ++c;
            if (c >= n_min) best = max(best, (static_cast<unsigned long long>(c) << 32) | static_cast<unsigned>(e));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) w_best[warp] = best;
    __syncthreads();
    unsigned long long *key = reinterpret_cast<unsigned long long *>(state);
    if (threadIdx.x == 0) {
        unsigned long long b = 0;
        for (int w = 0; w < NG_THREADS / 32; ++w) b = max(b, w_best[w]);
        if (b) atomicMax(key, b);
        __threadfence();  // the key is visible before this CTA counts itself in
        const unsigned arrived = atomicAdd(reinterpret_cast<unsigned *>(state + ST_COUNT), 1u);
        s_last = arrived == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;

    // ---- the last CTA: outputs, one-hot rows, state reset
    __threadfence();
    const unsigned long long won = atomicAdd(key, 0ull);
    const int c = static_cast<int>(won >> 32);
    const int e = c ? static_cast<int>(won & 0xffffffffu) : -1;
    int32_t p[TL_NGRAM_MAX_K];
    out[0] = c;
    out[1] = e;
    for (int t = 0; t < k; ++t) {
        const int i = e + 1 + t;  // e <= L - 2, so i - L < t: a continuation past s repeats the proposals themselves
        p[t] = !c ? -1 : i < length ? hist[i] : i < L ? s_app[i - length] : p[i - L];
        out[2 + t] = p[t];
    }
    if (onehot) {
        const int prev = min(state[ST_PREV_K], k);
        for (int t = 0; t < prev; ++t) {
            const int v = state[ST_PREV + t];
            if (v >= 0 && v < vocab) put_bits(onehot, static_cast<long long>(t) * vocab + v, esize, ninf_bits);
        }
        for (int t = 0; t < (c ? k : 0); ++t)
            if (p[t] >= 0 && p[t] < vocab) put_bits(onehot, static_cast<long long>(t) * vocab + p[t], esize, 0u);
        state[ST_PREV_K] = c ? k : 0;
        for (int t = 0; t < k; ++t) state[ST_PREV + t] = p[t];
    }
    *key = 0ull;
    state[ST_COUNT] = 0;
}

}  // namespace

int ngram_propose_grid(int length, int n_appended) {
    const long long ends = static_cast<long long>(length) + n_appended - 1;
    return ends <= NG_TILE ? 1 : static_cast<int>(ceil_div_ll(ends, NG_TILE));
}

int launch_ngram_propose(int32_t *history, int length, const int32_t *appended, int n_appended, int k, int n_min, int n_max, int32_t *out,
                         int32_t *state, void *onehot, int vocab, int dtype, int grid, cudaStream_t st) {
    Appended app{};
    for (int j = 0; j < n_appended; ++j) app.ids[j] = appended[j];
    const int esize = dtype == TL_F32 ? 4 : 2;
    const uint32_t ninf = dtype == TL_F32 ? 0xff800000u : dtype == TL_F16 ? 0xfc00u : 0xff80u;
    const int blocks = grid > 0 ? grid : ngram_propose_grid(length, n_appended);
    ngram_propose_kernel<<<blocks, NG_THREADS, 0, st>>>(history, length, app, n_appended, k, n_min, n_max, out, state, onehot, vocab, esize,
                                                        ninf);
    TL_LAUNCH_CHECK("ngram_propose");
    return TL_OK;
}

}  // namespace tl
