// Beam search's cross-beam selection (DESIGN.md section 15): one step's R x N candidates, ranked and walked in one CTA.
//
// Thread t < R * N owns candidate t = r * N + k: token top_ids[r, k] with score s = fl(cum[r] + top_lp[r, k]).  A
// candidate with id -1, or whose s is -inf or NaN, is never taken.  Its walk position is the number of takeable
// candidates before it in the order (s descending, t ascending) - (r, k) ascending is t ascending - counted over the
// staged scores, so the ranking needs no atomics and no sort.  Thread p then looks at the candidate at position p:
// warp ballots and per-warp prefix counts give, for a non-EOS candidate, the number of non-EOS candidates before it
// (its live-beam index while below W) and, for an EOS candidate, the number of EOS candidates before it (its
// finished index while p < W).  Every read of cum is staged before the first write, so cum is updated in place:
// entries [0, live) get the new beams' sums and [live, W) -inf, which keeps an idle row of a W-row step from ever
// being taken.  No host synchronisation and no allocation: the call captures into a CUDA graph.
#include "common.cuh"
#include "kernels.h"

#include <cmath>

namespace tl {

namespace {

constexpr int BS_THREADS = 128;
constexpr int BS_MAX_W = TL_BEAM_MAX_WIDTH;
constexpr int BS_MAX_C = TL_BEAM_MAX_WIDTH * TL_BEAM_MAX_N;
static_assert(BS_MAX_C <= BS_THREADS, "one thread per candidate");

struct EosIds {
    int32_t ids[TL_BEAM_MAX_EOS];
};

__global__ void __launch_bounds__(BS_THREADS) beam_select_kernel(const float *__restrict__ top_lp, const int32_t *__restrict__ top_ids,
                                                                 float *__restrict__ cum, int rows, int n, int width, EosIds eos,
                                                                 int num_eos, int32_t *__restrict__ result) {
    __shared__ float s_score[BS_MAX_C];
    __shared__ int32_t s_id[BS_MAX_C];
    __shared__ bool s_ok[BS_MAX_C];
    __shared__ int32_t s_at[BS_MAX_C];  // walk position -> candidate
    __shared__ int s_ok_warp[BS_THREADS / 32], s_live_warp[BS_THREADS / 32], s_eos_warp[BS_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int total = rows * n;

    bool ok = false;
    if (t < total) {
        const int r = t / n;
        const float lp = top_lp[t];
        const int32_t id = top_ids[t];
        const float s = __fadd_rn(cum[r], lp);
        s_score[t] = s;
        s_id[t] = id;
        ok = id >= 0 && !isnan(s) && s != -INFINITY;
        s_ok[t] = ok;
    }
    const unsigned ok_bits = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_ok_warp[warp] = __popc(ok_bits);
    __syncthreads();  // every input (cum included) is staged: the writes below may overwrite cum
    if (t < total && s_ok[t]) {
        const float s = s_score[t];
        int pos = 0;
        for (int u = 0; u < total; ++u) pos += s_ok[u] && (s_score[u] > s || (s_score[u] == s && u < t));
        s_at[pos] = t;
    }
    int taken = 0;
    for (int w = 0; w < BS_THREADS / 32; ++w) taken += s_ok_warp[w];
    __syncthreads();

    bool is_eos = false, is_live = false;
    int c = -1;
    if (t < taken) {
        c = s_at[t];
#pragma unroll
        for (int e = 0; e < TL_BEAM_MAX_EOS; ++e) is_eos |= e < num_eos && s_id[c] == eos.ids[e];
        is_live = !is_eos;
    }
    const unsigned below = (1u << lane) - 1u;
    const unsigned live_bits = __ballot_sync(0xffffffffu, is_live), eos_bits = __ballot_sync(0xffffffffu, is_eos);
    if (lane == 0) {
        s_live_warp[warp] = __popc(live_bits);
        s_eos_warp[warp] = __popc(eos_bits);
    }
    __syncthreads();
    int live_before = __popc(live_bits & below), eos_before = __popc(eos_bits & below), live_total = 0;
    for (int w = 0; w < BS_THREADS / 32; ++w) {
        if (w < warp) {
            live_before += s_live_warp[w];
            eos_before += s_eos_warp[w];
        }
        live_total += s_live_warp[w];
    }

    int32_t *live_parent = result + 2, *live_token = live_parent + BS_MAX_W, *live_cum = live_token + BS_MAX_W;
    int32_t *fin_parent = live_cum + BS_MAX_W, *fin_token = fin_parent + BS_MAX_W, *fin_sum = fin_token + BS_MAX_W,
            *fin_pos = fin_sum + BS_MAX_W;
    if (is_live && live_before < width) {
        live_parent[live_before] = c / n;
        live_token[live_before] = s_id[c];
        live_cum[live_before] = __float_as_int(s_score[c]);
        cum[live_before] = s_score[c];
    }
    if (is_eos && t < width) {
        fin_parent[eos_before] = c / n;
        fin_token[eos_before] = s_id[c];
        fin_sum[eos_before] = __float_as_int(s_score[c]);
        fin_pos[eos_before] = t;
    }
    const int live = min(live_total, width);
    if (t >= live && t < width) cum[t] = -INFINITY;
    // the finished count: EOS candidates at positions below W, i.e. eos_before + is_eos of thread W - 1 (or of the
    // last taken position when fewer than W candidates are takeable)
    const int last = min(width, taken) - 1;
    if (t == last) result[1] = eos_before + (is_eos ? 1 : 0);
    if (t == 0) {
        result[0] = live;
        if (last < 0) result[1] = 0;
    }
}

}  // namespace

int launch_beam_select(const float *top_lp, const int32_t *top_ids, float *cum, int rows, int n, int width, const int32_t *eos_ids,
                       int num_eos, int32_t *result, cudaStream_t st) {
    EosIds eos{};
    for (int e = 0; e < num_eos; ++e) eos.ids[e] = eos_ids[e];
    beam_select_kernel<<<1, BS_THREADS, 0, st>>>(top_lp, top_ids, cum, rows, n, width, eos, num_eos, result);
    TL_LAUNCH_CHECK("beam_select");
    return TL_OK;
}

}  // namespace tl
