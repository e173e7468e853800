// Paged causal FlashAttention prefill on the Hopper tensor cores (wgmma + TMA), bf16, head_dim 128, L > 8.
//
// Replaces paged_attention_mma_bf16_d128 (src/extensions_ref/src/
// paged_attention.metal:250-506): same arithmetic - fp32 scores in base 2 (:414 scale_log2),
// bottom-right causal limit key <= row + (context - L) (:411), fp32 running max / sum, the
// probabilities rounded to bf16 before P V (:439-444), output = O / sum (0 when nothing is visible).
//
// One CTA = one (request, KV head, block of RH query positions): its 128 MMA rows are the G = Hq/Hkv
// query heads of the KV head x RH = 128/G consecutive query positions, so every K/V tile the CTA
// fetches is shared by all the query heads that need it, and the causal frontier is almost the same
// for every row (RH <= 128 positions apart).  Per 64-key tile:
//
//   warp 0 (one lane)    TMA producer: Q once (3-D map [D, L, B*Hq], box 64 x RH x G, 128-byte
//                        swizzle = the K-major wgmma layout), then K and V tiles - a (page, kv head)
//                        slab is one contiguous [page x 128] bf16 block, fetched as 4-D boxes
//                        [64 d x 64 keys] keyed by block_table (invalid page ids land outside the
//                        tensor and are zero-filled by the TMA unit) - through a TC_STAGES ring;
//   warpgroups 1, 2      64 MMA rows each: S = Q K^T (wgmma m64n64k16 x 8, both operands K-major in
//                        shared memory, fp32 scores in registers), softmax in registers (a row lives
//                        in the four lanes of a quad: two shuffles for its maximum), the bf16
//                        probabilities stay in registers as the A operand of O += P V (wgmma
//                        m64n128k16 x 4, V tile = MN-major B operand straight from the page layout).
//                        O is rescaled only when a row's maximum grows by more than 2^8 since the last
//                        rescale: P and the row sum always use the same (possibly stale) maximum, so
//                        the result is exact.  Epilogue: O / sum -> bf16 -> global.
#include <math_constants.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace tl {

typedef __nv_bfloat16 bf16;

constexpr int TC_D = 128;         // head dim
constexpr int TC_BM = 128;        // MMA rows per CTA (G heads x RH query positions)
constexpr int TC_BN = 64;         // keys per tile
constexpr int TC_STAGES = 3;
constexpr int TC_CONSUMERS = 2;   // consumer warpgroups, 64 rows each
constexpr int TC_THREADS = 128 * (1 + TC_CONSUMERS);
constexpr int TC_Q_BYTES = TC_BM * TC_D * 2;        // 32 KiB: two 64-column halves of [128 rows x 128 B]
constexpr int TC_KV_TILE = TC_BN * TC_D * 2;        // 16 KiB: two 64-column halves of [64 rows x 128 B]
constexpr int TC_Q_OFF = 0;
constexpr int TC_K_OFF = TC_Q_OFF + TC_Q_BYTES;
constexpr int TC_V_OFF = TC_K_OFF + TC_STAGES * TC_KV_TILE;
constexpr int TC_BAR_OFF = TC_V_OFF + TC_STAGES * TC_KV_TILE;
constexpr int TC_SMEM_BYTES = TC_BAR_OFF + 256;
constexpr float TC_LOG2E = 1.44269504089f;
constexpr float TC_RESCALE_THRESHOLD = 8.0f;  // log2: rescale O when a row maximum grew by more than 2^8

// ex2.approx.ftz: one MUFU instruction (exp2f() adds denormal-range scaling).  Relative error 2^-22; the reference
// kernel uses fast::exp2 (paged_attention.metal:428-436).
__device__ __forceinline__ float tc_ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct TcArgs {
    const int32_t *block_table, *context_lens;
    bf16 *out;
    int L, Hq, Hkv, G, RH;       // RH = query positions per CTA = 128 / G
    int page_size, max_pages, num_pages;
    int tiles_per_page;          // page_size / 64
    float scale_log2;
    int is_causal;
    // split-KV (decode, L <= 8): CTA (query block, split) covers key tiles [split * tiles_per_split, ...) and
    // leaves an unnormalised partial (O fp32, running max in log2 units, sum) for paged_gqa_merge_kernel
    int splits, tiles_per_split;
    int out_token_major;  // out[(b, l, head), :] instead of [(b, head, l), :] (the layout the o-projection takes); split: the merge writes it
    float *ws_o, *ws_m, *ws_l;
    // Shared-prefix attention (TC_PREFIX / TC_SUFFIX, L = 1): group descriptors (first_slot, count, shared_pages) x
    // num_groups; the partial of split s of row r goes to slot r * split_stride + split_base + s.
    const int32_t *groups;
    int num_groups, split_base, split_stride;
    // Segment-causal attention (TC_SEGMENT, one packed request): row l sees the keys segment_start[l] <= key <= l.
    const int32_t *segment_start;
    // Prefixed-segment attention (TC_PREFIXED): row l also sees the keys prefix_start[l] <= key < prefix_end[l].
    const int32_t *prefix_start, *prefix_end;
};

// TC_PLAIN: tl_paged_attention.  TC_PREFIX: one CTA per (group, KV head, split) over the group's shared pages, its 128
// MMA rows the count x G query rows of the group's slots (slot-major), unmasked.  TC_SUFFIX: one CTA per (slot, KV head,
// split) over the slot's keys after its group's shared pages, as TC_PLAIN at L = 1 otherwise.  TC_SEGMENT: TC_PLAIN's
// causal token-major prefill of one request whose L rows are packed prompts: row l also masks the keys before
// segment_start[l], and a CTA starts at the tile holding the smallest segment_start of its rows.  TC_PREFIXED:
// TC_SEGMENT plus one more visible range per row, [prefix_start[l], prefix_end[l]) with prefix_end[l] <= segment_start[l]
// (a reranking pass: a query's prefix, then its documents, DESIGN.md section 19).  A CTA first walks the tiles of the
// hull of its rows' prefix ranges, then its segment tiles as TC_SEGMENT does, and skips every tile between them: the
// documents of one query lie one after another behind their prefix, so without the skip the last one's rows would walk
// all their siblings' tiles.  A tile whose keys a row masks adds exact zeros to it (p = exp2(-inf) = 0, no rescale), so
// the skip changes no bit; the masked K/V slots are multiplied by p = 0, which holds because every pool slot is finite
// (zero-initialised, or written by an earlier pass).
enum { TC_PLAIN = 0, TC_PREFIX = 1, TC_SUFFIX = 2, TC_SEGMENT = 3, TC_PREFIXED = 4 };

// The group of slot b: (first_slot, count, shared_pages), or (b, 1, 0) when no group with shared pages holds it.
__device__ __forceinline__ int3 tc_group_of(const int32_t *groups, int num_groups, int b) {
    for (int i = 0; i < num_groups; ++i) {
        const int f = groups[3 * i], c = groups[3 * i + 1], sp = groups[3 * i + 2];
        if (c > 0 && sp > 0 && b >= f && b < f + c) return make_int3(f, c, sp);
    }
    return make_int3(b, 1, 0);
}

template <int MODE, typename T = bf16>
__global__ void __launch_bounds__(TC_THREADS, 1)
paged_prefill_tc_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                        const __grid_constant__ CUtensorMap tmap_v, const TcArgs a) {
    extern __shared__ __align__(1024) unsigned char tsm[];
    griddep_launch();  // programmatic dependent launch (common.cuh): the successor may set itself up under this grid
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg_idx = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x) >> 7, 0);  // warpgroup, provably warp-uniform
    const int split = static_cast<int>(blockIdx.x) % a.splits;
    const int qb = static_cast<int>(gridDim.x) / a.splits - 1 - static_cast<int>(blockIdx.x) / a.splits;  // long (late) query blocks first
    const int kvh = blockIdx.y, b = blockIdx.z;
    const int q0 = qb * a.RH;
    const int cap = a.max_pages * a.page_size;
    int3 grp = make_int3(b, 1, 0);
    if (MODE == TC_PREFIX || MODE == TC_SUFFIX) grp = tc_group_of(a.groups, a.num_groups, b);
    if (MODE == TC_PREFIX && grp.x != b) return;  // the group's first slot covers its rows
    // The causal shift uses the whole context, the block table clamps afterwards (attention_decode.cu).
    const int ctx = MODE == TC_SEGMENT || MODE == TC_PREFIXED ? a.L : a.context_lens[b];  // the packed rows are the whole context
    // keys any row of this CTA may see: [0, key_end); the prefix pass sees the shared pages, the suffix pass what follows
    const int last_row = min(q0 + a.RH, a.L) - 1;
    const int shared_keys = min(grp.z * a.page_size, cap);
    const int key_end = MODE == TC_PREFIX ? shared_keys
                        : ctx <= 0 ? 0 : min(a.is_causal ? min(ctx, max(ctx - a.L + last_row + 1, 0)) : ctx, cap);
    const int all_tiles = (key_end + TC_BN - 1) / TC_BN;
    int seg_lo = 0;  // TC_SEGMENT / TC_PREFIXED: the smallest segment start of this CTA's rows
    if (MODE == TC_SEGMENT || MODE == TC_PREFIXED) {
        seg_lo = key_end;
        for (int r = q0; r <= last_row; ++r) seg_lo = min(seg_lo, max(a.segment_start[r], 0));
    }
    const int tile_lo = MODE == TC_SUFFIX ? min(shared_keys / TC_BN, all_tiles)
                        : MODE == TC_SEGMENT || MODE == TC_PREFIXED ? min(seg_lo / TC_BN, all_tiles) : 0;
    // TC_PREFIXED: the tiles pre_t0 .. pre_t0 + pre_n - 1 of the hull of the rows' prefix ranges come first (those at or
    // past tile_lo are segment tiles already); rows with an empty segment (padding) do not count.
    int pre_t0 = 0, pre_n = 0;
    if (MODE == TC_PREFIXED) {
        int p_lo = key_end, p_hi = 0;
        for (int r = q0; r <= last_row; ++r) {
            const int ps = max(a.prefix_start[r], 0), pe = min(a.prefix_end[r], key_end);
            if (ps < pe && a.segment_start[r] <= r) p_lo = min(p_lo, ps), p_hi = max(p_hi, pe);
        }
        pre_t0 = p_lo / TC_BN;
        pre_n = max(min((p_hi + TC_BN - 1) / TC_BN, tile_lo) - pre_t0, 0);
    }
    // Split-KV: the launch fixes the NUMBER of splits from the block table's width (the grid of a captured graph cannot
    // follow the context), the tiles are dealt out here from the request's real length, so a request far below the
    // bound still keeps all its splits busy.
    const int tps = a.splits > 1 ? max((all_tiles - tile_lo + a.splits - 1) / a.splits, 1) : a.tiles_per_split;
    const int t0 = tile_lo + min(split * tps, all_tiles - tile_lo);
    const int n_tiles = min(tps, all_tiles - t0) + pre_n;  // this CTA: global tiles t0 .. t0 + n_tiles - 1 (after the prefix tiles)
    // the global tile of this CTA's j-th tile
    auto tile_of = [&](int j) { return MODE != TC_PREFIXED ? t0 + j : j < pre_n ? pre_t0 + j : t0 + j - pre_n; };

    const uint32_t q_base = g_smem_u32(tsm + TC_Q_OFF);
    const uint32_t k_base = g_smem_u32(tsm + TC_K_OFF), v_base = g_smem_u32(tsm + TC_V_OFF);
    const uint32_t bar = g_smem_u32(tsm + TC_BAR_OFF);
    const uint32_t q_full = bar;
    const uint32_t k_full = bar + 8, k_empty = k_full + 8 * TC_STAGES, v_full = k_full + 16 * TC_STAGES, v_empty = k_full + 24 * TC_STAGES;

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_q) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_k) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_v) : "memory");
    }
    if (warp == 1 && lane == 0) {
        g_mbar_init(q_full, 1);
        for (int i = 0; i < TC_STAGES; ++i) {
            g_mbar_init(k_full + 8 * i, 1);
            g_mbar_init(k_empty + 8 * i, TC_CONSUMERS);  // one arrival per consumer warpgroup
            g_mbar_init(v_full + 8 * i, 1);
            g_mbar_init(v_empty + 8 * i, TC_CONSUMERS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // q and the newest K/V rows are the predecessor's output, and this grid overwrites buffers (output, split partials)
    // the predecessor may still read; block tables and context lengths are step inputs uploaded before the chain.
    griddep_wait();

    if (wg_idx == 0) {
        // ------------------------------------------------------------ TMA producer
        if (warp == 0 && n_tiles > 0) {  // whole warp, one elected lane issues
            const int head0 = b * a.Hq + kvh * a.G;
            if (g_elect_one()) {
                g_mbar_expect_tx(q_full, TC_Q_BYTES);
                if (MODE == TC_PREFIX) {  // 4-D map [D, G, Hkv, B], box 64 x G x 1 x RH: row = slot * G + head
                    g_tma_load_4d(q_base, &tmap_q, 0, 0, kvh, b, q_full);
                    g_tma_load_4d(q_base + TC_Q_BYTES / 2, &tmap_q, 64, 0, kvh, b, q_full);
                } else {
                    g_tma_load_3d(q_base, &tmap_q, 0, q0, head0, q_full);
                    g_tma_load_3d(q_base + TC_Q_BYTES / 2, &tmap_q, 64, q0, head0, q_full);
                }
            }
            __syncwarp();
            const int32_t *table = a.block_table + static_cast<size_t>(b) * a.max_pages;
            int s = 0;
            uint32_t ph = 1;  // producer side: first pass through the ring does not wait
            for (int j = 0; j < n_tiles; ++j) {
                const int tile = tile_of(j);
                const int lp = tile / a.tiles_per_page;
                int pid = table[lp];
                if (pid < 0 || pid >= a.num_pages) pid = a.num_pages;  // outside the tensor: the TMA unit writes zeros
                const int slot0 = (tile - lp * a.tiles_per_page) * TC_BN;
                g_mbar_wait(k_empty + 8 * s, ph);
                if (g_elect_one()) {
                    g_mbar_expect_tx(k_full + 8 * s, TC_KV_TILE);
                    g_tma_load_4d(k_base + s * TC_KV_TILE, &tmap_k, 0, slot0, kvh, pid, k_full + 8 * s);
                    g_tma_load_4d(k_base + s * TC_KV_TILE + TC_KV_TILE / 2, &tmap_k, 64, slot0, kvh, pid, k_full + 8 * s);
                }
                __syncwarp();
                g_mbar_wait(v_empty + 8 * s, ph);
                if (g_elect_one()) {
                    g_mbar_expect_tx(v_full + 8 * s, TC_KV_TILE);
                    g_tma_load_4d(v_base + s * TC_KV_TILE, &tmap_v, 0, slot0, kvh, pid, v_full + 8 * s);
                    g_tma_load_4d(v_base + s * TC_KV_TILE + TC_KV_TILE / 2, &tmap_v, 64, slot0, kvh, pid, v_full + 8 * s);
                }
                __syncwarp();
                if (++s == TC_STAGES) s = 0, ph ^= 1u;
            }
        }
    } else {
        // ------------------------------------------------------------ consumers: 64 MMA rows per warpgroup
        // Thread t of the warpgroup holds rows r0 = 16 (t / 32) + (t % 32) / 4 and r0 + 8 of the warpgroup's 64, and the
        // columns 8 j + 2 (t % 4) + {0, 1} of each (wgmma accumulator layout, wgmma.cuh).
        const int wg = wg_idx - 1;
        const int t = threadIdx.x & 127;
        // TC_PREFIX: l = the row's slot inside the group (a row past the group's count is not written)
        int lq[2], g[2], l[2], limit[2], lo[2] = {0, 0};  // lo: TC_SEGMENT's first visible key
        int pst[2] = {0, 0}, pen[2] = {0, 0};               // TC_PREFIXED: the prefix range [pst, pen)
        bool row_valid[2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * rr;  // MMA row 0..127
            if (MODE == TC_PREFIX) {  // row = (slot grp.x + s, head g) of the group; every shared key precedes every row
                l[rr] = r / a.G;
                g[rr] = r - l[rr] * a.G, lq[rr] = 0;
                const int c = l[rr] < grp.y ? a.context_lens[b + l[rr]] : 0;
                row_valid[rr] = c > 0;
                limit[rr] = !row_valid[rr] ? -1 : min(c, key_end) - 1;
                continue;
            }
            g[rr] = r / a.RH, lq[rr] = r - g[rr] * a.RH;                   // query head of the KV group, position inside the block
            l[rr] = q0 + lq[rr];
            row_valid[rr] = l[rr] < a.L && ctx > 0;
            // last key this row may see (bottom-right causal alignment, paged_attention.metal:411)
            limit[rr] = !row_valid[rr] ? -1 : min(a.is_causal ? min(ctx - 1, l[rr] + (ctx - a.L)) : ctx - 1, cap - 1);
            if ((MODE == TC_SEGMENT || MODE == TC_PREFIXED) && row_valid[rr]) {
                lo[rr] = max(a.segment_start[l[rr]], 0);
                if (lo[rr] > limit[rr]) row_valid[rr] = false, limit[rr] = -1;  // an empty segment (a padding row): output 0
                else if (MODE == TC_PREFIXED) pst[rr] = max(a.prefix_start[l[rr]], 0), pen[rr] = min(a.prefix_end[l[rr]], lo[rr]);
            }
        }
        float o[TC_D / 2];
#pragma unroll
        for (int i = 0; i < TC_D / 2; ++i) o[i] = 0.f;
        float m_used[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_sum[2] = {0.f, 0.f};  // l_sum: this thread's columns only
        const int32_t *table = a.block_table + static_cast<size_t>(b) * a.max_pages;
        const uint32_t q_wg = q_base + wg * (64 * 128);  // this warpgroup's 64 rows of each 64-column half of Q
        if (n_tiles > 0) g_mbar_wait(q_full, 0);
        int s = 0;
        uint32_t ph = 0;
        for (int j = 0; j < n_tiles; ++j) {
            const int tile = tile_of(j);
            const int lp = tile / a.tiles_per_page;
            const int pid = table[lp];
            const bool page_ok = pid >= 0 && pid < a.num_pages;
            // ---- S = Q K_j^T: both operands K-major, two 64-wide halves of the head dimension
            float sc[TC_BN / 2];  // fp32 scores
#pragma unroll
            for (int i = 0; i < TC_BN / 2; ++i) sc[i] = 0.f;
            g_mbar_wait(k_full + 8 * s, ph);
            wgmma_reg_fence(sc);
            wgmma_fence();
            {
                const uint32_t kb = k_base + s * TC_KV_TILE;
#pragma unroll
                for (int k = 0; k < TC_D / 16; ++k) {
                    const uint32_t half = k >> 2, kk = k & 3;
                    Wgmma<T, TC_BN>::ss(sc, g_wgmma_desc(q_wg + half * (TC_Q_BYTES / 2) + 32 * kk, 16, 1024),
                                           g_wgmma_desc(kb + half * (TC_KV_TILE / 2) + 32 * kk, 16, 1024), k > 0 ? 1u : 0u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_reg_fence(sc);
            if (t == 0) g_mbar_arrive(k_empty + 8 * s);  // K stage reusable: this warpgroup's MMAs have read it
            // ---- softmax of the tile: sc[4 c8 + 2 rr + e] = S[row rr, key 8 c8 + 2 (t % 4) + e]
            const int key0 = tile * TC_BN;
            uint32_t pa[TC_BN / 16][4];  // bf16 probabilities as the A operand of the four P V K steps
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int visible = page_ok ? min(limit[rr] - key0 + 1, TC_BN) : 0;  // keys [0, visible) of the tile
                const int first = lo[rr] - key0;                                        // TC_SEGMENT: and not below first
                const int pfirst = pst[rr] - key0, pend = page_ok ? pen[rr] - key0 : 0;  // TC_PREFIXED: or in [pfirst, pend)
                // raw maximum (the scale is positive, so it commutes with max); masking only on boundary tiles
                float raw_max = -CUDART_INF_F;
#pragma unroll
                for (int c8 = 0; c8 < TC_BN / 8; ++c8)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float &v = sc[4 * c8 + 2 * rr + e];
                        const int c = 8 * c8 + 2 * (lane & 3) + e;
                        const bool masked = MODE == TC_PREFIXED ? (c >= visible || c < first) && (c < pfirst || c >= pend)
                                            : MODE == TC_SEGMENT ? (c >= visible || c < first) : (visible < TC_BN && c >= visible);
                        if (masked) v = -CUDART_INF_F;  // exp2 gives exactly 0
                        raw_max = fmaxf(raw_max, v);
                    }
                raw_max = fmaxf(raw_max, __shfl_xor_sync(0xffffffffu, raw_max, 1));
                raw_max = fmaxf(raw_max, __shfl_xor_sync(0xffffffffu, raw_max, 2));
                const float tile_max = raw_max * a.scale_log2;  // -inf stays -inf
                // lazy rescale: keep the stale maximum unless this tile exceeds it by more than 2^8
                const bool grow = tile_max > m_used[rr] + TC_RESCALE_THRESHOLD || (m_used[rr] == -CUDART_INF_F && tile_max != -CUDART_INF_F);
                if (grow) {
                    if (j > 0) {
                        const float alpha = m_used[rr] != -CUDART_INF_F ? exp2f(m_used[rr] - tile_max) : 0.f;
                        l_sum[rr] *= alpha;
#pragma unroll
                        for (int c8 = 0; c8 < TC_D / 8; ++c8) {
                            o[4 * c8 + 2 * rr] *= alpha;
                            o[4 * c8 + 2 * rr + 1] *= alpha;
                        }
                    }
                    m_used[rr] = tile_max;
                }
                const float m_eff = m_used[rr] == -CUDART_INF_F ? 0.f : m_used[rr];
                float tile_sum = 0.f;
#pragma unroll
                for (int c8 = 0; c8 < TC_BN / 8; ++c8) {
                    const float p0 = tc_ex2(fmaf(sc[4 * c8 + 2 * rr], a.scale_log2, -m_eff));
                    const float p1 = tc_ex2(fmaf(sc[4 * c8 + 2 * rr + 1], a.scale_log2, -m_eff));
                    tile_sum += p0 + p1;
                    // K step c8 / 2: registers {row r0, keys +0..7}, {r0 + 8, +0..7}, {r0, +8..15}, {r0 + 8, +8..15}
                    pa[c8 >> 1][2 * (c8 & 1) + rr] = pack2<T>(p0, p1);
                }
                l_sum[rr] += tile_sum;
            }
            // ---- O += P V: P from registers, V MN-major [64 keys x 128 d] as loaded from the page
            g_mbar_wait(v_full + 8 * s, ph);
            wgmma_reg_fence(o);
            wgmma_fence();
            {
                const uint32_t vb = v_base + s * TC_KV_TILE;
#pragma unroll
                for (int k = 0; k < TC_BN / 16; ++k)  // 16 keys = two 8-row groups of 128 B
                    Wgmma<T, TC_D, 1>::rs(o, pa[k], g_wgmma_desc(vb + k * 2048, TC_KV_TILE / 2, 1024), 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_reg_fence(o);
            if (t == 0) g_mbar_arrive(v_empty + 8 * s);
            if (++s == TC_STAGES) s = 0, ph ^= 1u;
        }
        // ---- epilogue: O / sum -> bf16 -> out[(b*Hq + head) * L + l, :]
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            float lt = l_sum[rr];
            lt += __shfl_xor_sync(0xffffffffu, lt, 1);
            lt += __shfl_xor_sync(0xffffffffu, lt, 2);
            if (l[rr] >= (MODE == TC_PREFIX ? grp.y : a.L)) continue;
            const size_t out_row = MODE == TC_PREFIX ? static_cast<size_t>(b + l[rr]) * a.Hq + kvh * a.G + g[rr]
                                                     : static_cast<size_t>(b * a.Hq + kvh * a.G + g[rr]) * a.L + l[rr];
            const int col = 2 * (lane & 3);
            if (MODE == TC_PREFIX || MODE == TC_SUFFIX || a.splits > 1) {  // unnormalised partial for the merge kernel (attention_decode.cu: paged_gqa_merge_kernel)
                const size_t slot = out_row * a.split_stride + a.split_base + split;
                float *po = a.ws_o + slot * TC_D;
#pragma unroll
                for (int c8 = 0; c8 < TC_D / 8; ++c8)
                    *reinterpret_cast<float2 *>(po + 8 * c8 + col) = make_float2(o[4 * c8 + 2 * rr], o[4 * c8 + 2 * rr + 1]);
                if ((lane & 3) == 0) {
                    a.ws_m[slot] = (m_used[rr] == -CUDART_INF_F || !row_valid[rr]) ? -1e30f : m_used[rr];
                    a.ws_l[slot] = row_valid[rr] ? lt : 0.f;
                }
            } else {
                const float inv = (lt == 0.f || !row_valid[rr]) ? 0.f : 1.0f / lt;
                T *dst = reinterpret_cast<T *>(a.out) + (a.out_token_major ? (static_cast<size_t>(b) * a.L + l[rr]) * a.Hq + (kvh * a.G + g[rr]) : out_row) * TC_D;
#pragma unroll
                for (int c8 = 0; c8 < TC_D / 8; ++c8)
                    *reinterpret_cast<uint32_t *>(dst + 8 * c8 + col) = pack2<T>(o[4 * c8 + 2 * rr] * inv, o[4 * c8 + 2 * rr + 1] * inv);
            }
        }
    }
}

// ---------------------------------------------------------------- host side --
// bf16 Q / K / V with the 128-byte swizzle (the K-major wgmma layout), 256-byte L2 promotion.
static int tc_map(CUtensorMap *out, const void *ptr, int rank, const cuuint64_t *dims, const cuuint32_t *box,
                  CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
    return cached_tensor_map(out, ptr, dtype, rank, dims, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             "paged_attention");
}

bool paged_prefill_tc_supported(int L, int num_pages, int page_size, int num_kv_heads, int num_heads) {
    if (num_kv_heads < 1 || num_heads % num_kv_heads != 0) return false;
    const int G = num_heads / num_kv_heads;
    if (G < 1 || G > TC_BM || (TC_BM % G) != 0) return false;
    return L > 0 && num_pages > 0 && page_size >= TC_BN && page_size % TC_BN == 0;
}

// allow_split: the key range of every (request, KV head) is cut into up to PAGED_MAX_SPLITS pieces so that a small batch
// still fills the GPU; the partials are combined by paged_gqa_merge_kernel.  Decode (L <= 8, head-major output) splits
// at any width; the token-major form of a prefill chunk only when the block table spans more than PREFILL_SPLIT_MIN_KEYS
// keys (a long prefix: unsplit, a 128-row chunk at Qwen3-4B shapes is 32 CTAs that each walk the whole prefix).  Causal
// masking stays per row inside a split; a split past a row's last visible key leaves an empty partial (m = -1e30, l = 0)
// that the merge weights by zero.  The split count comes from the block table's width and the tiles are dealt out from
// the real context inside the kernel, so a row's result does not depend on the graph's grid.
// Split count: the one that minimises waves x (tiles per CTA + fixed cost) + merge launch, in units of one 64-key tile,
// with one CTA slot per SM, ~3 tiles of fixed cost per CTA (set-up, Q load, epilogue) and 2 + splits / 4 for the merge
// launch (it reads one partial per split and row).  base: CTAs per split; at most max_splits.
static int tc_wave_splits(long long base, long long max_tiles, long long max_splits) {
    const long long slots = sm_count();
    long long best = 1, best_cost = -1;
    for (long long sp = 1; sp <= max_splits && sp <= (max_tiles > 1 ? max_tiles : 1); ++sp) {
        const long long tps = (max_tiles + sp - 1) / sp;
        const long long real = (max_tiles + tps - 1) / tps;
        if (real != sp) continue;
        const long long waves = (base * sp + slots - 1) / slots;
        const long long cost = 4 * waves * (tps + 3) + (sp > 1 ? 8 + sp : 0);  // x 4: quarter-tile units
        if (best_cost < 0 || cost < best_cost) best_cost = cost, best = sp;
    }
    return static_cast<int>(best);
}

size_t paged_token_major_workspace(int rows, int L, int page_size, int max_pages) {
    if (static_cast<long long>(max_pages) * page_size <= PREFILL_SPLIT_MIN_KEYS) return 0;
    return static_cast<size_t>(rows) * L * PAGED_MAX_SPLITS * (TC_D + 2) * sizeof(float);
}

int launch_paged_prefill_tc(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl, void *out, int rows,
                            int L, int num_pages, int page_size, int max_pages, float scale, int is_causal, int num_kv_heads,
                            int num_heads, bool allow_split, void *ws, size_t ws_bytes, cudaStream_t st, bool out_token_major) {
    const int G = num_heads / num_kv_heads;
    const int B = rows / num_heads;
    TcArgs a{};
    a.block_table = bt, a.context_lens = cl, a.out = static_cast<bf16 *>(out);
    a.L = L, a.Hq = num_heads, a.Hkv = num_kv_heads, a.G = G, a.RH = TC_BM / G;
    a.page_size = page_size, a.max_pages = max_pages, a.num_pages = num_pages;
    a.tiles_per_page = page_size / TC_BN;
    a.scale_log2 = scale * TC_LOG2E;
    a.is_causal = is_causal;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(paged_prefill_tc_kernel<TC_PLAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES) != cudaSuccess ||
            cudaFuncSetAttribute(paged_prefill_tc_kernel<TC_PLAIN>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess)
            return fail(TL_ECUDA, "paged_attention: cannot raise shared memory limit");
        configured = true;
    }
    CUtensorMap mq, mk, mv;
    {
        const cuuint64_t dims[3] = {TC_D, static_cast<cuuint64_t>(L), static_cast<cuuint64_t>(rows)};
        const cuuint32_t box[3] = {64, static_cast<cuuint32_t>(a.RH), static_cast<cuuint32_t>(G)};
        if (int e = tc_map(&mq, q, 3, dims, box)) return e;
    }
    {
        const cuuint64_t dims[4] = {TC_D, static_cast<cuuint64_t>(page_size), static_cast<cuuint64_t>(num_kv_heads), static_cast<cuuint64_t>(num_pages)};
        const cuuint32_t box[4] = {64, TC_BN, 1, 1};
        if (int e = tc_map(&mk, kp, 4, dims, box)) return e;
        if (int e = tc_map(&mv, vp, 4, dims, box)) return e;
    }
    const int q_blocks = (L + a.RH - 1) / a.RH;
    const long long max_tiles = (static_cast<long long>(max_pages) * page_size + TC_BN - 1) / TC_BN;
    a.out_token_major = out_token_major ? 1 : 0;
    a.splits = 1;
    a.split_stride = 1;
    a.tiles_per_split = static_cast<int>(max_tiles < 1 ? 1 : max_tiles);
    if (allow_split && ws != nullptr && (!out_token_major || static_cast<long long>(max_pages) * page_size > PREFILL_SPLIT_MIN_KEYS)) {
        const size_t rows_total = static_cast<size_t>(rows) * L;
        const long long fit = static_cast<long long>(ws_bytes / (rows_total * (TC_D + 2) * sizeof(float)));  // splits the workspace holds
        const int best = tc_wave_splits(static_cast<long long>(q_blocks) * num_kv_heads * B, max_tiles,
                                        fit < PAGED_MAX_SPLITS ? fit : PAGED_MAX_SPLITS);
        if (best > 1) {
            a.splits = a.split_stride = best, a.tiles_per_split = static_cast<int>((max_tiles + best - 1) / best);
            a.ws_o = static_cast<float *>(ws);
            a.ws_m = a.ws_o + rows_total * best * TC_D;
            a.ws_l = a.ws_m + rows_total * best;
        }
    }
    dim3 grid(q_blocks * a.splits, num_kv_heads, B);
    if (grid.y > 65535 || grid.z > 65535) return fail(TL_EINVAL, "paged_attention: too many heads / requests for one launch");
    cudaError_t le = launch_chained(paged_prefill_tc_kernel<TC_PLAIN>, grid, dim3(TC_THREADS), TC_SMEM_BYTES, st, mq, mk, mv, a);
    if (le != cudaSuccess) return fail(TL_ECUDA, "paged_attention: launch failed: %s", cudaGetErrorString(le));
    TL_LAUNCH_CHECK("paged_prefill_tc");
    if (a.splits > 1) return launch_paged_gqa_merge(a.ws_o, a.ws_m, a.ws_l, out, rows * L, a.splits, st, L, num_heads, out_token_major);
    return TL_OK;
}

// ---------------------------------------------------------------- shared-prefix attention --
// The split counts follow from the engine's shapes alone (one captured graph serves every grouping): the prefix pass
// sizes its splits by the wave model for one group over the whole table, the suffix pass for every slot over the whole
// table (a slot in no group attends all its keys there); the two share the PAGED_MAX_SPLITS slots of a row.
void shared_prefix_splits(int batch, int num_kv_heads, int page_size, int max_pages, int *prefix, int *suffix) {
    const long long max_tiles = static_cast<long long>(max_pages) * page_size / TC_BN;
    *prefix = tc_wave_splits(num_kv_heads, max_tiles, PAGED_MAX_SPLITS / 2);
    *suffix = tc_wave_splits(static_cast<long long>(batch) * num_kv_heads, max_tiles, PAGED_MAX_SPLITS - *prefix);
}

size_t shared_prefix_workspace(int batch, int num_heads, int num_kv_heads, int page_size, int max_pages) {
    int sp, ss;
    shared_prefix_splits(batch, num_kv_heads, page_size, max_pages, &sp, &ss);
    return static_cast<size_t>(batch) * num_heads * (sp + ss) * (TC_D + 2) * sizeof(float);
}

int launch_shared_prefix_attention(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl,
                                   const int32_t *groups, int num_groups, void *out, int batch, int num_pages, int page_size,
                                   int max_pages, float scale, int num_kv_heads, int num_heads, void *ws, cudaStream_t st) {
    const int G = num_heads / num_kv_heads;
    int sp, ss;
    shared_prefix_splits(batch, num_kv_heads, page_size, max_pages, &sp, &ss);
    const size_t rows_total = static_cast<size_t>(batch) * num_heads;
    TcArgs a{};
    a.block_table = bt, a.context_lens = cl, a.out = static_cast<bf16 *>(out);
    a.L = 1, a.Hq = num_heads, a.Hkv = num_kv_heads, a.G = G, a.RH = TC_BM / G;
    a.page_size = page_size, a.max_pages = max_pages, a.num_pages = num_pages;
    a.tiles_per_page = page_size / TC_BN;
    a.scale_log2 = scale * TC_LOG2E;
    a.is_causal = 1;
    a.groups = groups, a.num_groups = num_groups;
    a.split_stride = sp + ss;
    a.ws_o = static_cast<float *>(ws);
    a.ws_m = a.ws_o + rows_total * a.split_stride * TC_D;
    a.ws_l = a.ws_m + rows_total * a.split_stride;
    const int max_tiles = max_pages * page_size / TC_BN;
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(paged_prefill_tc_kernel<TC_PREFIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES) != cudaSuccess ||
            cudaFuncSetAttribute(paged_prefill_tc_kernel<TC_SUFFIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES) != cudaSuccess)
            return fail(TL_ECUDA, "shared_prefix_attention: cannot raise shared memory limit");
        configured = true;
    }
    CUtensorMap mq4, mq3, mk, mv;
    {
        const cuuint64_t dims[4] = {TC_D, static_cast<cuuint64_t>(G), static_cast<cuuint64_t>(num_kv_heads), static_cast<cuuint64_t>(batch)};
        const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(G), 1, static_cast<cuuint32_t>(a.RH)};
        if (int e = tc_map(&mq4, q, 4, dims, box)) return e;
    }
    {
        const cuuint64_t dims[3] = {TC_D, 1, static_cast<cuuint64_t>(rows_total)};
        const cuuint32_t box[3] = {64, static_cast<cuuint32_t>(a.RH), static_cast<cuuint32_t>(G)};
        if (int e = tc_map(&mq3, q, 3, dims, box)) return e;
    }
    {
        const cuuint64_t dims[4] = {TC_D, static_cast<cuuint64_t>(page_size), static_cast<cuuint64_t>(num_kv_heads), static_cast<cuuint64_t>(num_pages)};
        const cuuint32_t box[4] = {64, TC_BN, 1, 1};
        if (int e = tc_map(&mk, kp, 4, dims, box)) return e;
        if (int e = tc_map(&mv, vp, 4, dims, box)) return e;
    }
    a.splits = sp, a.split_base = 0, a.tiles_per_split = (max_tiles + sp - 1) / sp;
    cudaError_t le = launch_chained(paged_prefill_tc_kernel<TC_PREFIX>, dim3(sp, num_kv_heads, batch), dim3(TC_THREADS), TC_SMEM_BYTES, st,
                                    mq4, mk, mv, a);
    if (le != cudaSuccess) return fail(TL_ECUDA, "shared_prefix_attention: launch failed: %s", cudaGetErrorString(le));
    TL_LAUNCH_CHECK("shared_prefix_attention_prefix");
    a.splits = ss, a.split_base = sp, a.tiles_per_split = (max_tiles + ss - 1) / ss;
    le = launch_chained(paged_prefill_tc_kernel<TC_SUFFIX>, dim3(ss, num_kv_heads, batch), dim3(TC_THREADS), TC_SMEM_BYTES, st, mq3, mk, mv, a);
    if (le != cudaSuccess) return fail(TL_ECUDA, "shared_prefix_attention: launch failed: %s", cudaGetErrorString(le));
    TL_LAUNCH_CHECK("shared_prefix_attention_suffix");
    return launch_paged_gqa_merge(a.ws_o, a.ws_m, a.ws_l, out, static_cast<int>(rows_total), sp + ss, st, 1, num_heads, false);
}

// ---------------------------------------------------------------- segment-causal attention --
// One packed request of L rows (B = 1, the chunk form's q [Hq, L, D] and token-major out [L, Hq * D]) whose keys are its
// own rows 0 .. L - 1: row l sees segment_start[l] <= key <= l (TC_SEGMENT), and also prefix_start[l] <= key <
// prefix_end[l] (TC_PREFIXED).  Unsplit (a pass of L <= 8,192 rows spans at most as many keys): the q-block grid of
// launch_paged_prefill_tc at B = 1.
template <int MODE, typename T>
static int launch_segment_t(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *seg, const int32_t *pre_start,
                            const int32_t *pre_end, void *out, int L, int num_pages, int page_size, int max_pages, float scale,
                            int num_kv_heads, int num_heads, CUtensorMapDataType dt, cudaStream_t st, const char *op) {
    static bool configured = false;
    if (!configured) {
        if (cudaFuncSetAttribute(paged_prefill_tc_kernel<MODE, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES) != cudaSuccess)
            return fail(TL_ECUDA, "%s: cannot raise shared memory limit", op);
        configured = true;
    }
    TcArgs a{};
    a.block_table = bt, a.context_lens = nullptr, a.out = static_cast<bf16 *>(out);
    a.L = L, a.Hq = num_heads, a.Hkv = num_kv_heads, a.G = num_heads / num_kv_heads, a.RH = TC_BM / a.G;
    a.page_size = page_size, a.max_pages = max_pages, a.num_pages = num_pages;
    a.tiles_per_page = page_size / TC_BN;
    a.scale_log2 = scale * TC_LOG2E;
    a.is_causal = 1;
    a.splits = a.split_stride = 1;
    a.tiles_per_split = (max_pages * page_size + TC_BN - 1) / TC_BN;
    a.out_token_major = 1;
    a.segment_start = seg;
    a.prefix_start = pre_start, a.prefix_end = pre_end;
    CUtensorMap mq, mk, mv;
    {
        const cuuint64_t dims[3] = {TC_D, static_cast<cuuint64_t>(L), static_cast<cuuint64_t>(num_heads)};
        const cuuint32_t box[3] = {64, static_cast<cuuint32_t>(a.RH), static_cast<cuuint32_t>(a.G)};
        if (int e = tc_map(&mq, q, 3, dims, box, dt)) return e;
    }
    {
        const cuuint64_t dims[4] = {TC_D, static_cast<cuuint64_t>(page_size), static_cast<cuuint64_t>(num_kv_heads), static_cast<cuuint64_t>(num_pages)};
        const cuuint32_t box[4] = {64, TC_BN, 1, 1};
        if (int e = tc_map(&mk, kp, 4, dims, box, dt)) return e;
        if (int e = tc_map(&mv, vp, 4, dims, box, dt)) return e;
    }
    const dim3 grid((L + a.RH - 1) / a.RH, num_kv_heads, 1);
    cudaError_t le = launch_chained(paged_prefill_tc_kernel<MODE, T>, grid, dim3(TC_THREADS), TC_SMEM_BYTES, st, mq, mk, mv, a);
    if (le != cudaSuccess) return fail(TL_ECUDA, "%s: launch failed: %s", op, cudaGetErrorString(le));
    TL_LAUNCH_CHECK(op);
    return TL_OK;
}

int launch_paged_attention_segments(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *seg, void *out, int L,
                                    int num_pages, int page_size, int max_pages, float scale, int num_kv_heads, int num_heads, int dtype,
                                    cudaStream_t st) {
    const char *op = "paged_attention_segments";
    if (dtype == TL_F16)
        return launch_segment_t<TC_SEGMENT, __half>(q, kp, vp, bt, seg, nullptr, nullptr, out, L, num_pages, page_size, max_pages, scale,
                                                    num_kv_heads, num_heads, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, st, op);
    return launch_segment_t<TC_SEGMENT, bf16>(q, kp, vp, bt, seg, nullptr, nullptr, out, L, num_pages, page_size, max_pages, scale,
                                              num_kv_heads, num_heads, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, st, op);
}

int launch_paged_attention_prefixed_segments(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *seg,
                                             const int32_t *pre_start, const int32_t *pre_end, void *out, int L, int num_pages, int page_size,
                                             int max_pages, float scale, int num_kv_heads, int num_heads, int dtype, cudaStream_t st) {
    const char *op = "paged_attention_prefixed_segments";
    if (dtype == TL_F16)
        return launch_segment_t<TC_PREFIXED, __half>(q, kp, vp, bt, seg, pre_start, pre_end, out, L, num_pages, page_size, max_pages, scale,
                                                     num_kv_heads, num_heads, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, st, op);
    return launch_segment_t<TC_PREFIXED, bf16>(q, kp, vp, bt, seg, pre_start, pre_end, out, L, num_pages, page_size, max_pages, scale,
                                               num_kv_heads, num_heads, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, st, op);
}

}  // namespace tl
