// tl_lora_apply: per-row bf16 low-rank adapters added to a projection's output (contract: include/tiny_llm_b200.h,
// DESIGN.md section 12).  One launch per site; one cluster of LORA_CLUSTER CTAs per group of R rows.
//
//   shrink   every CTA stages its slice of the R input rows (N / LORA_CLUSTER elements each, whole 8-element chunks) in
//            shared memory.  A warp takes LORA_JB rows of A at a time; a lane walks its chunks of the slice in ascending
//            order with one 16-byte load of A per chunk and one fmaf per element, the warp adds its lanes with the xor
//            butterfly, and the CTA publishes nseg * r partial sums per row.
//   merge    after a cluster barrier every CTA adds the LORA_CLUSTER partials of each t_j in CTA order over distributed
//            shared memory and rounds t_j to T.  A second barrier keeps every CTA resident until its partials were read.
//   expand   each thread takes outputs o = rank * 256 + tid, + 2048, ...: 16-byte loads of B's row, fmaf over j ascending
//            against the broadcast t, then y = T(fmaf(sc, d, float(y))) and, with a residual, y = T(float(residual) + float(y)).
//
// The order of every sum depends on N, r and LORA_CLUSTER only, never on the row index, the row count or R: with R = 8
// (launches of more than 64 rows, whose 8-row groups usually belong to one prefill chunk and so to one adapter) the rows
// of a group share each load of A and B and are otherwise computed exactly as alone, so both routes give the same bits.
// A group whose rows name different adapters runs its rows one after the other.
//
// adapter_ids is read after griddepcontrol.wait, like x and y: nothing that depends on it can be requested earlier, and
// the part that does not (the site descriptor) travels as a kernel argument.
#include <cooperative_groups.h>

#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

namespace tl {

namespace {

constexpr int LORA_CLUSTER = 8;
constexpr int LORA_THREADS = 256;
constexpr int LORA_WARPS = LORA_THREADS / 32;
constexpr int LORA_JB = 4;                                            // rows of A in flight per warp
constexpr int LORA_MAX_N = 12288;                                     // input width: 1,536 staged elements per CTA and row
constexpr int LORA_SLICE = LORA_MAX_N / LORA_CLUSTER;
constexpr int LORA_MAX_J = TL_LORA_MAX_SEGMENTS * TL_LORA_MAX_RANK;  // 192 intermediates per row
constexpr int LORA_TILE_ROWS = 8;

using bf16 = __nv_bfloat16;

__device__ __forceinline__ uint4 ldg_nc(const uint4 *p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ void unpack8(const uint4 &v, float (&f)[8]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 p = unpack2<bf16>(w[k]);
        f[2 * k] = p.x;
        f[2 * k + 1] = p.y;
    }
}

struct Smem {
    uint4 xs[LORA_TILE_ROWS][LORA_SLICE / 8];
    float part[LORA_TILE_ROWS][LORA_MAX_J];
    float t[LORA_TILE_ROWS][LORA_MAX_J];
};

// Where the outputs live: segment s of row m at y[s] + m * ld[s] (the segments of one packed projection side by side, or
// one tensor per projection), the residual in the same layout.
struct Out {
    bf16 *y[TL_LORA_MAX_SEGMENTS];
    const bf16 *residual[TL_LORA_MAX_SEGMENTS];
    long long ld[TL_LORA_MAX_SEGMENTS];
};

// y[row] = T(residual[row] + y[row]) for the outputs of this CTA: rows without an adapter, when the launch carries the add.
__device__ void residual_only(const tl_lora_site &site, const Out &out, int row, int ktot, int rank) {
    for (int o = rank * LORA_THREADS + threadIdx.x; o < ktot; o += LORA_CLUSTER * LORA_THREADS) {
        int s = 0, os = o;
        while (os >= site.K[s]) os -= site.K[s], ++s;
        const size_t at = static_cast<size_t>(row) * out.ld[s] + os;
        out.y[s][at] = from_f<bf16>(to_f(ld_cg(out.residual[s] + at)) + to_f(ld_cg(out.y[s] + at)));
    }
}

// R consecutive rows from row0, all on adapter a >= 0 (rows >= nrows do not exist: staged as zeros, never stored).
template <int R>
__device__ void apply_rows(Smem &sm, cg::cluster_group &cluster, const tl_lora_site &site, const bf16 *x, const Out &out, int row0, int nrows,
                           int a) {
    const int rank = static_cast<int>(cluster.block_rank());
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int N = site.N, rmax = site.r_max, nseg = site.nseg;
    const int J = nseg * rmax;
    const int r_a = site.ranks[a];
    const int mask = site.seg_mask[a];
    const float sc = site.scales[a];

    // ---- shrink
    const int chunks = N / 8;
    const int per = (chunks + LORA_CLUSTER - 1) / LORA_CLUSTER;
    const int c0 = min(chunks, rank * per);
    const int nc = min(chunks, c0 + per) - c0;
    for (int i = threadIdx.x; i < R * nc; i += LORA_THREADS) {
        const int r = i / nc, c = i - r * nc;
        sm.xs[r][c] = r < nrows ? ld_cg(reinterpret_cast<const uint4 *>(x + static_cast<size_t>(row0 + r) * N) + c0 + c) : make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
    const uint4 *A = reinterpret_cast<const uint4 *>(static_cast<const bf16 *>(site.a) + static_cast<size_t>(a) * J * N) + c0;
    for (int j0 = warp * LORA_JB; j0 < J; j0 += LORA_WARPS * LORA_JB) {
        bool live[LORA_JB];
        bool any = false;
#pragma unroll
        for (int q = 0; q < LORA_JB; ++q) {
            const int j = j0 + q;
            live[q] = j < J && ((mask >> (j / rmax)) & 1) && (j % rmax) < r_a;
            any |= live[q];
        }
        if (!any) continue;
        float acc[LORA_JB][R];
#pragma unroll
        for (int q = 0; q < LORA_JB; ++q)
#pragma unroll
            for (int r = 0; r < R; ++r) acc[q][r] = 0.f;
        for (int c = lane; c < nc; c += 32) {
            uint4 av[LORA_JB];
#pragma unroll
            for (int q = 0; q < LORA_JB; ++q)
                if (live[q]) av[q] = ldg_nc(A + static_cast<size_t>(j0 + q) * chunks + c);
#pragma unroll
            for (int r = 0; r < R; ++r) {
                float xf[8];
                unpack8(sm.xs[r][c], xf);
#pragma unroll
                for (int q = 0; q < LORA_JB; ++q) {
                    if (!live[q]) continue;
                    float af[8];
                    unpack8(av[q], af);
#pragma unroll
                    for (int k = 0; k < 8; ++k) acc[q][r] = fmaf(af[k], xf[k], acc[q][r]);
                }
            }
        }
#pragma unroll
        for (int q = 0; q < LORA_JB; ++q) {
            if (!live[q]) continue;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const float s = warp_sum(acc[q][r]);
                if (lane == 0) sm.part[r][j0 + q] = s;
            }
        }
    }

    // ---- merge, in CTA order
    cluster.sync();
    for (int i = threadIdx.x; i < R * J; i += LORA_THREADS) {
        const int r = i / J, j = i - r * J;
        float s = 0.f;
        if (((mask >> (j / rmax)) & 1) && (j % rmax) < r_a) {
            for (int c = 0; c < LORA_CLUSTER; ++c) s += *cluster.map_shared_rank(&sm.part[r][j], c);
            s = to_f(from_f<bf16>(s));
        }
        sm.t[r][j] = s;
    }
    cluster.sync();  // no CTA overwrites its partials or leaves while another may still read them; also orders t for the CTA

    // ---- expand
    int ktot = 0;
    for (int s = 0; s < nseg; ++s) ktot += site.K[s];
    const int steps = r_a / 8;
    const bool with_residual = out.residual[0] != nullptr;
    for (int o = rank * LORA_THREADS + threadIdx.x; o < ktot; o += LORA_CLUSTER * LORA_THREADS) {
        int s = 0, os = o;
        while (os >= site.K[s]) os -= site.K[s], ++s;
        const bool hit = (mask >> s) & 1;
        float d[R];
#pragma unroll
        for (int r = 0; r < R; ++r) d[r] = 0.f;
        if (hit) {
            const uint4 *Brow = reinterpret_cast<const uint4 *>(static_cast<const bf16 *>(site.b[s]) +
                                                                (static_cast<size_t>(a) * site.K[s] + os) * rmax);
            for (int q = 0; q < steps; ++q) {
                float bf[8];
                unpack8(ldg_nc(Brow + q), bf);
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const float *t = &sm.t[r][s * rmax + q * 8];
#pragma unroll
                    for (int k = 0; k < 8; ++k) d[r] = fmaf(bf[k], t[k], d[r]);
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (r >= nrows) break;
            if (!hit && !with_residual) continue;
            const size_t at = static_cast<size_t>(row0 + r) * out.ld[s] + os;
            bf16 v = ld_cg(out.y[s] + at);
            if (hit) v = from_f<bf16>(__fmaf_rn(sc, d[r], to_f(v)));  // one fp32 rounding, as the contract states it
            if (with_residual) v = from_f<bf16>(to_f(ld_cg(out.residual[s] + at)) + to_f(v));
            out.y[s][at] = v;
        }
    }
}

template <int R>
__global__ void __launch_bounds__(LORA_THREADS) lora_apply_kernel(const bf16 *x, const __grid_constant__ Out out, const int32_t *adapter_ids,
                                                                  const __grid_constant__ tl_lora_site site, int M) {
    __shared__ Smem sm;
    griddep_launch();
    griddep_wait();  // x and y are the previous kernels' outputs: read through L2 (common.cuh: programmatic dependent launch)
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = static_cast<int>(cluster.block_rank());
    const int row0 = blockIdx.y * R;
    const int nrows = min(R, M - row0);
    int ktot = 0;
    for (int s = 0; s < site.nseg; ++s) ktot += site.K[s];

    const int first = ld_cg(adapter_ids + row0);
    bool uniform = true;
    if constexpr (R > 1) {
        for (int r = 1; r < nrows; ++r) uniform &= ld_cg(adapter_ids + row0 + r) == first;
    }
    if (uniform) {  // every CTA of the cluster reads the same ids, so all of them take the same branch (and the same barriers)
        if (first >= 0) {
            apply_rows<R>(sm, cluster, site, x, out, row0, nrows, first);
        } else if (out.residual[0] != nullptr) {
            for (int r = 0; r < nrows; ++r) residual_only(site, out, row0 + r, ktot, rank);
        }
        return;
    }
    if constexpr (R > 1) {
        for (int r = 0; r < nrows; ++r) {
            const int a = ld_cg(adapter_ids + row0 + r);
            if (a >= 0) {
                __syncthreads();  // the previous row's staged slice and t are no longer read
                apply_rows<1>(sm, cluster, site, x, out, row0 + r, 1, a);
            } else if (out.residual[0] != nullptr) {
                residual_only(site, out, row0 + r, ktot, rank);
            }
        }
    }
}

template <int R>
int launch_t(const void *x, const Out &out, const int32_t *adapter_ids, const tl_lora_site &site, int M, cudaStream_t st) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(LORA_CLUSTER, ceil_div(M, R));
    cfg.blockDim = dim3(LORA_THREADS);
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = LORA_CLUSTER;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 2 : 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, lora_apply_kernel<R>, static_cast<const bf16 *>(x), out, adapter_ids, site, M);
    if (e != cudaSuccess) return fail(TL_ECUDA, "lora_apply: launch failed: %s", cudaGetErrorString(e));
    TL_LAUNCH_CHECK("lora_apply");
    return TL_OK;
}

}  // namespace

int lora_route(int M, int dtype, const tl_lora_site *site) {
    if (dtype != TL_BF16) return fail(TL_EDTYPE, "lora_apply: activations must be bfloat16");
    if (!site) return fail(TL_EINVAL, "lora_apply: null site");
    if (M < 0 || M > 65535 * LORA_TILE_ROWS) return fail(TL_EINVAL, "lora_apply: bad row count %d", M);
    if (site->nseg < 1 || site->nseg > TL_LORA_MAX_SEGMENTS) return fail(TL_EINVAL, "lora_apply: a site has 1 to %d segments", TL_LORA_MAX_SEGMENTS);
    if (site->n_adapters < 1 || site->n_adapters > TL_LORA_MAX_ADAPTERS)
        return fail(TL_EINVAL, "lora_apply: a set holds 1 to %d adapters", TL_LORA_MAX_ADAPTERS);
    if (site->r_max < 8 || site->r_max > TL_LORA_MAX_RANK || site->r_max % 8 != 0)
        return fail(TL_EINVAL, "lora_apply: r_max must be a multiple of 8 in [8, %d]", TL_LORA_MAX_RANK);
    if (site->N <= 0 || site->N % 8 != 0 || site->N > LORA_MAX_N)
        return fail(TL_EINVAL, "lora_apply: input width %d must be a multiple of 8 up to %d", site->N, LORA_MAX_N);
    for (int s = 0; s < site->nseg; ++s)
        if (site->K[s] <= 0) return fail(TL_EINVAL, "lora_apply: segment %d has no outputs", s);
    return M > 64 ? TL_LORA_TILES : TL_LORA_ROWS;
}

int launch_lora_apply(const void *x, void *const *y, const void *const *residual, const long long *ldy, const int32_t *adapter_ids,
                      const tl_lora_site &site, int M, int route, cudaStream_t st) {
    Out out{};
    for (int s = 0; s < site.nseg; ++s) {
        out.y[s] = static_cast<bf16 *>(y[s]);
        out.residual[s] = residual ? static_cast<const bf16 *>(residual[s]) : nullptr;
        out.ld[s] = ldy[s];
    }
    return route == TL_LORA_TILES ? launch_t<LORA_TILE_ROWS>(x, out, adapter_ids, site, M, st) : launch_t<1>(x, out, adapter_ids, site, M, st);
}

}  // namespace tl
