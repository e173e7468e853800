// extern "C" entry points of libtiny_llm_b200.so (see include/tiny_llm_b200.h).
// Each launcher checks what can be checked from pointers and sizes, picks the
// kernel, enqueues it on the caller's stream and returns; it never allocates,
// synchronises or throws.
#include <stdarg.h>
#include <stdio.h>

#include <atomic>
#include <vector>

#include "common.cuh"
#include "kernels.h"
#include "trace.cuh"

namespace tl {

static thread_local char g_error[512] = "";
static std::atomic<long long> g_launches{0};

int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
    return code;
}

int check_launch(const char *what) {
    cudaError_t e = cudaPeekAtLastError();
    if (e == cudaSuccess) return TL_OK;
    cudaGetLastError();  // clear the sticky launch error so later calls can report their own
    return fail(TL_ECUDA, "%s: kernel launch failed: %s", what, cudaGetErrorString(e));
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
    static int cached = 0;
    if (cached == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            cached = n;
        else
            cached = 132;  // H100 SXM
    }
    return cached;
}

static bool float_dtype(int dtype) { return dtype == TL_F32 || dtype == TL_F16 || dtype == TL_BF16; }

// ------------------------------------------------------- kernel selection --
// W4A16 projections, by activation rows M: up to 8 the weight-streaming kernel (w4a16_matvec.cu, the reference's matvec
// limit, quantize.py:162-163); 9..128 the swap-AB wgmma kernel with the reduction split over CTAs (w4a16_skinny.cu),
// one token tile; above that the same kernel on 128-token tiles.  !use_simdgroup is the scalar control kernel.
// Row counts 9..128 share that kernel and its split count (a function of N and K), so the decode engine's 16-, 32- and
// 64-row graphs give a row the same bits.
constexpr int SKINNY_MIN_ROWS = TL_MATVEC_REF_ROWS + 1;
enum class W4Path { VANILLA, STREAM, SKINNY, TILES };

// `fused`: the call is one of the fused forms.  Only the split-reduction launch carries their epilogues, so they keep
// M > 128 on the streaming kernel.  The wgmma kernels read a plain [M, N] activation through TMA: a prologue or a row
// stride other than N needs the streaming kernel.
static W4Path w4a16_path(int M, int N, int K, int dtype, bool use_simdgroup, bool fused, int prologue, int lda) {
    if (!use_simdgroup) return W4Path::VANILLA;
    const bool wgmma = (dtype == TL_BF16 || dtype == TL_F16) && K > 0 && N % 128 == 0 && prologue == TL_PRO_NONE && lda == N;
    if (wgmma && M >= SKINNY_MIN_ROWS && M <= 128) return W4Path::SKINNY;
    if (wgmma && !fused && M > 128) return W4Path::TILES;
    return W4Path::STREAM;
}

// Paged attention.  bf16 with D = 128 has the tensor-core and GQA-grouped kernels, which read q and K/V in 16-byte
// vectors; everything else runs the row-wise kernel.  Decode steps (L <= PAGED_DECODE_ROWS) split each request's key
// range over CTAs so that a small batch still fills the GPU.  Their workspace follows from dtype and D alone
// (tl_paged_attention_workspace); pointer alignment only chooses between kernels that fit it.
enum class PagedPath { ROWWISE = TL_PAGED_ROWWISE, GQA = TL_PAGED_GQA, FLASH = TL_PAGED_FLASH, WGMMA = TL_PAGED_WGMMA };
constexpr int PAGED_D = 128;
constexpr int PAGED_DECODE_ROWS = 8;  // query positions of a decode step (the reference's decode branch, paged_attention.cpp:168)
// From this key range (max_pages x page_size) decode streams K/V through TMA into the wgmma kernel; below it the
// cp.async GQA kernel, whose fixed cost per CTA is lower, is faster.
constexpr long long PAGED_WGMMA_MIN_KEYS = 1024;

// `decode`: L <= PAGED_DECODE_ROWS on tl_paged_attention; the token-major form has only the unsplit wgmma kernel and
// passes false.
static PagedPath paged_attention_path(const void *q, const void *kp, const void *vp, const void *out, int rows, int L, int D, int num_pages,
                                      int page_size, int max_pages, int num_kv_heads, int num_heads, int dtype, bool decode) {
    if (dtype != TL_BF16 || D != PAGED_D || !aligned16(q) || !aligned16(kp) || !aligned16(vp)) return PagedPath::ROWWISE;
    const bool wgmma = aligned16(out) && paged_prefill_tc_supported(L, num_pages, page_size, num_kv_heads, num_heads);
    if (decode) {
        const bool one_tile = L <= 128 / (num_heads / num_kv_heads);  // the G x L query rows of a KV head fill one 128-row MMA tile
        return wgmma && one_tile && static_cast<long long>(max_pages) * page_size >= PAGED_WGMMA_MIN_KEYS ? PagedPath::WGMMA : PagedPath::GQA;
    }
    if (wgmma) return PagedPath::WGMMA;
    return rows <= 65535 ? PagedPath::FLASH : PagedPath::GQA;  // the mma.sync kernel puts the query rows on grid.y
}

}  // namespace tl

using namespace tl;

extern "C" {

int tl_abi_version(void) { return 1; }

const char *tl_last_error(void) { return g_error; }

long long tl_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int tl_device_info(int *sms, int *major, int *minor) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return fail(TL_ENODEVICE, "no CUDA device: %s", cudaGetErrorString(e));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return fail(TL_ENODEVICE, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (sms) *sms = prop.multiProcessorCount;
    if (major) *major = prop.major;
    if (minor) *minor = prop.minor;
    return TL_OK;
}

// ------------------------------------------------------------ W4A16 ------
// Every entry that takes packed weights has a *_bits sibling for 4- or 8-bit codes (group 128 at both widths); the
// entry without the suffix is its bits = 4 form.  The kernel choice does not depend on the width.
static bool bad_bits(int bits) { return bits != 4 && bits != 8; }
#define TL_CHECK_BITS(op) \
    if (bad_bits(bits)) return fail(TL_EINVAL, op ": bits must be 4 or 8 (got %d)", bits)

size_t tl_quantized_matmul_workspace(int M, int N, int K, int dtype, int use_simdgroup, int use_split_k) {
    return tl_quantized_matmul_workspace_bits(M, N, K, dtype, 4, use_simdgroup, use_split_k);
}

size_t tl_quantized_matmul_workspace_bits(int M, int N, int K, int dtype, int bits, int use_simdgroup, int /*use_split_k*/) {
    if (bad_bits(bits)) return 0;  // the launch refuses the width
    if (w4a16_path(M, N, K, dtype, use_simdgroup, false, TL_PRO_NONE, N) == W4Path::SKINNY) return w4a16_skinny_workspace(M, N, K);
    return 0;
}

int tl_quantized_matmul(const void *scales, const void *biases, const void *a, const void *b, void *out, int M, int N,
                        int K, int dtype, int use_simdgroup, int use_split_k, void *workspace, size_t workspace_bytes,
                        void *stream) {
    return tl_quantized_matmul_bits(scales, biases, a, b, out, M, N, K, dtype, 4, use_simdgroup, use_split_k, workspace, workspace_bytes, stream);
}

int tl_quantized_matmul_bits(const void *scales, const void *biases, const void *a, const void *b, void *out, int M, int N, int K, int dtype,
                             int bits, int use_simdgroup, int /*use_split_k*/, void *workspace, size_t workspace_bytes, void *stream) {
    if (dtype != TL_F16 && dtype != TL_BF16) return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
    TL_CHECK_BITS("quantized_matmul");
    if (M < 0 || N <= 0 || K < 0) return fail(TL_EINVAL, "quantized_matmul: negative dimension");
    if (N % 128 != 0) return fail(TL_EINVAL, "quantized_matmul: N must be divisible by group_size");
    if (!scales || !biases || !a || !b || !out) {
        if (M == 0 || K == 0) return TL_OK;
        return fail(TL_EINVAL, "quantized_matmul: null pointer");
    }
    cudaStream_t st = as_stream(stream);
    switch (w4a16_path(M, N, K, dtype, use_simdgroup, false, TL_PRO_NONE, N)) {
        case W4Path::VANILLA: return launch_w4a16_vanilla(scales, biases, a, b, out, M, N, K, dtype, st, bits);
        case W4Path::SKINNY:
            return launch_w4a16_skinny(scales, biases, a, b, out, nullptr, M, N, K, TL_EPI_NONE, dtype, workspace, workspace_bytes, st, nullptr, 0.f,
                                       nullptr, nullptr, nullptr, bits);
        case W4Path::TILES: return launch_w4a16_tiles(scales, biases, a, b, out, M, N, K, dtype, st, bits);
        case W4Path::STREAM: break;
    }
    return launch_w4a16_fused(scales, biases, b, out, a, nullptr, nullptr, M, N, K, N, TL_PRO_NONE, TL_EPI_NONE, 0.f, dtype, st, bits);
}

int tl_quantized_embedding(const void *indices, const void *scales, const void *biases, const void *weight, void *out,
                           int tokens, int vocab, int dim, int dtype, void *stream) {
    return tl_quantized_embedding_bits(indices, scales, biases, weight, out, tokens, vocab, dim, dtype, 4, stream);
}

int tl_quantized_embedding_bits(const void *indices, const void *scales, const void *biases, const void *weight, void *out, int tokens, int vocab,
                                int dim, int dtype, int bits, void *stream) {
    if (tokens < 0 || vocab <= 0 || dim <= 0 || dim % 128 != 0 || bad_bits(bits))
        return fail(TL_EINVAL, bits == 4 ? "quantized_embedding: expected 4-bit weights with group size 128"
                                         : "quantized_embedding: expected 4- or 8-bit weights with group size 128");
    if (tokens == 0) return TL_OK;
    if (!indices || !scales || !biases || !weight || !out) return fail(TL_EINVAL, "quantized_embedding: null pointer");
    if (bits == 8 && (reinterpret_cast<uintptr_t>(weight) & 7u) != 0) return fail(TL_EINVAL, "quantized_embedding: 8-bit weight must be 8-byte aligned");
    return launch_quantized_embedding(indices, scales, biases, weight, out, tokens, vocab, dim, dtype, as_stream(stream), bits);
}

// ----------------------------------------------------- fused model ops ----
int tl_rms_norm(const void *x, const void *weight, void *out, int rows, int dim, float eps, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "rms_norm: expected float32, float16, or bfloat16");
    if (rows < 0 || dim <= 0) return fail(TL_EINVAL, "rms_norm: bad shape");
    if (rows == 0) return TL_OK;
    if (!x || !weight || !out) return fail(TL_EINVAL, "rms_norm: null pointer");
    return launch_rms_norm(x, weight, out, rows, dim, eps, dtype, as_stream(stream));
}

int tl_rope(const void *x, const int32_t *offsets, void *out, int B, int L, int H, int D, int dims, float base,
            int traditional, int dtype, void *stream) {
    return tl_rope_table(x, offsets, out, B, L, H, D, dims, base, traditional, dtype, stream, nullptr);
}

int tl_rope_table(const void *x, const int32_t *offsets, void *out, int B, int L, int H, int D, int dims, float base,
                  int traditional, int dtype, void *stream, const double *inv_freq) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "rope: expected float32, float16, or bfloat16");
    if (B < 0 || L < 0 || H < 0 || D <= 0) return fail(TL_EINVAL, "rope: expected x=[B,L,H,D] and one int32 offset per batch row");
    if (dims <= 0 || dims > D || dims % 2 != 0)
        return fail(TL_EINVAL, "rope: dims must be positive, even, and no larger than the head dimension");
    if (static_cast<long long>(B) * L * H == 0) return TL_OK;
    if (!x || !offsets || !out) return fail(TL_EINVAL, "rope: null pointer");
    return launch_rope(x, offsets, out, B, L, H, D, dims, base, inv_freq, traditional, dtype, as_stream(stream));
}

int tl_rope_inv_freq(double *out, int head_dim, float base, void *stream) {
    if (head_dim <= 0 || head_dim % 2 != 0) return fail(TL_EINVAL, "rope_inv_freq: head_dim must be positive and even");
    if (!out) return fail(TL_EINVAL, "rope_inv_freq: null pointer");
    return launch_rope_inv_freq(out, head_dim / 2, base, as_stream(stream));
}

int tl_rms_norm_route(int dim, int dtype, const void *x, const void *weight, const void *out, int *vec) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "rms_norm: expected float32, float16, or bfloat16");
    if (dim <= 0) return fail(TL_EINVAL, "rms_norm: bad shape");
    bool v;
    const int tpr = rms_norm_path(dim, dtype, x, weight, out, &v);
    if (vec) *vec = v;
    return tpr;
}

int tl_rope_route(int B, int L, int H, int D, int dims, int dtype) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "rope: expected float32, float16, or bfloat16");
    if (B < 0 || L < 0 || H < 0 || D <= 0) return fail(TL_EINVAL, "rope: expected x=[B,L,H,D] and one int32 offset per batch row");
    if (dims <= 0 || dims > D || dims % 2 != 0)
        return fail(TL_EINVAL, "rope: dims must be positive, even, and no larger than the head dimension");
    return rope_heads_path(B, L, H, D, dims) ? TL_ROPE_HEADS : TL_ROPE_ELEMENT;
}

int tl_swiglu(const void *gate, const void *up, void *out, long long size, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "swiglu: expected float32, float16, or bfloat16");
    if (size < 0) return fail(TL_EINVAL, "swiglu: negative size");
    if (size == 0) return TL_OK;
    if (!gate || !up || !out) return fail(TL_EINVAL, "swiglu: null pointer");
    return launch_swiglu(gate, up, out, size, dtype, as_stream(stream));
}

int tl_add(const void *a, const void *b, void *out, long long size, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "add: expected float32, float16, or bfloat16");
    if (size < 0) return fail(TL_EINVAL, "add: negative size");
    if (size == 0) return TL_OK;
    if (!a || !b || !out) return fail(TL_EINVAL, "add: null pointer");
    return launch_add(a, b, out, size, dtype, as_stream(stream));
}

int tl_decode_attention(const void *q, const void *k, const void *v, const float *mask, void *out, int q_rows, int L,
                        int S, int D, int num_heads, int num_kv_heads, float scale, int is_causal, int has_mask,
                        int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "decode_attention: expected float32, float16, or bfloat16");
    if (q_rows < 0 || L < 0 || S < 0 || D <= 0 || D > 256 || num_heads <= 0 || num_kv_heads <= 0 ||
        num_heads % num_kv_heads != 0 || q_rows % num_heads != 0)
        return fail(TL_EINVAL, "decode_attention: incompatible attention shapes");
    if (static_cast<long long>(q_rows) * L == 0) return TL_OK;
    if (!q || !k || !v || !out || (has_mask && !mask)) return fail(TL_EINVAL, "decode_attention: null pointer");
    return launch_decode_attention(q, k, v, mask, out, q_rows, L, S, D, num_heads, num_kv_heads, scale, is_causal,
                                   has_mask, dtype, as_stream(stream));
}

// --------------------------------------------------------------- paged KV --
int tl_paged_cache_update(void *pages, const void *values, int num_pages, int heads, int page_size, int head_dim,
                          int length, int page_id, int start, int dtype, void *stream) {
    if (dtype != TL_F32 && dtype != TL_BF16)
        return fail(TL_EDTYPE, "paged_cache_update: pages and values must have the same float32 or bfloat16 dtype");
    if (num_pages <= 0 || heads <= 0 || page_size <= 0 || head_dim <= 0 || length < 0)
        return fail(TL_EINVAL, "paged_cache_update: expected pages [P, H, page_size, D] and values [1, H, length, D]");
    if (page_id < 0 || page_id >= num_pages || start < 0 || start + length > page_size)
        return fail(TL_EINVAL, "paged_cache_update: destination slice is outside page storage");
    if (length == 0) return TL_OK;
    if (!pages || !values) return fail(TL_EINVAL, "paged_cache_update: null pointer");
    return launch_paged_cache_update(pages, values, heads, page_size, head_dim, length, page_id, start, dtype,
                                     as_stream(stream));
}

int tl_paged_cache_append_decode(void *key_pages, void *value_pages, const void *keys, const void *values,
                                 const int32_t *block_table, const int32_t *context_lens, int batch, int num_pages,
                                 int heads, int page_size, int head_dim, int max_pages, int dtype, void *stream) {
    if (dtype != TL_F32 && dtype != TL_BF16)
        return fail(TL_EDTYPE, "paged_cache_append_decode: float32 or bfloat16 pages required");
    if (batch < 0 || num_pages <= 0 || heads <= 0 || page_size <= 0 || head_dim <= 0 || max_pages <= 0)
        return fail(TL_EINVAL, "paged_cache_append_decode: bad shape");
    if (batch == 0) return TL_OK;
    if (!key_pages || !value_pages || !keys || !values || !block_table || !context_lens)
        return fail(TL_EINVAL, "paged_cache_append_decode: null pointer");
    return launch_paged_cache_append_decode(key_pages, value_pages, keys, values, block_table, context_lens, batch,
                                            num_pages, heads, page_size, head_dim, max_pages, dtype, as_stream(stream));
}

int tl_paged_cache_append_chunk(void *key_pages, void *value_pages, const void *keys, const void *values,
                                const tl_page_span_list *spans, int num_pages, int heads, int page_size, int head_dim,
                                long long src_head_stride, long long src_token_stride, int dtype, void *stream) {
    if (dtype != TL_F32 && dtype != TL_BF16) return fail(TL_EDTYPE, "paged_cache_append_chunk: float32 or bfloat16 pages required");
    if (!spans || spans->n < 0 || spans->n > TL_PAGE_SPANS) return fail(TL_EINVAL, "paged_cache_append_chunk: bad span list");
    if (num_pages <= 0 || heads <= 0 || page_size <= 0 || head_dim <= 0 || src_token_stride < head_dim)
        return fail(TL_EINVAL, "paged_cache_append_chunk: bad shape");
    if (spans->n == 0) return TL_OK;
    if (!key_pages || !value_pages || !keys || !values) return fail(TL_EINVAL, "paged_cache_append_chunk: null pointer");
    for (int i = 0; i < spans->n; ++i)
        if (spans->page_id[i] < 0 || spans->page_id[i] >= num_pages || spans->start[i] < 0 || spans->count[i] < 0 || spans->src[i] < 0 ||
            spans->start[i] + spans->count[i] > page_size)
            return fail(TL_EINVAL, "paged_cache_append_chunk: destination slice is outside page storage");
    return launch_paged_cache_append_chunk(key_pages, value_pages, keys, values, *spans, heads, page_size, head_dim, src_head_stride,
                                           src_token_stride, dtype, as_stream(stream));
}

int tl_paged_cache_copy_prefix(const tl_kv_slab_table *slabs, const tl_prefix_copy_list *copies, int heads, int page_size,
                               int head_dim, int dtype, void *stream) {
    if (dtype != TL_F32 && dtype != TL_BF16) return fail(TL_EDTYPE, "paged_cache_copy_prefix: float32 or bfloat16 pages required");
    if (!slabs || slabs->n < 0 || slabs->n > TL_PREFIX_COPY_LAYERS) return fail(TL_EINVAL, "paged_cache_copy_prefix: bad slab table");
    if (!copies || copies->n < 0 || copies->n > TL_PREFIX_COPIES) return fail(TL_EINVAL, "paged_cache_copy_prefix: bad copy list");
    if (heads <= 0 || page_size <= 0 || head_dim <= 0) return fail(TL_EINVAL, "paged_cache_copy_prefix: bad shape");
    for (int i = 0; i < copies->n; ++i) {
        const int layer = copies->layer[i], src = copies->src[i], dst = copies->dst[i], slots = copies->slots[i];
        if (layer < 0 || layer >= slabs->n) return fail(TL_EINVAL, "paged_cache_copy_prefix: record %d names layer %d of %d", i, layer, slabs->n);
        if (!slabs->key[layer] || !slabs->value[layer]) return fail(TL_EINVAL, "paged_cache_copy_prefix: null slab of layer %d", layer);
        const int pages = slabs->num_pages[layer];
        if (src < 0 || src >= pages || dst < 0 || dst >= pages)
            return fail(TL_EINVAL, "paged_cache_copy_prefix: record %d: page outside the %d pages of layer %d", i, pages, layer);
        if (slots < 1 || slots > page_size)
            return fail(TL_EINVAL, "paged_cache_copy_prefix: record %d: slots %d outside [1, %d]", i, slots, page_size);
        if (src == dst) return fail(TL_EINVAL, "paged_cache_copy_prefix: record %d copies page %d onto itself", i, src);
        for (int j = 0; j < i; ++j) {
            if (copies->layer[j] != layer) continue;
            if (copies->dst[j] == dst)
                return fail(TL_EINVAL, "paged_cache_copy_prefix: destination page %d named twice in layer %d", dst, layer);
            if (copies->dst[j] == src || copies->src[j] == dst)  // the records would race within the launch
                return fail(TL_EINVAL, "paged_cache_copy_prefix: page %d is both a source and a destination in layer %d",
                            copies->dst[j] == src ? src : dst, layer);
        }
    }
    return launch_paged_cache_copy_prefix(*slabs, *copies, heads, page_size, head_dim, dtype, as_stream(stream));
}

size_t tl_paged_attention_workspace(int rows, int L, int D, int /*num_kv_heads*/, int /*num_heads*/, int dtype) {
    // partial O, running max and sum of every query row and split of the split-KV decode kernels
    if (L > PAGED_DECODE_ROWS || dtype != TL_BF16 || D != PAGED_D) return 0;
    return static_cast<size_t>(rows) * L * PAGED_MAX_SPLITS * (PAGED_D + 2) * sizeof(float);
}

static int check_paged_attention(int rows, int L, int D, int num_pages, int page_size, int max_pages, int num_kv_heads, int num_heads, int dtype) {
    if (dtype != TL_F32 && dtype != TL_BF16)
        return fail(TL_EDTYPE, "paged_attention: q, key_pages, and value_pages must have the same float32 or bfloat16 dtype");
    if (num_heads <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0)
        return fail(TL_EINVAL, "paged_attention: num_heads must be divisible by num_kv_heads");
    if (rows < 0 || rows % num_heads != 0) return fail(TL_EINVAL, "paged_attention: q.shape[0] must be divisible by num_heads");
    if (D <= 0 || D > 128) return fail(TL_EINVAL, "paged_attention: head dimension must be in the range [1, 128]");
    if (L < 0 || num_pages <= 0 || page_size <= 0 || max_pages <= 0) return fail(TL_EINVAL, "paged_attention: bad shape");
    if (L > 8 && dtype == TL_BF16 && D != 128)
        return fail(TL_EINVAL, "paged_attention: bfloat16 prefill requires head dimension 128");
    return TL_OK;
}

int tl_paged_attention_route(const void *q, const void *key_pages, const void *value_pages, const void *out, int rows, int L, int D,
                             int num_pages, int page_size, int max_pages, int num_kv_heads, int num_heads, int dtype) {
    if (int e = check_paged_attention(rows, L, D, num_pages, page_size, max_pages, num_kv_heads, num_heads, dtype)) return e;
    return static_cast<int>(paged_attention_path(q, key_pages, value_pages, out, rows, L, D, num_pages, page_size, max_pages, num_kv_heads,
                                                 num_heads, dtype, L <= PAGED_DECODE_ROWS));
}

int tl_paged_attention(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                       const int32_t *context_lens, void *out, int rows, int L, int D, int num_pages, int page_size,
                       int max_pages, float scale, int is_causal, int num_kv_heads, int num_heads, int dtype,
                       void *workspace, size_t workspace_bytes, void *stream) {
    if (int e = check_paged_attention(rows, L, D, num_pages, page_size, max_pages, num_kv_heads, num_heads, dtype)) return e;
    if (static_cast<long long>(rows) * L == 0) return TL_OK;
    if (!q || !key_pages || !value_pages || !block_table || !context_lens || !out)
        return fail(TL_EINVAL, "paged_attention: null pointer");
    cudaStream_t st = as_stream(stream);
    const bool decode = L <= PAGED_DECODE_ROWS;
    switch (paged_attention_path(q, key_pages, value_pages, out, rows, L, D, num_pages, page_size, max_pages, num_kv_heads, num_heads, dtype,
                                 decode)) {
        case PagedPath::WGMMA:
            return launch_paged_prefill_tc(q, key_pages, value_pages, block_table, context_lens, out, rows, L, num_pages, page_size, max_pages,
                                           scale, is_causal, num_kv_heads, num_heads, decode, workspace, workspace_bytes, st);
        case PagedPath::FLASH:
            return launch_paged_prefill_fa(q, key_pages, value_pages, block_table, context_lens, out, rows, L, num_pages, page_size, max_pages,
                                           scale, is_causal, num_kv_heads, num_heads, st);
        case PagedPath::GQA:
            return launch_paged_gqa(q, key_pages, value_pages, block_table, context_lens, out, rows, L, num_pages, page_size, max_pages, scale,
                                    is_causal, num_kv_heads, num_heads, decode, workspace, workspace_bytes, st);
        case PagedPath::ROWWISE: break;
    }
    return launch_paged_rowwise(q, key_pages, value_pages, block_table, context_lens, out, rows, L, D, num_pages, page_size, max_pages, scale,
                                is_causal, num_kv_heads, num_heads, dtype, st);
}

int tl_paged_attention_token_major(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                   const int32_t *context_lens, void *out, int rows, int L, int num_pages, int page_size, int max_pages,
                                   float scale, int is_causal, int num_kv_heads, int num_heads, void *stream) {
    return tl_paged_attention_token_major_split(q, key_pages, value_pages, block_table, context_lens, out, rows, L, num_pages, page_size,
                                                max_pages, scale, is_causal, num_kv_heads, num_heads, nullptr, 0, stream);
}

size_t tl_paged_attention_token_major_workspace(int rows, int L, int page_size, int max_pages) {
    if (rows <= 0 || L <= 0 || page_size <= 0 || max_pages <= 0) return 0;
    return paged_token_major_workspace(rows, L, page_size, max_pages);
}

int tl_paged_attention_token_major_split(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                         const int32_t *context_lens, void *out, int rows, int L, int num_pages, int page_size, int max_pages,
                                         float scale, int is_causal, int num_kv_heads, int num_heads, void *workspace, size_t workspace_bytes,
                                         void *stream) {
    if (num_heads <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0 || rows < 0 || rows % num_heads != 0 || L < 0 || num_pages <= 0 ||
        page_size <= 0 || max_pages <= 0)
        return fail(TL_EINVAL, "paged_attention_token_major: bad shape");
    if (static_cast<long long>(rows) * L == 0) return TL_OK;
    if (!q || !key_pages || !value_pages || !block_table || !context_lens || !out) return fail(TL_EINVAL, "paged_attention: null pointer");
    if (paged_attention_path(q, key_pages, value_pages, out, rows, L, PAGED_D, num_pages, page_size, max_pages, num_kv_heads, num_heads, TL_BF16,
                             false) != PagedPath::WGMMA)
        return fail(TL_EINVAL, "paged_attention_token_major: needs the wgmma kernel (bf16, D = 128, pages a multiple of 64 slots)");
    return launch_paged_prefill_tc(q, key_pages, value_pages, block_table, context_lens, out, rows, L, num_pages, page_size, max_pages, scale,
                                   is_causal, num_kv_heads, num_heads, workspace != nullptr, workspace, workspace_bytes, as_stream(stream), true);
}

size_t tl_shared_prefix_attention_workspace(int batch, int num_heads, int num_kv_heads, int page_size, int max_pages) {
    if (batch <= 0 || num_heads <= 0 || num_kv_heads <= 0 || page_size <= 0 || max_pages <= 0) return 0;
    return shared_prefix_workspace(batch, num_heads, num_kv_heads, page_size, max_pages);
}

int tl_shared_prefix_attention(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                               const int32_t *context_lens, const int32_t *groups, const int32_t *groups_host, int num_groups,
                               void *out, int batch, int D, int num_pages, int page_size, int max_pages, float scale,
                               int num_kv_heads, int num_heads, int dtype, void *workspace, size_t workspace_bytes, void *stream) {
    if (dtype != TL_BF16) return fail(TL_EDTYPE, "shared_prefix_attention: bfloat16 only");
    if (D != PAGED_D) return fail(TL_EINVAL, "shared_prefix_attention: head dimension must be %d", PAGED_D);
    if (num_heads <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0 || 128 % (num_heads / num_kv_heads) != 0)
        return fail(TL_EINVAL, "shared_prefix_attention: num_heads / num_kv_heads must be a whole divisor of 128");
    if (batch <= 0 || num_pages <= 0 || max_pages <= 0 || page_size <= 0 || page_size % 64 != 0)
        return fail(TL_EINVAL, "shared_prefix_attention: bad shape (page_size must be a multiple of 64)");
    if (num_groups < 0 || num_groups > batch) return fail(TL_EINVAL, "shared_prefix_attention: num_groups must be in [0, batch]");
    if (!q || !key_pages || !value_pages || !block_table || !context_lens || !out || !workspace || (num_groups > 0 && (!groups || !groups_host)))
        return fail(TL_EINVAL, "shared_prefix_attention: null pointer");
    const int G = num_heads / num_kv_heads;
    std::vector<char> taken(batch, 0);
    for (int i = 0; i < num_groups; ++i) {
        const int f = groups_host[3 * i], c = groups_host[3 * i + 1], sp = groups_host[3 * i + 2];
        if (c == 0) continue;
        if (c < 0 || f < 0 || f > batch - c) return fail(TL_EINVAL, "shared_prefix_attention: group %d leaves the slots [0, %d)", i, batch);
        if (static_cast<long long>(c) * G > 128)
            return fail(TL_EINVAL, "shared_prefix_attention: group %d has %d x %d query rows, more than 128", i, c, G);
        if (sp < 0 || sp > max_pages) return fail(TL_EINVAL, "shared_prefix_attention: group %d shares %d pages, outside [0, %d]", i, sp, max_pages);
        for (int b = f; b < f + c; ++b) {
            if (taken[b]) return fail(TL_EINVAL, "shared_prefix_attention: slot %d is in two groups", b);
            taken[b] = 1;
        }
    }
    if (workspace_bytes < shared_prefix_workspace(batch, num_heads, num_kv_heads, page_size, max_pages))
        return fail(TL_EINVAL, "shared_prefix_attention: workspace too small");
    return launch_shared_prefix_attention(q, key_pages, value_pages, block_table, context_lens, groups, num_groups, out, batch, num_pages,
                                          page_size, max_pages, scale, num_kv_heads, num_heads, workspace, as_stream(stream));
}

int tl_paged_attention_segments(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                const int32_t *segment_start, void *out, int L, int D, int num_pages, int page_size, int max_pages, float scale,
                                int num_kv_heads, int num_heads, int dtype, void *stream) {
    if (dtype != TL_BF16 && dtype != TL_F16) return fail(TL_EDTYPE, "paged_attention_segments: expected float16 or bfloat16");
    if (D != PAGED_D) return fail(TL_EINVAL, "paged_attention_segments: head dimension must be %d", PAGED_D);
    if (num_heads <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0 || 128 % (num_heads / num_kv_heads) != 0)
        return fail(TL_EINVAL, "paged_attention_segments: num_heads / num_kv_heads must be a whole divisor of 128");
    if (L < 0 || num_pages <= 0 || max_pages <= 0 || page_size <= 0 || page_size % 64 != 0)
        return fail(TL_EINVAL, "paged_attention_segments: bad shape (page_size must be a multiple of 64)");
    if (static_cast<long long>(L) > static_cast<long long>(max_pages) * page_size)
        return fail(TL_EINVAL, "paged_attention_segments: %d rows do not fit the block table's %d pages", L, max_pages);
    if (L == 0) return TL_OK;
    if (!q || !key_pages || !value_pages || !block_table || !segment_start || !out)
        return fail(TL_EINVAL, "paged_attention_segments: null pointer");
    if (!aligned16(q) || !aligned16(key_pages) || !aligned16(value_pages) || !aligned16(out))
        return fail(TL_EINVAL, "paged_attention_segments: q, pages and out must be 16-byte aligned");
    return launch_paged_attention_segments(q, key_pages, value_pages, block_table, segment_start, out, L, num_pages, page_size, max_pages, scale,
                                           num_kv_heads, num_heads, dtype, as_stream(stream));
}

int tl_embed_pool(const void *hidden, const void *norm_weight, float eps, const int32_t *segment_start, int num_segments, int rows, int hidden_size,
                  int dimensions, int pooling, int normalize, float *out, int dtype, void *stream) {
    if (dtype != TL_BF16 && dtype != TL_F16) return fail(TL_EDTYPE, "embed_pool: expected float16 or bfloat16");
    if (num_segments < 0 || rows < 0 || hidden_size <= 0 || hidden_size > TL_EMBED_MAX_HIDDEN)
        return fail(TL_EINVAL, "embed_pool: bad shape (hidden size must be in [1, %d])", TL_EMBED_MAX_HIDDEN);
    if (dimensions < 1 || dimensions > hidden_size) return fail(TL_EINVAL, "embed_pool: dimensions must be in [1, %d]", hidden_size);
    if (pooling != TL_EMBED_LAST && pooling != TL_EMBED_MEAN) return fail(TL_EINVAL, "embed_pool: pooling must be TL_EMBED_LAST or TL_EMBED_MEAN");
    if (num_segments == 0) return TL_OK;
    if (!hidden || !norm_weight || !segment_start || !out) return fail(TL_EINVAL, "embed_pool: null pointer");
    return launch_embed_pool(hidden, norm_weight, eps, segment_start, num_segments, rows, hidden_size, dimensions, pooling == TL_EMBED_MEAN,
                             normalize != 0, out, dtype, as_stream(stream));
}

int tl_paged_attention_prefixed_segments(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                         const int32_t *segment_start, const int32_t *prefix_start, const int32_t *prefix_end, void *out, int L,
                                         int D, int num_pages, int page_size, int max_pages, float scale, int num_kv_heads, int num_heads,
                                         int dtype, void *stream) {
    const char *op = "paged_attention_prefixed_segments";
    if (dtype != TL_BF16 && dtype != TL_F16) return fail(TL_EDTYPE, "%s: expected float16 or bfloat16", op);
    if (D != PAGED_D) return fail(TL_EINVAL, "%s: head dimension must be %d", op, PAGED_D);
    if (num_heads <= 0 || num_kv_heads <= 0 || num_heads % num_kv_heads != 0 || 128 % (num_heads / num_kv_heads) != 0)
        return fail(TL_EINVAL, "%s: num_heads / num_kv_heads must be a whole divisor of 128", op);
    if (L < 0 || num_pages <= 0 || max_pages <= 0 || page_size <= 0 || page_size % 64 != 0)
        return fail(TL_EINVAL, "%s: bad shape (page_size must be a multiple of 64)", op);
    if (static_cast<long long>(L) > static_cast<long long>(max_pages) * page_size)
        return fail(TL_EINVAL, "%s: %d rows do not fit the block table's %d pages", op, L, max_pages);
    if (L == 0) return TL_OK;
    if (!q || !key_pages || !value_pages || !block_table || !segment_start || !prefix_start || !prefix_end || !out)
        return fail(TL_EINVAL, "%s: null pointer", op);
    if (!aligned16(q) || !aligned16(key_pages) || !aligned16(value_pages) || !aligned16(out))
        return fail(TL_EINVAL, "%s: q, pages and out must be 16-byte aligned", op);
    return launch_paged_attention_prefixed_segments(q, key_pages, value_pages, block_table, segment_start, prefix_start, prefix_end, out, L,
                                                    num_pages, page_size, max_pages, scale, num_kv_heads, num_heads, dtype, as_stream(stream));
}

int tl_select_logits(const void *hidden, const void *norm_weight, float eps, const int32_t *row_index, int n, int rows, int hidden_size,
                     const void *weight, const void *scales, const void *biases, int vocab, int bits, const int32_t *token_ids, int m,
                     float *logits, float *logprobs, int dtype, void *stream) {
    if (dtype != TL_BF16 && dtype != TL_F16) return fail(TL_EDTYPE, "select_logits: expected float16 or bfloat16");
    if (bits != 4 && bits != 8) return fail(TL_EINVAL, "select_logits: bits must be 4 or 8, got %d", bits);
    if (m < 1 || m > TL_SELECT_MAX_IDS) return fail(TL_EINVAL, "select_logits: %d token ids, expected 1 to %d", m, TL_SELECT_MAX_IDS);
    if (hidden_size <= 0 || hidden_size > TL_EMBED_MAX_HIDDEN || hidden_size % 128 != 0)
        return fail(TL_EINVAL, "select_logits: hidden size %d is not a multiple of 128 in [128, %d]", hidden_size, TL_EMBED_MAX_HIDDEN);
    if (n < 0 || rows < 0 || vocab <= 0) return fail(TL_EINVAL, "select_logits: bad shape");
    if (n == 0) return TL_OK;
    if (!hidden || !norm_weight || !row_index || !weight || !scales || !biases || !token_ids || !logits || !logprobs)
        return fail(TL_EINVAL, "select_logits: null pointer");
    return launch_select_logits(hidden, norm_weight, eps, row_index, n, rows, hidden_size, weight, scales, biases, vocab, bits, token_ids, m,
                                logits, logprobs, dtype, as_stream(stream));
}

// ------------------------------------------------------------------ misc --
size_t tl_argmax_workspace(int rows, int vocab) { return argmax_workspace(rows, vocab); }

int tl_argmax(const void *logits, int32_t *out_tokens, int rows, int vocab, int dtype, void *workspace,
              size_t workspace_bytes, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "argmax: expected float32, float16, or bfloat16");
    if (rows < 0 || vocab <= 0) return fail(TL_EINVAL, "argmax: bad shape");
    if (rows == 0) return TL_OK;
    if (!logits || !out_tokens) return fail(TL_EINVAL, "argmax: null pointer");
    return launch_argmax(logits, out_tokens, rows, vocab, dtype, workspace, workspace_bytes, as_stream(stream));
}

int tl_sample(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
              const int32_t *positions, int32_t *out_tokens, int rows, int vocab, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "sample: expected float32, float16, or bfloat16");
    if (rows < 0 || rows > 65535 || vocab <= 0) return fail(TL_EINVAL, "sample: bad shape");
    if (int e = sample_plan(vocab, nullptr, nullptr)) return e;
    if (rows == 0) return TL_OK;
    if (!logits || !temperature || !top_k || !top_p || !seed || !positions || !out_tokens) return fail(TL_EINVAL, "sample: null pointer");
    return launch_sample(logits, temperature, top_k, top_p, seed, positions, out_tokens, rows, vocab, dtype, as_stream(stream));
}

int tl_sample_penalized(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                        const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                        const float *min_p, int32_t *state, int32_t *out_tokens, int rows, int vocab, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "sample_penalized: expected float32, float16, or bfloat16");
    if (rows < 0 || rows > 65535 || vocab <= 0) return fail(TL_EINVAL, "sample_penalized: bad shape");
    if (int e = sample_plan(vocab, nullptr, nullptr)) return e;
    if (rows == 0) return TL_OK;
    if (!logits || !temperature || !top_k || !top_p || !seed || !positions || !repetition || !presence || !frequency || !min_p || !state ||
        !out_tokens)
        return fail(TL_EINVAL, "sample_penalized: null pointer");
    return launch_sample_penalized(logits, temperature, top_k, top_p, seed, positions, repetition, presence, frequency, min_p, state,
                                   out_tokens, rows, vocab, dtype, as_stream(stream));
}

int tl_sample_constrained(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                          const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                          const float *min_p, int32_t *state, tl_constraint_row *constraints, int32_t *out_tokens, int rows, int vocab,
                          int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "sample_constrained: expected float32, float16, or bfloat16");
    if (rows < 0 || rows > 65535 || vocab <= 0) return fail(TL_EINVAL, "sample_constrained: bad shape");
    if (int e = sample_plan(vocab, nullptr, nullptr)) return e;
    if (rows == 0) return TL_OK;
    if (!logits || !temperature || !top_k || !top_p || !seed || !positions || !constraints || !out_tokens)
        return fail(TL_EINVAL, "sample_constrained: null pointer");
    const int given = !!repetition + !!presence + !!frequency + !!min_p + !!state;
    if (given != 0 && given != 5) return fail(TL_EINVAL, "sample_constrained: give every penalty array and the state, or none");
    return launch_sample_constrained(logits, temperature, top_k, top_p, seed, positions, repetition, presence, frequency, min_p, state,
                                     constraints, out_tokens, rows, vocab, dtype, as_stream(stream));
}

int tl_speculative_sample(const void *target, const void *draft, const int32_t *proposals, const float *temperature,
                          const int32_t *top_k, const float *top_p, const int64_t *seed, const int32_t *positions, int32_t *out_tokens,
                          int rows, int vocab, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "speculative_sample: expected float32, float16, or bfloat16");
    if (rows < 0 || rows > 65535 || vocab <= 0) return fail(TL_EINVAL, "speculative_sample: bad shape");
    if (int e = speculative_sample_plan(vocab, nullptr, nullptr)) return e;
    if (rows == 0) return TL_OK;
    if (!target || !temperature || !top_k || !top_p || !seed || !positions || !out_tokens || (rows > 1 && (!draft || !proposals)))
        return fail(TL_EINVAL, "speculative_sample: null pointer");
    return launch_speculative_sample(target, draft, proposals, temperature, top_k, top_p, seed, positions, out_tokens, rows, vocab, dtype,
                                     as_stream(stream));
}

int tl_log_rows(const void *src, void *dst, const int32_t *out_index, int capacity, long long bytes, void *stream) {
    if (capacity < 0 || bytes < 0) return fail(TL_EINVAL, "log_rows: bad shape");
    if (bytes == 0 || capacity == 0) return TL_OK;
    if (!src || !dst || !out_index) return fail(TL_EINVAL, "log_rows: null pointer");
    return launch_log_rows(src, dst, out_index, capacity, bytes, as_stream(stream));
}

int tl_ngram_propose(int32_t *history, int capacity, int length, const int32_t *appended, int n_appended, int k, int n_min, int n_max,
                     int32_t *out, int32_t *state, void *onehot, int vocab, int dtype, int grid, void *stream) {
    if (k < 1 || k > TL_NGRAM_MAX_K) return fail(TL_EINVAL, "ngram_propose: k must be in [1, %d]", TL_NGRAM_MAX_K);
    if (n_min < 1 || n_min > n_max || n_max > TL_NGRAM_MAX_N)
        return fail(TL_EINVAL, "ngram_propose: need 1 <= n_min <= n_max <= %d", TL_NGRAM_MAX_N);
    if (n_appended < 0 || n_appended > TL_NGRAM_MAX_APPEND)
        return fail(TL_EINVAL, "ngram_propose: at most %d appended tokens", TL_NGRAM_MAX_APPEND);
    if (length < 0 || capacity < 0 || static_cast<long long>(length) + n_appended > capacity)
        return fail(TL_EINVAL, "ngram_propose: %d + %d tokens exceed the history's capacity %d", length, n_appended, capacity);
    if (grid < 0) return fail(TL_EINVAL, "ngram_propose: grid must be >= 0");
    if (!history || !out || !state || (n_appended > 0 && !appended)) return fail(TL_EINVAL, "ngram_propose: null pointer");
    if (reinterpret_cast<uintptr_t>(state) % 8 != 0) return fail(TL_EINVAL, "ngram_propose: state must be 8-byte aligned");
    if (onehot) {
        if (!float_dtype(dtype)) return fail(TL_EDTYPE, "ngram_propose: expected float32, float16, or bfloat16");
        if (vocab < 1 || vocab > TL_NGRAM_MAX_VOCAB) return fail(TL_EINVAL, "ngram_propose: vocab must be in [1, %d]", TL_NGRAM_MAX_VOCAB);
    }
    return launch_ngram_propose(history, length, appended, n_appended, k, n_min, n_max, out, state, onehot, vocab, dtype, grid,
                                as_stream(stream));
}

int tl_beam_select(const float *top_lp, const int32_t *top_ids, float *cum, int rows, int n, int num_beams, const int32_t *eos_ids,
                   int num_eos, int32_t *result, void *stream) {
    if (num_beams < 1 || num_beams > TL_BEAM_MAX_WIDTH) return fail(TL_EINVAL, "beam_select: num_beams must be in [1, %d]", TL_BEAM_MAX_WIDTH);
    if (num_eos < 0 || num_eos > TL_BEAM_MAX_EOS) return fail(TL_EINVAL, "beam_select: at most %d EOS ids", TL_BEAM_MAX_EOS);
    if (rows < 1 || rows > num_beams) return fail(TL_EINVAL, "beam_select: rows must be in [1, num_beams = %d]", num_beams);
    if (n != num_beams + num_eos) return fail(TL_EINVAL, "beam_select: n must be num_beams + num_eos = %d", num_beams + num_eos);
    if (!top_lp || !top_ids || !cum || !result || (num_eos > 0 && !eos_ids)) return fail(TL_EINVAL, "beam_select: null pointer");
    for (int e = 0; e < num_eos; ++e) {
        if (eos_ids[e] < 0) return fail(TL_EINVAL, "beam_select: EOS ids must be non-negative");
        for (int f = 0; f < e; ++f)
            if (eos_ids[f] == eos_ids[e]) return fail(TL_EINVAL, "beam_select: EOS id %d given twice", eos_ids[e]);
    }
    return launch_beam_select(top_lp, top_ids, cum, rows, n, num_beams, eos_ids, num_eos, result, as_stream(stream));
}

int tl_constraint_token_masks(const int32_t *dfa, const uint8_t *accept, int num_states, const int32_t *token_offsets,
                              const uint8_t *token_bytes, int vocab, const int32_t *eos_ids, int num_eos, uint32_t *masks, uint32_t *reach,
                              void *stream) {
    if (num_states <= 0 || vocab <= 0 || num_eos < 0) return fail(TL_EINVAL, "constraint_token_masks: bad shape");
    if (!dfa || !accept || !token_offsets || !token_bytes || (num_eos > 0 && !eos_ids) || !masks || !reach)
        return fail(TL_EINVAL, "constraint_token_masks: null pointer");
    return launch_constraint_token_masks(dfa, accept, num_states, token_offsets, token_bytes, vocab, eos_ids, num_eos, masks, reach,
                                         as_stream(stream));
}

int tl_json_token_masks(const tl_constraint_row *constraints, const int64_t *json_states, int rows, int vocab, void *stream) {
    if (rows < 0 || rows > 65535 || vocab <= 0) return fail(TL_EINVAL, "json_token_masks: bad shape");
    if (rows > 0 && (!constraints || !json_states)) return fail(TL_EINVAL, "json_token_masks: null pointer");
    return launch_json_token_masks(constraints, json_states, rows, vocab, as_stream(stream));
}

int tl_json_advance(const tl_constraint_row *constraints, int64_t *json_states, const int32_t *tokens, const int32_t *positions, int rows,
                    void *stream) {
    if (rows < 0) return fail(TL_EINVAL, "json_advance: bad shape");
    if (rows > 0 && (!constraints || !json_states || !tokens || !positions)) return fail(TL_EINVAL, "json_advance: null pointer");
    return launch_json_advance(constraints, json_states, tokens, positions, rows, as_stream(stream));
}

int tl_schema_token_masks(const tl_constraint_row *constraints, const int64_t *schema_states, int rows, int vocab, int smem_bytes,
                          void *stream) {
    if (rows < 0 || rows > 65535 || vocab <= 0) return fail(TL_EINVAL, "schema_token_masks: bad shape");
    if (smem_bytes < 0 || smem_bytes > TL_SCHEMA_SMEM_BYTES || smem_bytes % 16) return fail(TL_EINVAL, "schema_token_masks: bad smem_bytes");
    if (rows > 0 && (!constraints || !schema_states)) return fail(TL_EINVAL, "schema_token_masks: null pointer");
    return launch_schema_token_masks(constraints, schema_states, rows, vocab, smem_bytes, as_stream(stream));
}

int tl_schema_advance(const tl_constraint_row *constraints, int64_t *schema_states, const int32_t *tokens, const int32_t *positions,
                      int rows, void *stream) {
    if (rows < 0) return fail(TL_EINVAL, "schema_advance: bad shape");
    if (rows > 0 && (!constraints || !schema_states || !tokens || !positions)) return fail(TL_EINVAL, "schema_advance: null pointer");
    return launch_schema_advance(constraints, schema_states, tokens, positions, rows, as_stream(stream));
}

int tl_logprobs(const void *logits, const int32_t *targets, const int32_t *top_n, const int32_t *out_index, float *lse, float *target_lp,
                int32_t *target_rank, int32_t *top_ids, float *top_lp, int rows, int vocab, int max_n, int out_capacity, int dtype,
                void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "logprobs: expected float32, float16, or bfloat16");
    if (rows < 0 || rows > 65535 || vocab <= 0) return fail(TL_EINVAL, "logprobs: bad shape");
    if (max_n < 0 || max_n > TL_LOGPROBS_MAX_N) return fail(TL_EINVAL, "logprobs: max_n must be in [0, %d]", TL_LOGPROBS_MAX_N);
    if (out_index && out_capacity < 0) return fail(TL_EINVAL, "logprobs: bad out_capacity");
    if (int e = sample_plan(vocab, nullptr, nullptr)) return e;
    if (rows == 0) return TL_OK;
    if (!logits || !lse || !target_lp || !target_rank || (max_n > 0 && (!top_ids || !top_lp))) return fail(TL_EINVAL, "logprobs: null pointer");
    return launch_logprobs(logits, targets, top_n, out_index, lse, target_lp, target_rank, top_ids, top_lp, rows, vocab, max_n,
                           out_index ? out_capacity : 1, dtype, as_stream(stream));
}

int tl_quantized_matmul_route(int M, int N, int K, int lda, int prologue, int fused, int use_simdgroup, int dtype, const void *a, const void *b,
                              const void *scales, const void *biases, int *splits, int *gb_per_split, int *rows_per_pass, int *units) {
    return tl_quantized_matmul_route_bits(M, N, K, lda, prologue, fused, use_simdgroup, dtype, 4, a, b, scales, biases, splits, gb_per_split,
                                          rows_per_pass, units);
}

int tl_quantized_matmul_route_bits(int M, int N, int K, int lda, int prologue, int fused, int use_simdgroup, int dtype, int bits, const void *a,
                                   const void *b, const void *scales, const void *biases, int *splits, int *gb_per_split, int *rows_per_pass,
                                   int *units) {
    if (dtype != TL_F16 && dtype != TL_BF16) return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
    TL_CHECK_BITS("quantized_matmul_route");
    if (M < 0 || N <= 0 || K < 0 || lda < N || N % 128 != 0) return fail(TL_EINVAL, "quantized_matmul_route: bad shape");
    if (prologue < TL_PRO_NONE || prologue > TL_PRO_SWIGLU || (!fused && (prologue != TL_PRO_NONE || lda != N)))
        return fail(TL_EINVAL, "quantized_matmul_route: a prologue or a row stride needs a fused form");
    int s = 0, gbps = 0, rpp = 0, u = 0;
    const W4Path path = w4a16_path(M, N, K, dtype, use_simdgroup != 0, fused != 0, prologue, lda);
    if (path == W4Path::SKINNY || path == W4Path::TILES) {
        if (!aligned16(a) || !aligned16(b)) return fail(TL_EINVAL, "quantized_matmul: a and b must be 16-byte aligned");
        if (path == W4Path::SKINNY)
            s = w4a16_skinny_splits(M, N, K, &gbps);
        else
            s = 1, gbps = N / 128;
    } else if (path == W4Path::STREAM) {
        if (int e = w4a16_stream_plan(M, N, K, lda, a, nullptr, b, scales, biases, &rpp, &u, bits)) return e;
    }
    if (splits) *splits = s;
    if (gb_per_split) *gb_per_split = gbps;
    if (rows_per_pass) *rows_per_pass = rpp;
    if (units) *units = u;
    switch (path) {
        case W4Path::VANILLA: return TL_W4_VANILLA;
        case W4Path::STREAM: return TL_W4_STREAM;
        case W4Path::SKINNY: return TL_W4_SKINNY;
        case W4Path::TILES: break;
    }
    return TL_W4_TILES;
}

size_t tl_quantized_matmul_fused_workspace(int M, int N, int K, int lda, int prologue, int dtype) {
    return tl_quantized_matmul_fused_workspace_bits(M, N, K, lda, prologue, dtype, 4);
}

size_t tl_quantized_matmul_fused_workspace_bits(int M, int N, int K, int lda, int prologue, int dtype, int bits) {
    if (bad_bits(bits)) return 0;  // the launch refuses the width
    if (w4a16_path(M, N, K, dtype, true, true, prologue, lda) == W4Path::SKINNY) return w4a16_skinny_workspace(M, N, K);
    return 0;
}

int tl_quantized_matmul_fused(const void *scales, const void *biases, const void *b, void *out, const void *p0,
                              const void *p1, const void *residual, int M, int N, int K, int lda, int prologue,
                              int epilogue, float eps, int dtype, void *workspace, size_t workspace_bytes, void *stream) {
    return tl_quantized_matmul_fused_bits(scales, biases, b, out, p0, p1, residual, M, N, K, lda, prologue, epilogue, eps, dtype, 4, workspace,
                                          workspace_bytes, stream);
}

int tl_quantized_matmul_fused_bits(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *p1,
                                   const void *residual, int M, int N, int K, int lda, int prologue, int epilogue, float eps, int dtype, int bits,
                                   void *workspace, size_t workspace_bytes, void *stream) {
    if (dtype != TL_F16 && dtype != TL_BF16) return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
    TL_CHECK_BITS("quantized_matmul_fused");
    if (M < 0 || N <= 0 || K < 0 || lda < N) return fail(TL_EINVAL, "quantized_matmul_fused: bad shape");
    if (N % 128 != 0) return fail(TL_EINVAL, "quantized_matmul: N must be divisible by group_size");
    if (prologue < TL_PRO_NONE || prologue > TL_PRO_SWIGLU || epilogue < TL_EPI_NONE || epilogue > TL_EPI_SWIGLU_PAIRS)
        return fail(TL_EINVAL, "quantized_matmul_fused: unknown prologue/epilogue");
    if (epilogue == TL_EPI_SWIGLU_PAIRS && K % 16 != 0)
        return fail(TL_EINVAL, "quantized_matmul_fused: interleaved gate|up rows need K %% 16 == 0");
    if (M == 0 || K == 0) return TL_OK;
    if (!scales || !biases || !b || !out || !p0 || (prologue != TL_PRO_NONE && !p1) || (epilogue == TL_EPI_RESIDUAL && !residual))
        return fail(TL_EINVAL, "quantized_matmul_fused: null pointer");
    if (w4a16_path(M, N, K, dtype, true, true, prologue, lda) == W4Path::SKINNY)
        return launch_w4a16_skinny(scales, biases, p0, b, out, residual, M, N, K, epilogue, dtype, workspace, workspace_bytes, as_stream(stream), nullptr,
                                   0.f, nullptr, nullptr, nullptr, bits);
    return launch_w4a16_fused(scales, biases, b, out, p0, p1, residual, M, N, K, lda, prologue, epilogue, eps, dtype,
                              as_stream(stream), bits);
}

int tl_quantized_matmul_residual_norm(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *residual,
                                      const void *norm_weight, void *normed_out, int M, int N, int K, float norm_eps, int dtype, void *workspace,
                                      size_t workspace_bytes, void *stream) {
    return tl_quantized_matmul_residual_norm_bits(scales, biases, b, out, p0, residual, norm_weight, normed_out, M, N, K, norm_eps, dtype, 4,
                                                  workspace, workspace_bytes, stream);
}

int tl_quantized_matmul_residual_norm_bits(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *residual,
                                           const void *norm_weight, void *normed_out, int M, int N, int K, float norm_eps, int dtype, int bits,
                                           void *workspace, size_t workspace_bytes, void *stream) {
    if (!norm_weight || !normed_out) return fail(TL_EINVAL, "quantized_matmul_residual_norm: null pointer");
    if (dtype != TL_F16 && dtype != TL_BF16) return fail(TL_EDTYPE, "quantized_matmul: scales must be float16 or bfloat16");
    TL_CHECK_BITS("quantized_matmul_residual_norm");
    if (M < 0 || N <= 0 || K < 0 || N % 128 != 0) return fail(TL_EINVAL, "quantized_matmul_residual_norm: bad shape");
    if (M == 0 || K == 0) return TL_OK;
    if (!scales || !biases || !b || !out || !p0 || !residual) return fail(TL_EINVAL, "quantized_matmul_residual_norm: null pointer");
    bool norm_done = false;
    int rc;
    if (w4a16_path(M, N, K, dtype, true, true, TL_PRO_NONE, N) == W4Path::SKINNY)
        rc = launch_w4a16_skinny(scales, biases, p0, b, out, residual, M, N, K, TL_EPI_RESIDUAL, dtype, workspace, workspace_bytes, as_stream(stream),
                                 norm_weight, norm_eps, normed_out, &norm_done, nullptr, bits);
    else
        rc = launch_w4a16_fused(scales, biases, b, out, p0, nullptr, residual, M, N, K, N, TL_PRO_NONE, TL_EPI_RESIDUAL, 0.f, dtype, as_stream(stream),
                                bits);
    if (rc != TL_OK || norm_done) return rc;
    return launch_rms_norm(out, norm_weight, normed_out, M, K, norm_eps, dtype, as_stream(stream));
}

int tl_qkv_project_rope_append(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch, const void *q_norm_weight,
                               const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table, const int32_t *context_lens, void *q_out,
                               void *key_pages, void *value_pages, int rows, int N, int num_heads, int num_kv_heads, int head_dim, float base, float eps,
                               int num_pages, int page_size, int max_pages, int chunk, int dtype, void *workspace, size_t workspace_bytes, void *stream) {
    return tl_qkv_project_rope_append_table_bits(scales, biases, b, p0, qkv_scratch, q_norm_weight, k_norm_weight, offsets, block_table, context_lens,
                                                 q_out, key_pages, value_pages, rows, N, num_heads, num_kv_heads, head_dim, base, eps, num_pages,
                                                 page_size, max_pages, chunk, dtype, 4, workspace, workspace_bytes, stream, nullptr);
}

int tl_qkv_project_rope_append_bits(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch,
                                    const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table,
                                    const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int rows, int N, int num_heads,
                                    int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size, int max_pages, int chunk,
                                    int dtype, int bits, void *workspace, size_t workspace_bytes, void *stream) {
    return tl_qkv_project_rope_append_table_bits(scales, biases, b, p0, qkv_scratch, q_norm_weight, k_norm_weight, offsets, block_table, context_lens,
                                                 q_out, key_pages, value_pages, rows, N, num_heads, num_kv_heads, head_dim, base, eps, num_pages,
                                                 page_size, max_pages, chunk, dtype, bits, workspace, workspace_bytes, stream, nullptr);
}

int tl_qkv_project_rope_append_table(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch,
                                     const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table,
                                     const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int rows, int N, int num_heads,
                                     int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size, int max_pages, int chunk,
                                     int dtype, void *workspace, size_t workspace_bytes, void *stream, const double *inv_freq) {
    return tl_qkv_project_rope_append_table_bits(scales, biases, b, p0, qkv_scratch, q_norm_weight, k_norm_weight, offsets, block_table, context_lens,
                                                 q_out, key_pages, value_pages, rows, N, num_heads, num_kv_heads, head_dim, base, eps, num_pages,
                                                 page_size, max_pages, chunk, dtype, 4, workspace, workspace_bytes, stream, inv_freq);
}

int tl_qkv_project_rope_append_table_bits(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch,
                                          const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table,
                                          const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int rows, int N, int num_heads,
                                          int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size, int max_pages,
                                          int chunk, int dtype, int bits, void *workspace, size_t workspace_bytes, void *stream,
                                          const double *inv_freq) {
    if (dtype != TL_BF16) return fail(TL_EDTYPE, "qkv_project_rope_append: bfloat16 required");
    TL_CHECK_BITS("qkv_project_rope_append");
    if (rows < 0 || N <= 0 || N % 128 != 0 || num_heads <= 0 || num_kv_heads <= 0 || head_dim <= 0 || head_dim % 2 != 0 || head_dim > 512 || num_pages <= 0 ||
        page_size <= 0 || max_pages <= 0)
        return fail(TL_EINVAL, "qkv_project_rope_append: bad shape");
    if (rows == 0) return TL_OK;
    if (!scales || !biases || !b || !p0 || !qkv_scratch || !q_norm_weight || !k_norm_weight || !offsets || !block_table || !context_lens || !q_out ||
        !key_pages || !value_pages)
        return fail(TL_EINVAL, "qkv_project_rope_append: null pointer");
    const int K = (num_heads + 2 * num_kv_heads) * head_dim;
    cudaStream_t st = as_stream(stream);
    int planes = 1;
    int rc;
    if (w4a16_path(rows, N, K, dtype, true, true, TL_PRO_NONE, N) == W4Path::SKINNY && qkv_planes_rope_supported(num_heads, num_kv_heads, head_dim, dtype))
        rc = launch_w4a16_skinny(scales, biases, p0, b, qkv_scratch, nullptr, rows, N, K, TL_EPI_NONE, dtype, workspace, workspace_bytes, st, nullptr, 0.f,
                                 nullptr, nullptr, &planes, bits);
    else
        rc = tl_quantized_matmul_fused_bits(scales, biases, b, qkv_scratch, p0, nullptr, nullptr, rows, N, K, N, TL_PRO_NONE, TL_EPI_NONE, 0.f, dtype,
                                            bits, workspace, workspace_bytes, stream);
    if (rc != TL_OK) return rc;
    if (planes > 1)  // the split-reduction planes go straight into the norm / RoPE / append kernel: q|k|v is never written
        return launch_qkv_planes_rope_append(static_cast<const float *>(workspace), planes, q_norm_weight, k_norm_weight, offsets, block_table,
                                             context_lens, q_out, key_pages, value_pages, rows, num_heads, num_kv_heads, base, inv_freq, eps,
                                             num_pages, page_size, max_pages, st, chunk != 0);
    return launch_decode_qk_norm_rope_append(qkv_scratch, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, q_out, key_pages,
                                             value_pages, rows, num_heads, num_kv_heads, head_dim, base, inv_freq, eps, num_pages, page_size, max_pages,
                                             dtype, st, chunk != 0);
}

int tl_qk_norm_rope_route(int num_heads, int num_kv_heads, int head_dim, int dtype) {
    if (dtype != TL_F32 && dtype != TL_BF16) return fail(TL_EDTYPE, "decode_qk_norm_rope_append: bfloat16 or float32 required");
    if (num_heads <= 0 || num_kv_heads <= 0 || head_dim <= 0 || head_dim % 2 != 0 || head_dim > 512)
        return fail(TL_EINVAL, "decode_qk_norm_rope_append: bad shape");
    return qkv_planes_rope_supported(num_heads, num_kv_heads, head_dim, dtype) ? TL_QKN_ROW : TL_QKN_HEAD;
}

int tl_decode_qk_norm_rope_append(const void *qkv, const void *q_norm_weight, const void *k_norm_weight,
                                  const int32_t *offsets, const int32_t *block_table, const int32_t *context_lens,
                                  void *q_out, void *key_pages, void *value_pages, int batch, int num_heads,
                                  int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size,
                                  int max_pages, int dtype, void *stream) {
    return tl_decode_qk_norm_rope_append_table(qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, q_out, key_pages, value_pages,
                                               batch, num_heads, num_kv_heads, head_dim, base, eps, num_pages, page_size, max_pages, dtype, stream,
                                               nullptr);
}

int tl_decode_qk_norm_rope_append_table(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                        const int32_t *block_table, const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages,
                                        int batch, int num_heads, int num_kv_heads, int head_dim, float base, float eps, int num_pages,
                                        int page_size, int max_pages, int dtype, void *stream, const double *inv_freq) {
    if (dtype != TL_F32 && dtype != TL_BF16) return fail(TL_EDTYPE, "decode_qk_norm_rope_append: bfloat16 or float32 required");
    if (batch < 0 || num_heads <= 0 || num_kv_heads <= 0 || head_dim <= 0 || head_dim % 2 != 0 || head_dim > 512 ||
        num_pages <= 0 || page_size <= 0 || max_pages <= 0)
        return fail(TL_EINVAL, "decode_qk_norm_rope_append: bad shape");
    if (batch == 0) return TL_OK;
    if (!qkv || !q_norm_weight || !k_norm_weight || !offsets || !block_table || !context_lens || !q_out || !key_pages || !value_pages)
        return fail(TL_EINVAL, "decode_qk_norm_rope_append: null pointer");
    return launch_decode_qk_norm_rope_append(qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, q_out,
                                             key_pages, value_pages, batch, num_heads, num_kv_heads, head_dim, base, inv_freq, eps,
                                             num_pages, page_size, max_pages, dtype, as_stream(stream));
}

int tl_chunk_qk_norm_rope_append(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                 const int32_t *block_table_row, const int32_t *context_lens, void *q_out, void *key_pages,
                                 void *value_pages, int tokens, int num_heads, int num_kv_heads, int head_dim, float base, float eps,
                                 int num_pages, int page_size, int max_pages, int dtype, void *stream) {
    return tl_chunk_qk_norm_rope_append_table(qkv, q_norm_weight, k_norm_weight, offsets, block_table_row, context_lens, q_out, key_pages,
                                              value_pages, tokens, num_heads, num_kv_heads, head_dim, base, eps, num_pages, page_size, max_pages,
                                              dtype, stream, nullptr);
}

int tl_chunk_qk_norm_rope_append_table(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                       const int32_t *block_table_row, const int32_t *context_lens, void *q_out, void *key_pages,
                                       void *value_pages, int tokens, int num_heads, int num_kv_heads, int head_dim, float base, float eps,
                                       int num_pages, int page_size, int max_pages, int dtype, void *stream, const double *inv_freq) {
    if (dtype != TL_F32 && dtype != TL_BF16) return fail(TL_EDTYPE, "chunk_qk_norm_rope_append: bfloat16 or float32 required");
    if (tokens < 0 || num_heads <= 0 || num_kv_heads <= 0 || head_dim <= 0 || head_dim % 2 != 0 || head_dim > 512 || num_pages <= 0 ||
        page_size <= 0 || max_pages <= 0)
        return fail(TL_EINVAL, "chunk_qk_norm_rope_append: bad shape");
    if (tokens == 0) return TL_OK;
    if (!qkv || !q_norm_weight || !k_norm_weight || !offsets || !block_table_row || !context_lens || !q_out || !key_pages || !value_pages)
        return fail(TL_EINVAL, "chunk_qk_norm_rope_append: null pointer");
    return launch_decode_qk_norm_rope_append(qkv, q_norm_weight, k_norm_weight, offsets, block_table_row, context_lens, q_out, key_pages,
                                             value_pages, tokens, num_heads, num_kv_heads, head_dim, base, inv_freq, eps, num_pages,
                                             page_size, max_pages, dtype, as_stream(stream), true);
}

size_t tl_decode_attention_fused_workspace(int batch, int num_heads, int num_kv_heads) {
    if (batch < 1 || num_heads < 1 || num_kv_heads < 1) return 0;
    return decode_attention_fused_workspace(batch, 1, num_heads, num_kv_heads);
}

int tl_decode_attention_fused(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                              const int32_t *block_table, const int32_t *context_lens, const double *rope_inv_freq,
                              void *key_pages, void *value_pages, void *out, float *workspace, int batch, int num_heads,
                              int num_kv_heads, int head_dim, float eps, float scale, int num_pages, int page_size,
                              int max_pages, int max_context, int dtype, void *stream) {
    return tl_decode_attention_fused_rows(qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, rope_inv_freq,
                                          key_pages, value_pages, out, workspace, batch, 1, num_heads, num_kv_heads, head_dim, eps,
                                          scale, num_pages, page_size, max_pages, max_context, dtype, stream);
}

size_t tl_decode_attention_fused_rows_workspace(int batch, int rows_per_request, int num_heads, int num_kv_heads) {
    if (batch < 1 || rows_per_request < 1 || rows_per_request > 8 || num_heads < 1 || num_kv_heads < 1) return 0;
    return decode_attention_fused_workspace(batch, rows_per_request, num_heads, num_kv_heads);
}

int tl_decode_attention_fused_rows(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                   const int32_t *block_table, const int32_t *context_lens, const double *rope_inv_freq,
                                   void *key_pages, void *value_pages, void *out, float *workspace, int batch,
                                   int rows_per_request, int num_heads, int num_kv_heads, int head_dim, float eps, float scale,
                                   int num_pages, int page_size, int max_pages, int max_context, int dtype, void *stream) {
    if (batch == 0) return TL_OK;
    if (!qkv || !q_norm_weight || !k_norm_weight || !offsets || !block_table || !context_lens || !rope_inv_freq || !key_pages ||
        !value_pages || !out || !workspace)
        return fail(TL_EINVAL, "decode_attention_fused: null pointer");
    if (batch < 0 || page_size < 1 || max_pages < 1 || num_pages < 0) return fail(TL_EINVAL, "decode_attention_fused: bad sizes");
    return launch_decode_attention_fused(qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, rope_inv_freq,
                                         key_pages, value_pages, out, workspace, batch, rows_per_request, num_heads, num_kv_heads,
                                         head_dim, eps, scale, num_pages, page_size, max_pages, max_context, dtype, as_stream(stream));
}

#if TL_TRACE
extern "C" int tl_debug_trace(unsigned long long *device_events, unsigned int *device_count, unsigned int capacity) {
    trace_bind_matvec(device_events, device_count, capacity);
    trace_bind_attention(device_events, device_count, capacity);
    trace_bind_skinny(device_events, device_count, capacity);
    return TL_OK;
}
#endif

int tl_set_pdl(int enabled) {
    set_use_pdl(enabled != 0);
    return TL_OK;
}

int tl_decode_advance(int32_t *tokens, const int32_t *next_tokens, int32_t *offsets, int32_t *context_lens,
                      int32_t *out_log, int32_t *step_counter, int batch, int log_capacity, void *stream) {
    if (batch <= 0 || log_capacity < 0) return fail(TL_EINVAL, "decode_advance: bad shape");
    if (!tokens || !next_tokens || !offsets || !context_lens || !out_log || !step_counter)
        return fail(TL_EINVAL, "decode_advance: null pointer");
    return launch_decode_advance(tokens, next_tokens, offsets, context_lens, out_log, step_counter, batch, log_capacity,
                                 as_stream(stream));
}

// ------------------------------------------------------------- Qwen3-MoE --
static int moe_shape(const char *op, int T, int k, int E) {
    if (T < 0 || E <= 0 || k <= 0) return fail(TL_EINVAL, "%s: bad shape (T = %d, k = %d, E = %d)", op, T, k, E);
    if (E > TL_MOE_MAX_EXPERTS) return fail(TL_EINVAL, "%s: at most %d experts (got %d)", op, TL_MOE_MAX_EXPERTS, E);
    if (k > TL_MOE_MAX_TOPK || k > E) return fail(TL_EINVAL, "%s: top-k must be in [1, min(%d, experts)] (got k = %d, E = %d)", op, TL_MOE_MAX_TOPK, k, E);
    if (static_cast<long long>(T) * k > (1 << 30)) return fail(TL_EINVAL, "%s: too many rows", op);
    return TL_OK;
}

// Upper bound of the tiles of R rows over at most min(E, R) non-empty experts: sum ceil(c_e / nt) <= (R + (nt - 1) min(E, R)) / nt.
static int moe_max_tiles(int R, int E, int nt) { return static_cast<int>((static_cast<long long>(R) + static_cast<long long>(nt - 1) * (E < R ? E : R)) / nt); }

int tl_moe_topk(const void *logits, void *probs, int32_t *ids, void *scores, int T, int E, int k, int norm_topk_prob, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "moe_topk: expected float32, float16, or bfloat16");
    if (int e = moe_shape("moe_topk", T, k, E)) return e;
    if (T == 0) return TL_OK;
    if (!logits || !probs || !ids || !scores) return fail(TL_EINVAL, "moe_topk: null pointer");
    return launch_moe_topk(logits, probs, ids, scores, T, E, k, norm_topk_prob != 0, dtype, as_stream(stream));
}

int tl_moe_tile_table_size(int R, int E, int nt) {
    if (R < 0 || E <= 0 || E > TL_MOE_MAX_EXPERTS || nt < 0) return fail(TL_EINVAL, "moe_group: bad shape");
    return nt > 0 ? 1 + 2 * moe_max_tiles(R, E, nt) : 0;
}

int tl_moe_group(const int32_t *ids, int R, int E, int nt, int32_t *offsets, int32_t *perm, int32_t *tiles, void *stream) {
    if (R < 0 || E <= 0 || nt < 0) return fail(TL_EINVAL, "moe_group: bad shape (R = %d, E = %d, nt = %d)", R, E, nt);
    if (E > TL_MOE_MAX_EXPERTS) return fail(TL_EINVAL, "moe_group: at most %d experts (got %d)", TL_MOE_MAX_EXPERTS, E);
    if (!offsets || (R > 0 && (!ids || !perm)) || (nt > 0 && !tiles)) return fail(TL_EINVAL, "moe_group: null pointer");
    return launch_moe_group(ids, R, E, nt, offsets, perm, tiles, as_stream(stream));
}

int tl_moe_gather(const void *x, const int32_t *perm, const void *norm_weight, float eps, void *xs, int R, int rows_per_source, int H, int dtype,
                  void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "moe_gather: expected float32, float16, or bfloat16");
    if (R < 0 || rows_per_source <= 0 || H <= 0) return fail(TL_EINVAL, "moe_gather: bad shape");
    if (R == 0) return TL_OK;
    if (!x || !perm || !xs) return fail(TL_EINVAL, "moe_gather: null pointer");
    return launch_moe_gather(x, perm, norm_weight, eps, xs, R, rows_per_source, H, dtype, as_stream(stream));
}

int tl_moe_grouped_matmul_route(int T, int k, int E, int N, int K, int epilogue, int dtype, const void *a, const void *b, int *nt, int *max_tiles) {
    if (nt) *nt = 0;
    if (max_tiles) *max_tiles = 0;
    if (int e = moe_shape("moe_grouped_matmul", T, k, E)) return e;
    if (N <= 0 || N % 128 != 0 || K <= 0) return fail(TL_EINVAL, "moe_grouped_matmul: N must be a positive multiple of 128 and K positive");
    if (epilogue != TL_EPI_NONE && epilogue != TL_EPI_SWIGLU_PAIRS) return fail(TL_EINVAL, "moe_grouped_matmul: epilogue must be none or swiglu pairs");
    if (epilogue == TL_EPI_SWIGLU_PAIRS && K % 16 != 0) return fail(TL_EINVAL, "moe_grouped_matmul: interleaved gate|up rows need K %% 16 == 0");
    if (dtype != TL_F16 && dtype != TL_BF16) return fail(TL_EDTYPE, "moe_grouped_matmul: scales must be float16 or bfloat16");
    const int R = T * k;
    if (K % 128 != 0 || !aligned16(a) || !aligned16(b)) return TL_MOE_CONTROL;
    const int per = (R + E - 1) / E;
    const int n = per <= 16 ? 16 : (per <= 32 ? 32 : (per <= 64 ? 64 : 128));
    const int tiles = moe_max_tiles(R, E, n);
    if (tiles > 65535) return TL_MOE_CONTROL;
    if (nt) *nt = n;
    if (max_tiles) *max_tiles = tiles;
    return TL_MOE_WGMMA;
}

int tl_moe_grouped_matmul(const void *scales, const void *biases, const void *b, const void *a, void *out, const int32_t *offsets,
                          const int32_t *tiles, const int32_t *out_index, int T, int k, int E, int N, int K, int epilogue, int dtype, void *stream) {
    int nt = 0, max_tiles = 0;
    const int route = tl_moe_grouped_matmul_route(T, k, E, N, K, epilogue, dtype, a, b, &nt, &max_tiles);
    if (route < 0) return route;
    const int R = T * k;
    if (R == 0) return TL_OK;
    if (!scales || !biases || !b || !a || !out || !offsets) return fail(TL_EINVAL, "moe_grouped_matmul: null pointer");
    if (route == TL_MOE_CONTROL)
        return launch_moe_grouped_vanilla(scales, biases, a, b, out, offsets, out_index, R, E, N, K, epilogue, dtype, as_stream(stream));
    if (!tiles) return fail(TL_EINVAL, "moe_grouped_matmul: the wgmma route needs the tile table");
    return launch_w4a16_grouped(scales, biases, a, b, out, offsets, tiles, out_index, R, E, N, K, epilogue, nt, max_tiles, dtype, as_stream(stream));
}

int tl_moe_combine(const void *y, const void *scores, const void *residual, const void *norm_weight, float eps, void *out, void *normed_out,
                   int T, int k, int H, int dtype, void *stream) {
    if (!float_dtype(dtype)) return fail(TL_EDTYPE, "moe_combine: expected float32, float16, or bfloat16");
    if (T < 0 || k <= 0 || k > TL_MOE_MAX_TOPK || H <= 0) return fail(TL_EINVAL, "moe_combine: bad shape (T = %d, k = %d, H = %d)", T, k, H);
    if ((norm_weight == nullptr) != (normed_out == nullptr)) return fail(TL_EINVAL, "moe_combine: norm weight and normed output go together");
    if (norm_weight != nullptr && H > 4096) return fail(TL_EINVAL, "moe_combine: the fused norm takes H <= 4096");
    if (T == 0) return TL_OK;
    if (!y || !scores || !out) return fail(TL_EINVAL, "moe_combine: null pointer");
    return launch_moe_combine(y, scores, residual, norm_weight, eps, out, normed_out, T, k, H, dtype, as_stream(stream));
}

int tl_moe_router(const void *x, const void *norm_weight, float eps, const void *w, const void *scales, const void *biases, void *logits, int T,
                  int E, int H, int dtype, void *stream) {
    if (dtype != TL_F16 && dtype != TL_BF16) return fail(TL_EINVAL, "moe_router: x must be float16 or bfloat16");
    if (T < 0 || T > TL_MOE_ROUTER_MAX_ROWS) return fail(TL_EINVAL, "moe_router: rows must be in [0, %d] (got %d)", TL_MOE_ROUTER_MAX_ROWS, T);
    if (E <= 0 || E > TL_MOE_MAX_EXPERTS) return fail(TL_EINVAL, "moe_router: 1 to %d experts (got %d)", TL_MOE_MAX_EXPERTS, E);
    if (H <= 0 || H % 64 != 0) return fail(TL_EINVAL, "moe_router: the hidden size must be a positive multiple of 64 (got %d)", H);
    if (T == 0) return TL_OK;
    if (!x || !w || !scales || !biases || !logits) return fail(TL_EINVAL, "moe_router: null pointer");
    if (!aligned16(x) || !aligned16(w) || (norm_weight && !aligned16(norm_weight)))
        return fail(TL_EINVAL, "moe_router: x, the codes and the norm weight must be 16-byte aligned");
    return launch_moe_router(x, norm_weight, eps, w, scales, biases, logits, T, E, H, dtype, as_stream(stream));
}

int tl_lora_apply_route(int M, int dtype, const tl_lora_site *site) { return lora_route(M, dtype, site); }

int tl_lora_apply(const void *x, void *const *y, const void *const *residual, const long long *ldy, const int32_t *adapter_ids,
                  const tl_lora_site *site, int M, int dtype, void *stream) {
    const int route = lora_route(M, dtype, site);
    if (route < 0) return route;
    if (M == 0) return TL_OK;
    if (!x || !y || !ldy || !adapter_ids || !site->a || !site->scales || !site->ranks || !site->seg_mask) return fail(TL_EINVAL, "lora_apply: null pointer");
    if (!aligned16(x) || !aligned16(site->a)) return fail(TL_EINVAL, "lora_apply: x and A must be 16-byte aligned");
    for (int s = 0; s < site->nseg; ++s)
        if (!site->b[s] || !aligned16(site->b[s])) return fail(TL_EINVAL, "lora_apply: B of segment %d must be a 16-byte aligned pointer", s);
    for (int s = 0; s < site->nseg; ++s)
        if (!y[s] || ldy[s] < site->K[s] || (residual && !residual[s])) return fail(TL_EINVAL, "lora_apply: bad output of segment %d", s);
    return launch_lora_apply(x, y, residual, ldy, adapter_ids, *site, M, route, as_stream(stream));
}

}  // extern "C"
