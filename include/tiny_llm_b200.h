/*
 * tiny_llm_b200.h - C ABI of the H100 (sm_90a) backend for tiny-llm's Qwen3
 * W4A16 inference hot path.
 *
 * This is the drop-in boundary: one launcher per native primitive of the
 * reference's extension (declared in
 * src/extensions_ref/src/tiny_llm_ext.h:10-141 and exported to
 * Python by src/extensions_ref/bindings.cpp:14-46).  Where the
 * reference builds a lazy `mx::array` whose `eval_gpu` encodes a Metal
 * dispatch, a launcher here enqueues sm_90a kernels on the caller's CUDA
 * stream.  Conventions:
 *
 *   - plain device pointers and sizes; no torch / MLX types;
 *   - the caller owns every buffer (outputs and workspaces included); a
 *     launcher never allocates, frees or synchronises, so it is legal inside
 *     CUDA-graph capture;
 *   - `stream` is a `cudaStream_t` passed as `void*` (NULL = legacy default);
 *   - return 0 on success, a negative TL_E* code otherwise; the message is
 *     available from tl_last_error() (thread-local); nothing throws across
 *     the boundary;
 *   - `dtype` is one of TL_F32 / TL_F16 / TL_BF16 and names the activation /
 *     storage type; all accumulation is fp32.
 *
 * Naming quirk kept from the reference (quantized_matmul.cpp:125-127):
 * in quantized_matmul `a` is [M, N] with N the REDUCTION length, `b` is
 * [K, N/8] packed words with K the number of OUTPUT features, out is [M, K].
 */
#ifndef TINY_LLM_B200_H
#define TINY_LLM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { TL_F32 = 0, TL_F16 = 1, TL_BF16 = 2 };

enum {
    TL_OK = 0,
    TL_EINVAL = -1,      /* bad argument (shape, alignment, unsupported combination) */
    TL_EDTYPE = -2,      /* dtype not supported by this primitive */
    TL_EWORKSPACE = -3,  /* workspace missing or too small */
    TL_ECUDA = -4,       /* CUDA runtime / driver error at launch */
    TL_ENODEVICE = -5    /* no sm_90 device */
};

/* Library identity / diagnostics. */
int tl_abi_version(void);
const char *tl_last_error(void);
/* Fills SM count and compute capability of the current device. */
int tl_device_info(int *sm_count, int *cc_major, int *cc_minor);
/* Number of kernels this library has launched since load (bench bookkeeping). */
long long tl_launch_count(void);

/* ---- W4A16 (4-bit, group 128) projections -------------------------------
 * Replaces quantized_matmul (tiny_llm_ext.h:12-21, quantized_matmul.cpp:14-80,
 * eval_gpu :111-240).  scales/biases [K, N/128] (f16|bf16), a [M, N],
 * b [K, N/8] u32, out [M, K].  Kernel selection:
 *   !use_simdgroup                  : scalar control kernel;
 *   M <= TL_MATVEC_REF_ROWS         : weight-streaming tensor-core matvec, weights kept fp32-exact (reference:
 *       M <= 8 matvec, quantize.py:162-163), up to TL_MATVEC_MAX_ROWS rows per pass;
 *   TL_MATVEC_REF_ROWS < M <= 128   : swap-AB wgmma GEMM with the reduction split over
 *       CTAs (reference: quantized_matmul_splitk, quantized_matmul.metal:251-293), weights rounded to
 *       the activation dtype before the MMA, fp32 partial planes added in split order;
 *   M > 128                         : the same wgmma kernel on 128-token tiles, weights rounded to
 *       the activation dtype before the MMA (reference: simdgroup tile).
 * The wgmma kernels need a and b 16-byte aligned; otherwise the call returns TL_EINVAL.
 * The split of the reduction is a scheduling decision of this backend (SURVEY 8a' item 12): it depends only on
 * (N, K), never on use_split_k, so a split request and a plain request run the very same kernel with
 * bit-identical results (tests_refsol/test_week_2_day_7.py:80-109).
 * workspace: tl_quantized_matmul_workspace() bytes (0 = none; fp32 partial planes of a split reduction,
 * no initialisation needed). */
#define TL_MATVEC_REF_ROWS 8
#define TL_MATVEC_MAX_ROWS 32
/* The kernel a W4A16 projection runs (nothing is launched or read; the pointers only count for their alignment):
 * TL_W4_VANILLA / TL_W4_STREAM / TL_W4_SKINNY / TL_W4_TILES as selected above, or a negative TL_E* code for arguments
 * the launch rejects (a or b not 16-byte aligned on the wgmma paths, misaligned operands or too wide a row on the
 * streaming kernel).  `fused` selects the rule of tl_quantized_matmul_fused / tl_quantized_matmul_residual_norm (which
 * keep M > 128 on the streaming kernel and take a prologue and a row stride lda >= N); the plain call needs
 * prologue TL_PRO_NONE and lda == N.  The facts of the chosen kernel are written, 0 where they do not apply:
 *   *splits, *gb_per_split : SKINNY / TILES, the reduction split and the 128-wide groups per split (TILES: 1 and N/128);
 *   *rows_per_pass, *units : STREAM, activation rows per pass (a power of two <= TL_MATVEC_MAX_ROWS: larger M runs in
 *                            several passes) and 128-column groups per weight unit (2 when N % 256 == 0, scales and
 *                            biases are 4-byte aligned and M <= 16; otherwise 1).
 * The split count depends on the SM count of the current device. */
enum { TL_W4_VANILLA = 0, TL_W4_STREAM = 1, TL_W4_SKINNY = 2, TL_W4_TILES = 3 };
int tl_quantized_matmul_route(int M, int N, int K, int lda, int prologue, int fused, int use_simdgroup, int dtype, const void *a, const void *b,
                              const void *scales, const void *biases, int *splits, int *gb_per_split, int *rows_per_pass, int *units);
size_t tl_quantized_matmul_workspace(int M, int N, int K, int dtype, int use_simdgroup, int use_split_k);
int tl_quantized_matmul(const void *scales, const void *biases, const void *a, const void *b, void *out, int M,
                        int N, int K, int dtype, int use_simdgroup, int use_split_k, void *workspace,
                        size_t workspace_bytes, void *stream);
/* W8A16: every entry that takes packed weights has a *_bits sibling whose `bits` (after dtype) is 4 or 8; the entry
 * without the suffix is its bits = 4 form.  8-bit weights are MLX affine at group 128: b [K, N/4] u32, code i of a word
 * = (w >> 8i) & 255, scales/biases [K, N/128], weight = code * scale + bias.  Kernel choice, row thresholds and
 * workspace sizes are those of 4 bits.  Any other `bits` is TL_EINVAL (the two workspace queries return 0 for it). */
int tl_quantized_matmul_route_bits(int M, int N, int K, int lda, int prologue, int fused, int use_simdgroup, int dtype, int bits, const void *a,
                                   const void *b, const void *scales, const void *biases, int *splits, int *gb_per_split, int *rows_per_pass,
                                   int *units);
size_t tl_quantized_matmul_workspace_bits(int M, int N, int K, int dtype, int bits, int use_simdgroup, int use_split_k);
int tl_quantized_matmul_bits(const void *scales, const void *biases, const void *a, const void *b, void *out, int M, int N, int K, int dtype,
                             int bits, int use_simdgroup, int use_split_k, void *workspace, size_t workspace_bytes, void *stream);

/* Replaces quantized_embedding (tiny_llm_ext.h:40-41, quantized_matmul.cpp:82-101,
 * :242-273).  indices int32/uint32 [tokens] (bit pattern), weight [vocab, dim/8] u32,
 * scales/biases [vocab, dim/128], out [tokens, dim]. */
int tl_quantized_embedding(const void *indices, const void *scales, const void *biases, const void *weight,
                           void *out, int tokens, int vocab, int dim, int dtype, void *stream);
/* weight [vocab, dim * bits / 32] u32; at 8 bits 8-byte aligned. */
int tl_quantized_embedding_bits(const void *indices, const void *scales, const void *biases, const void *weight, void *out, int tokens, int vocab,
                                int dim, int dtype, int bits, void *stream);

/* ---- fused model kernels (week2_kernels.cpp:36-84, :104-211) ------------- */
/* x [rows, dim], weight [dim], out [rows, dim]:  x * rsqrt(mean(x^2)+eps) * w */
int tl_rms_norm(const void *x, const void *weight, void *out, int rows, int dim, float eps, int dtype,
                void *stream);
/* x,out [B, L, H, D]; offsets int32 [B]; rotates the first `dims` of D. */
int tl_rope(const void *x, const int32_t *offsets, void *out, int B, int L, int H, int D, int dims, float base,
            int traditional, int dtype, void *stream);
/* RoPE frequency tables.  Every RoPE entry point below has a *_table form taking one more, trailing argument
 * `const double *inv_freq`: a DEVICE float64 [dims / 2] table of frequencies that replaces base^(-i / (dims / 2))
 * (base is then unused).  Null is the entry point without the suffix.  A scaled RoPE (YaRN, DESIGN.md "Long
 * context") passes its blended table; every site of one model must read the same table so that keys written at
 * prefill and queries rotated at decode use identical angles.  tl_rope_inv_freq writes the unscaled table,
 * out[i] = base^(-i / (head_dim / 2)) for i < head_dim / 2, with the kernels' own double-precision expression:
 * a site given that table returns the bits of its base path. */
int tl_rope_inv_freq(double *out, int head_dim, float base, void *stream);
int tl_rope_table(const void *x, const int32_t *offsets, void *out, int B, int L, int H, int D, int dims, float base,
                  int traditional, int dtype, void *stream, const double *inv_freq);
/* The kernels tl_rms_norm and tl_rope run (nothing is launched or read; pointers only count for their 16-byte
 * alignment), or a negative TL_E* code for arguments the launch rejects.
 *   tl_rms_norm_route : threads per row, 32 (one warp; dim <= 512) or 256 (one CTA); *vec = 1 when every access is a
 *                       16-byte vector (dim a multiple of 16 bytes, x, weight and out 16-byte aligned), else 0;
 *   tl_rope_route     : TL_ROPE_HEADS, one thread per (token, pair) walking the H heads (dims == D, H > 1, B * L >= 64),
 *                       else TL_ROPE_ELEMENT, one thread per (token, head, pair or copied tail element). */
enum { TL_ROPE_ELEMENT = 0, TL_ROPE_HEADS = 1 };
int tl_rms_norm_route(int dim, int dtype, const void *x, const void *weight, const void *out, int *vec);
int tl_rope_route(int B, int L, int H, int D, int dims, int dtype);
/* out = gate / (1 + exp(-gate)) * up, `size` elements. */
int tl_swiglu(const void *gate, const void *up, void *out, long long size, int dtype, void *stream);
/* Dense-KV GQA attention: q,out [q_rows, L, D] with q_rows = B*Hq; k,v [B*Hkv, S, D];
 * mask fp32 [q_rows, L, S] when has_mask (ignored otherwise).  D <= 256. */
int tl_decode_attention(const void *q, const void *k, const void *v, const float *mask, void *out, int q_rows,
                        int L, int S, int D, int num_heads, int num_kv_heads, float scale, int is_causal,
                        int has_mask, int dtype, void *stream);

/* ---- paged KV (paged_attention.cpp:14-31, :38-70, :77-122, :129-225) ------ */
/* In-place: pages[page_id, :, start:start+length, :] = values[0]; pages [P,H,page,D],
 * values [1,H,length,D]. */
int tl_paged_cache_update(void *pages, const void *values, int num_pages, int heads, int page_size, int head_dim,
                          int length, int page_id, int start, int dtype, void *stream);
/* q,out [B*Hq, L, D]; pages [P, Hkv, page, D]; block_table int32 [B, max_pages]
 * (-1 padded); context_lens int32 [B] (post-append).  D <= 128; the tensor-core
 * prefill branch (L > 8, bf16) requires D == 128.  Query row l of request b
 * sees the keys < min(clamp(ctx - L + l + 1, 0, ctx), max_pages * page_size)
 * when causal (< min(ctx, max_pages * page_size) otherwise), ctx =
 * context_lens[b]: a context longer than the block table keeps its causal
 * alignment and loses the keys past the table.  Keys in pages whose id is < 0
 * or >= num_pages are skipped.  Rows that see no key are written as zeros.
 * Workspace holds split-KV partials for the decode branch. */
size_t tl_paged_attention_workspace(int rows, int L, int D, int num_kv_heads, int num_heads, int dtype);
int tl_paged_attention(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                       const int32_t *context_lens, void *out, int rows, int L, int D, int num_pages,
                       int page_size, int max_pages, float scale, int is_causal, int num_kv_heads, int num_heads,
                       int dtype, void *workspace, size_t workspace_bytes, void *stream);
/* The kernel tl_paged_attention would run for these arguments (nothing is launched or read; the pointers only count
 * for their 16-byte alignment): one of TL_PAGED_*, or a negative TL_E* code for arguments tl_paged_attention rejects.
 *   TL_PAGED_ROWWISE : one CTA per query row; every dtype, head size and page size;
 *   TL_PAGED_GQA     : bf16, D == 128, 16-byte aligned q / K / V; CUDA cores, the query heads of a KV head together;
 *                      decode steps (L <= 8) split the key range over CTAs (plus a merge launch);
 *   TL_PAGED_FLASH   : bf16, D == 128 prefill (L > 8) on mma.sync, for page sizes or head ratios the wgmma kernel
 *                      does not take;
 *   TL_PAGED_WGMMA   : bf16, D == 128, pages a multiple of 64 slots, Hq / Hkv divides 128, out 16-byte aligned; every
 *                      prefill, and decode steps whose G x L query rows fill one 128-row tile and whose block table
 *                      spans at least 1024 keys (split like the GQA kernel). */
enum { TL_PAGED_ROWWISE = 0, TL_PAGED_GQA = 1, TL_PAGED_FLASH = 2, TL_PAGED_WGMMA = 3 };
int tl_paged_attention_route(const void *q, const void *key_pages, const void *value_pages, const void *out, int rows, int L, int D,
                             int num_pages, int page_size, int max_pages, int num_kv_heads, int num_heads, int dtype);
/* The prefill form with the output written token-major: out [B, L, Hq * D] (the layout the o-projection takes; saves
 * the transpose copy of a chunked-prefill step).  bf16, D == 128, pages a multiple of 64 slots (the wgmma kernel);
 * TL_EINVAL otherwise - callers then use tl_paged_attention and transpose. */
int tl_paged_attention_token_major(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                   const int32_t *context_lens, void *out, int rows, int L, int num_pages, int page_size, int max_pages,
                                   float scale, int is_causal, int num_kv_heads, int num_heads, void *stream);
/* The same with a split of the key range for a prefill chunk with a long prefix: when the block table spans more than
 * 8,192 keys (max_pages * page_size) the key range of every (request, KV head) is cut into up to 32 pieces (the count
 * from a wave cost model, the tiles dealt out from each request's real context) and a merge launch writes the
 * token-major output.  workspace: tl_paged_attention_token_major_workspace() bytes (0 at <= 8,192 keys, where the call
 * is tl_paged_attention_token_major); null never splits. */
size_t tl_paged_attention_token_major_workspace(int rows, int L, int page_size, int max_pages);
int tl_paged_attention_token_major_split(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                         const int32_t *context_lens, void *out, int rows, int L, int num_pages, int page_size, int max_pages,
                                         float scale, int is_causal, int num_kv_heads, int num_heads, void *workspace, size_t workspace_bytes,
                                         void *stream);
/* Shared-prefix decode attention: the result of tl_paged_attention at L = 1, causal, for every slot on its own block
 * table, computed with each group's shared pages streamed once for all its query rows.  q, out [batch * Hq, 1, 128]
 * bf16; pages, block_table [batch, max_pages] and context_lens [batch] as tl_paged_attention.  groups: num_groups
 * int32 triples (first_slot, count, shared_pages) on the device; slots first_slot .. first_slot + count - 1 hold the
 * same page ids in their first shared_pages table entries (not checked) and each row's context covers them.  Entries
 * with count 0 are unused; slots in no group, and groups with shared_pages 0, attend all their keys in the suffix pass.
 * groups_host: the same triples in host memory, checked here: groups in [0, batch), not overlapping, count * Hq / Hkv
 * <= 128, 0 <= shared_pages <= max_pages.  bf16, D = 128, page_size a multiple of 64.  The launch grid and split
 * counts depend only on (batch, heads, page_size, max_pages): one captured graph serves every grouping.  Three
 * launches (prefix pass, suffix pass, merge); workspace of tl_shared_prefix_attention_workspace bytes. */
size_t tl_shared_prefix_attention_workspace(int batch, int num_heads, int num_kv_heads, int page_size, int max_pages);
int tl_shared_prefix_attention(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                               const int32_t *context_lens, const int32_t *groups, const int32_t *groups_host, int num_groups,
                               void *out, int batch, int D, int num_pages, int page_size, int max_pages, float scale,
                               int num_kv_heads, int num_heads, int dtype, void *workspace, size_t workspace_bytes, void *stream);
/* Segment-causal attention for packed prefill (embedding passes): one request whose L rows are several prompts laid
 * end to end, each row's K/V already appended at slot = row through the one block-table row block_table [max_pages].
 * Row l sees exactly the keys segment_start[l] <= key <= l (segment_start: int32 [L] on the device, the first row of
 * l's prompt); a row with segment_start[l] > l (padding) sees nothing and its output is 0.  A CTA skips the key tiles
 * before the smallest segment_start of its rows.  q [Hq, L, 128] (the chunk form's layout), out [L, Hq * 128]
 * token-major; bf16 or fp16 q / pages / out, 16-byte aligned; page_size a multiple of 64; Hq / Hkv divides 128;
 * L <= max_pages * page_size.  One launch, no workspace, no synchronisation (capturable). */
int tl_paged_attention_segments(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                const int32_t *segment_start, void *out, int L, int D, int num_pages, int page_size, int max_pages, float scale,
                                int num_kv_heads, int num_heads, int dtype, void *stream);
/* Pooled embeddings of packed hidden states (DESIGN.md section 17).  hidden [rows, hidden_size] and norm_weight
 * [hidden_size] bf16 or fp16; segment_start int32 [num_segments + 1] on the device, segment s = rows
 * segment_start[s] .. segment_start[s + 1] - 1.  Each pooled row is RMS-normalised exactly as tl_rms_norm does it
 * (same bits); TL_EMBED_LAST takes the segment's last row, TL_EMBED_MEAN the fp32 mean of its normalised,
 * dtype-rounded rows summed in row order.  The result is truncated to the first `dimensions` features and, with
 * normalize, divided by its fp32 L2 norm (a zero vector stays zero).  out: fp32 [num_segments, dimensions].  An
 * empty segment gives zeros.  hidden_size <= TL_EMBED_MAX_HIDDEN. */
enum { TL_EMBED_LAST = 0, TL_EMBED_MEAN = 1, TL_EMBED_MAX_HIDDEN = 12288 };
int tl_embed_pool(const void *hidden, const void *norm_weight, float eps, const int32_t *segment_start, int num_segments, int rows, int hidden_size,
                  int dimensions, int pooling, int normalize, float *out, int dtype, void *stream);
/* Prefixed-segment attention for packed reranking passes (DESIGN.md section 19): tl_paged_attention_segments with one
 * more visible key range per row.  Row l sees exactly the keys in [prefix_start[l], prefix_end[l]) and in
 * [segment_start[l], l].  prefix_start / prefix_end: int32 [L] on the device; precondition prefix_end[l] <=
 * segment_start[l] (a larger prefix_end is cut there); prefix_start[l] == prefix_end[l] is an empty prefix.  A padding
 * row has an empty prefix and segment_start[l] > l (L): its output is 0.  A CTA visits the key tiles of the hull of
 * its rows' prefix ranges, then those from its rows' smallest segment start to its last row, and skips the tiles
 * between; skipped and masked keys change no bit of the result.  Masked K/V slots are multiplied by zero
 * probabilities, so every slot the block table reaches must hold finite values.  Other arguments, layouts and checks
 * as tl_paged_attention_segments. */
int tl_paged_attention_prefixed_segments(const void *q, const void *key_pages, const void *value_pages, const int32_t *block_table,
                                         const int32_t *segment_start, const int32_t *prefix_start, const int32_t *prefix_end, void *out, int L,
                                         int D, int num_pages, int page_size, int max_pages, float scale, int num_kv_heads, int num_heads,
                                         int dtype, void *stream);
/* Selected-token logits of packed hidden states (DESIGN.md section 19), in place of the LM head.  hidden [rows,
 * hidden_size] and norm_weight [hidden_size] bf16 or fp16; row_index int32 [n] and token_ids int32 [m] on the device,
 * 1 <= m <= TL_SELECT_MAX_IDS.  The LM head (or the tied embedding) is MLX affine at group 128: weight [vocab,
 * hidden_size * bits / 32] u32, scales / biases [vocab, hidden_size / 128] of the hidden dtype, bits 4 or 8.  Row
 * row_index[i] is RMS-normalised exactly as tl_rms_norm does it; the logit of token_ids[j] is the fp32 sum, in a fixed
 * order, of the normalised row times the weights T(code * scale + bias), rounded to the hidden dtype T.  logits [n, m]
 * fp32 (T-rounded values) and logprobs [n, m] fp32, the log-softmax over the m logits of a row.  Valid ranges:
 * 0 <= row_index[i] < rows, 0 <= token_ids[j] < vocab; an index outside gives NaN in what it touches and reads
 * nothing.  hidden_size a multiple of 128, at most TL_EMBED_MAX_HIDDEN.  One launch, no workspace. */
enum { TL_SELECT_MAX_IDS = 32 };
int tl_select_logits(const void *hidden, const void *norm_weight, float eps, const int32_t *row_index, int n, int rows, int hidden_size,
                     const void *weight, const void *scales, const void *biases, int vocab, int bits, const int32_t *token_ids, int m,
                     float *logits, float *logprobs, int dtype, void *stream);

/* ---- CUDA extension behind the same per-op semantics ---------------------
 * Device-driven K/V append for a decode batch (the batched form of
 * paged_kv_cache.py:196-234 called once per request, kv_cache.py:191-199):
 * row b writes keys[b]/values[b] ([B, Hkv, 1, D]) to the slot of token
 * context_lens[b]-1, resolved through block_table; rows with context 0 are
 * skipped.  Page ids and slots come from device memory, so the call is
 * CUDA-graph replayable. */
int tl_paged_cache_append_decode(void *key_pages, void *value_pages, const void *keys, const void *values,
                                 const int32_t *block_table, const int32_t *context_lens, int batch,
                                 int num_pages, int heads, int page_size, int head_dim, int max_pages, int dtype,
                                 void *stream);
/* out = a + b (residual adds of qwen3_week3.py:204-206), `size` elements. */
int tl_add(const void *a, const void *b, void *out, long long size, int dtype, void *stream);
/* Greedy sampler of batch.py:8-13: out_tokens[r] = argmax(logits[r, :]) (the
 * log-softmax shift is argmax-invariant).  logits [rows, vocab], out int32 [rows]. */
int tl_argmax(const void *logits, int32_t *out_tokens, int rows, int vocab, int dtype, void *workspace,
              size_t workspace_bytes, void *stream);
size_t tl_argmax_workspace(int rows, int vocab);
/* Seeded sampling of one token per row of logits [rows, vocab] (rows <= 65535, vocab <= 409,600), parameters per row
 * as device arrays: temperature f32, top_k i32 (on when 0 < k < vocab), top_p f32 (on when 0 < p < 1), seed i64 and
 * positions i32 (the index of the token being drawn).  temperature == 0, or a row whose maximum is not finite, returns
 * tl_argmax's token.  Otherwise the token is argmax over the keep set {x >= max(x_(k), v*)} of
 * x / temperature - log(-log u), u from Philox4x32-10 at counter (i >> 2, position, 0, 0) and key (seed low word,
 * seed high word), word i % 4 (DESIGN.md section 8): a pure function of (row, parameters, seed, position).
 * No workspace; deterministic. */
int tl_sample(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
              const int32_t *positions, int32_t *out_tokens, int rows, int vocab, int dtype, void *stream);
/* tl_sample with token-history penalties and min-p (DESIGN.md section 8b).  Extra per-row device arrays: repetition,
 * presence, frequency and min_p (f32), and state (int32 [rows, vocab], read and written) with, for token i of row r,
 * bit 30 set when i occurs in the request's prompt and bits 0-29 the number of times i has been drawn for the request
 * so far (the first token, drawn from the last prefill chunk, included).  Repetition applies to prompt and generated
 * tokens, presence and frequency to generated tokens only (vLLM's semantics).
 * With s = state[r, i], c = s & (2^30 - 1), seen = (s & 2^30) || c > 0, each staged fp32 logit x becomes, one IEEE
 * round-to-nearest operation per step and in this order:
 *   x1 = seen && rep != 1 ? (x > 0 ? x / rep : x * rep) : x;
 *   x2 = c > 0 ? x1 - fl(freq * (float)c) : x1;
 *   x3 = c > 0 ? x2 - presence : x2;
 * (NaN stays NaN).  Everything tl_sample does then runs on the penalised row x3: the first-maximum argmax (so
 * temperature 0 is greedy on the penalised row), the non-finite-maximum rule, top-k, top-p and the Gumbel draw.
 * min_p (on for min_p > 0; values above 1 act as 1) adds the bound x >= thr, thr = fl(m + fl(T * L)), m the penalised
 * maximum and L = log(min_p) in double rounded once to f32: the keep set is {x >= max(x_(k), v*, thr)}, all three
 * bounds taken over the whole penalised row.  A row with rep == 1, presence == 0 and frequency == 0 does not read its
 * state, and its draw is tl_sample's.
 * After the draw, state[r, token] += 1 for every row with positions[r] > 0 (idle decode slots and capture warm-ups
 * run at position 0 and change nothing).  A draw is a pure function of (logits row, state row, parameters, seed,
 * position). */
int tl_sample_penalized(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                        const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                        const float *min_p, int32_t *state, int32_t *out_tokens, int rows, int vocab, int dtype, void *stream);
/* tl_sample_penalized with XTC (DESIGN.md section 24): xtc_threshold and xtc_probability, per-row f32 device arrays
 * (both NULL: tl_sample_penalized, bit for bit).  For a row with temperature > 0, a finite maximum and probability q > 0, let K be
 * the keep set above, e_i = fl(expf(fl(fl(x_i - m) / T)) * 2^40) rounded to an integer for i in K, S their (exact,
 * integer) sum, and A = {i in K : (double)e_i >= (double)theta * (double)S}.  u = (2 (w >> 9) + 1) 2^-24 with w word
 * 0 of Philox4x32-10 at counter (0, position, 3, 0) under the seed key (counter word 2 is the stream: 0 the draw,
 * 1 acceptance, 2 residual, 3 XTC).  When u < q and |A| >= 2, every i in A with x_i > min over A of x leaves K
 * (ties at that minimum stay), and the draw runs on the smaller set.  |e_i / S - p_i| stays below 2^-20 for the
 * exact softmax p over K (expf's 2 ulp, the 2^-40 rounding of each term), so A agrees with {p_i >= theta} for every
 * i whose p_i lies farther than 2^-20 from theta.  Temperature 0 is unaffected. */
int tl_sample_penalized_xtc(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                            const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                            const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability,
                            int32_t *out_tokens, int rows, int vocab, int dtype, void *stream);
/* tl_sample_penalized_xtc with the truncation samplers (DESIGN.md section 25): typical_p, top_n_sigma, mirostat_tau and
 * mirostat_eta, per-row f32 device arrays, and mirostat_mu, a per-row f32 device array read and written (all NULL:
 * tl_sample_penalized_xtc, bit for bit; any of them NULL when no row of the launch uses it).  For a row with temperature
 * > 0 and a finite maximum m (z_i = fl(x_i - m), e_i the 2^-40 fixed-point masses as tl_sample_penalized_xtc defines
 * them):
 *   top-n-sigma  n = top_n_sigma > 0: tau also bounds x >= m - n sigma, sigma the population standard deviation of the
 *                row's finite entries (sums in double, the bound rounded up to fp32);
 *   typical      0 < p = typical_p < 1: over the keep set K and its T = 1 masses, d_i = |z_bar - z_i| with
 *                z_bar = sum e_i z_i / sum e_i; K keeps the entries whose d (rounded to fp32) is at most the smallest
 *                d* with mass(d <= d*) >= p S_K, the others become NaN; XTC then runs on what is left;
 *   Mirostat     mirostat_tau > 0 (mirostat_eta and mirostat_mu then required): top-k, top-p, min-p, top-n-sigma,
 *                typical and XTC are ignored; with e_i at the row's temperature over the non-NaN entries and S their
 *                sum, the row keeps {(double)e_i >= min(S 2^-mu, 2^40)} (the maximum always), draws among them, and
 *                for rows with position > 0 writes mu' = fl32(mu - eta (log2 S_K - log2 e_token - tau)) in double.
 * Temperature 0 and a non-finite maximum are unaffected, and leave mu alone. */
int tl_sample_penalized_trunc(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                              const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                              const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability,
                              const float *typical_p, const float *top_n_sigma, const float *mirostat_tau, const float *mirostat_eta,
                              float *mirostat_mu, int32_t *out_tokens, int rows, int vocab, int dtype, void *stream);
/* Speculative sampling (DESIGN.md section 8d): the rejection rule over one verify pass of T = k + 1 rows
 * (1 <= T <= 65535, vocab <= TL_SPECULATIVE_SAMPLE_MAX_VOCAB).  target [T, vocab] are the target's logits rows,
 * draft [k, vocab] the draft's rows each proposal proposals[j] (int32, device) was drawn from, the parameters per row
 * as tl_sample takes them (all T rows normally carry one request's values) and positions[j] = n_j, the index of the
 * token row j predicts.  Every device input is read after the programmatic-dependent-launch wait.
 * Row distributions: temperature 0, or a row whose maximum is not finite, is the point mass at the row's tl_argmax
 * token; otherwise p_i = exp((x_i - m) / T) / sum over K of the same, K = tl_sample's keep set of x (top-k, top-p),
 * and 0 outside K; q likewise from the draft row.  q is the distribution tl_sample drew d_j from.
 * Row j < k accepts iff q_d > 0 and u q_d <= p_d, u = (2 (w >> 9) + 1) 2^-24, w word 0 of Philox4x32-10 at counter
 * (0, n_j, 1, 0) under the seed key; then out[j] = d_j.  Otherwise out[j] = argmax over {i : p_i > q_i} of
 * log(p_i - q_i) + g_i, g_i = -log(-log u_i) with u_i from word i % 4 at counter (i >> 2, n_j, 2, 0).  If rounding
 * left that set empty the row returns the tl_argmax token of x (the kernel compares exact integer masses, so a
 * rejection always leaves it non-empty).  Row k (the bonus row) is tl_sample's draw on target row k at n_k, bit for
 * bit.  Counter word 2 is the stream: 0 the ordinary draw (the draft's, the bonus row's), 1 the acceptance uniform,
 * 2 the residual noise.  The emitted token at n_j is distributed as the target's tl_sample draw; with temperature 0
 * it is greedy verification; a rejected proposal with q_d > 0 is never the residual.  The kernel sums masses as
 * 2^-40 fixed-point integers and compares p and q exactly on them: deterministic whatever T or the row index. */
#define TL_SPECULATIVE_SAMPLE_MAX_VOCAB 204800
int tl_speculative_sample(const void *target, const void *draft, const int32_t *proposals, const float *temperature,
                          const int32_t *top_k, const float *top_p, const int64_t *seed, const int32_t *positions,
                          int32_t *out_tokens, int rows, int vocab, int dtype, void *stream);
/* Copy `bytes` from src to dst + out_index[0] * bytes when 0 <= out_index[0] < capacity (device index; nothing
 * otherwise): a captured decode step logs its logits rows at the step counter, as tl_logprobs logs. */
int tl_log_rows(const void *src, void *dst, const int32_t *out_index, int capacity, long long bytes, void *stream);
/* Regex-constrained sampling (DESIGN.md section 8c).  One descriptor per row, in device memory (40 bytes):
 *   mask           uint32 [num_states + 1, ceil(vocab / 32)]: bit t of row s set iff token t is allowed in state s;
 *                  NULL: the row is unconstrained and draws exactly as tl_sample / tl_sample_penalized;
 *   dfa            int32 [num_states, 256], the byte DFA (-1: dead);
 *   token_offsets  int32 [vocab + 1] and token_bytes: each token's bytes (EOS and never-emitted ids: none);
 *   num_states     S, the DFA's state count; state S is the terminal state after EOS;
 *   state          the row's current state, read and (rank 0, after the draw) written by tl_sample_constrained. */
typedef struct tl_constraint_row {
    const uint32_t *mask;
    const int32_t *dfa;
    const int32_t *token_offsets;
    const uint8_t *token_bytes;
    int32_t num_states;
    int32_t state;
} tl_constraint_row;
/* The token masks of a byte DFA over a vocabulary, in one launch.  dfa int32 [num_states, 256] (-1: dead; every state
 * live), accept uint8 [num_states], token_offsets int32 [vocab + 1] with token_bytes, eos_ids int32 [num_eos].
 * masks (uint32 [num_states + 1, ceil(vocab / 32)], written whole) gets, for s < S, bit t iff token t has bytes and
 * walking them from s never reaches -1, or t is an EOS id and accept[s]; row S (terminal) has exactly the EOS bits.
 * reach (uint32 [num_states, ceil(num_states / 32)], zeroed by the caller) gets bit e of row s for every allowed token
 * with bytes that leads from s to e.  The table is staged in shared memory up to 192 states (16-byte aligned dfa),
 * read from global memory beyond.  Deterministic. */
int tl_constraint_token_masks(const int32_t *dfa, const uint8_t *accept, int num_states, const int32_t *token_offsets,
                              const uint8_t *token_bytes, int vocab, const int32_t *eos_ids, int num_eos, uint32_t *masks, uint32_t *reach,
                              void *stream);
/* tl_sample (repetition, presence, frequency, min_p and state all NULL) or tl_sample_penalized (all given) restricted
 * per row to the tokens constraints[r] allows (read after the programmatic-dependent-launch wait).  For a row with a
 * mask, after staging and after the penalty rewrite the entries of disallowed tokens (every entry when the state is
 * outside [0, S]) are dropped as NaN entries are: the first-maximum argmax of greedy and non-finite-maximum rows,
 * the top-k count, the top-p mass, min-p's maximum and the Gumbel draw (Philox counters unchanged) all run on the
 * allowed entries.  A row whose mask allows every token therefore draws exactly the unconstrained kernel's token.
 * The token is always allowed: a row without an allowed non-NaN entry returns the lowest allowed id (0 if none).
 * After the draw, for rows with a mask and positions[r] > 0, constraints[r].state becomes S when the token has no
 * bytes (EOS) or the state was S, else the DFA walk of its bytes.  Log-probabilities (tl_logprobs) are unaffected. */
int tl_sample_constrained(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                          const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                          const float *min_p, int32_t *state, tl_constraint_row *constraints, int32_t *out_tokens, int rows, int vocab,
                          int dtype, void *stream);
/* tl_sample_constrained with xtc_threshold and xtc_probability as tl_sample_penalized_xtc takes them (both NULL, or
 * both given with the penalty arrays): K, S and A are taken over the allowed entries only. */
int tl_sample_constrained_xtc(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                              const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                              const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability,
                              tl_constraint_row *constraints, int32_t *out_tokens, int rows, int vocab, int dtype, void *stream);
/* tl_sample_constrained_xtc with the truncation arrays as tl_sample_penalized_trunc takes them (with the penalty arrays):
 * every sum and keep set is taken over the allowed entries only. */
int tl_sample_constrained_trunc(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                                const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                                const float *min_p, int32_t *state, const float *xtc_threshold, const float *xtc_probability,
                                const float *typical_p, const float *top_n_sigma, const float *mirostat_tau, const float *mirostat_eta,
                                float *mirostat_mu, tl_constraint_row *constraints, int32_t *out_tokens, int rows, int vocab, int dtype,
                                void *stream);
/* JSON mode (DESIGN.md section 20): a byte-level pushdown automaton over RFC 8259 `ws object ws`, with at most
 * TL_JSON_MAX_DEPTH open containers and at most TL_JSON_MAX_WS_RUN consecutive whitespace bytes.  A JSON row is a
 * tl_constraint_row with num_states = 1 whose mask is the row's own uint32 [2, ceil(vocab / 32)] buffer (row 0: this
 * step's mask, written by tl_json_token_masks; row 1: EOS only) and whose dfa is an all-zero int32 [1, 256] table, so
 * tl_sample_constrained keeps state 0 for a token with bytes and moves to 1 (terminal) on EOS.  Its automaton state is
 * two int64 words per row:
 *   word 0         the container stack: bit d set iff the container at depth d + 1 is an array;
 *   word 1         bits 0-6 depth, 8-12 lexer state, 16-21 current whitespace run, 24-26 and 27-29 the lexer state's
 *                  progress (UTF-8 bytes to go and the next byte's range, hex digits to go, literal and index),
 *                  30 the open string is a key, 32 the row is in JSON mode, 33 terminal (after EOS).
 * Lexer state 7 is "closed": the top-level object has closed and only whitespace and EOS may follow. */
#define TL_JSON_MAX_DEPTH 64
#define TL_JSON_MAX_WS_RUN 32
/* Row 0 of every JSON row's mask (rows with bit 32 set and bit 33 clear; others are not touched), in one launch: bit t
 * iff token t has bytes and walking them from the row's state stays in the language within both caps, or t has no
 * bytes, the text is complete and bit t of the row's mask row 1 is set.  The vocabulary is the row's descriptor's
 * token_offsets / token_bytes.  Deterministic, no atomics. */
int tl_json_token_masks(const tl_constraint_row *constraints, const int64_t *json_states, int rows, int vocab, void *stream);
/* After the draw: for JSON rows with positions[r] > 0 and not terminal, the state becomes the walk of tokens[r]'s
 * bytes, or terminal when the token has no bytes (EOS).  Other rows are unchanged. */
int tl_json_advance(const tl_constraint_row *constraints, int64_t *json_states, const int32_t *tokens, const int32_t *positions, int rows,
                    void *stream);
/* JSON Schema structured outputs (DESIGN.md section 21): a byte-level pushdown automaton compiled from a schema into
 * one table blob per schema (json_schema.py writes it; 16-byte aligned):
 *   int32 num_states S, num_classes C, blob bytes, num_actions A;  uint8 class_of[256];
 *   uint32 info[S]      bit 0 whitespace counts here, bit 1 accepting, bits 8-15 need (stack entries the cheapest
 *                       completion from the state still pushes);
 *   uint32 actions[A]   bits 0-1 kind (0 checked shift, 1 call, 2 return, 3 return and reprocess the byte), 2-16
 *                       target, 17-31 return;
 *   uint16 trans[S, C]  0 fail, 1-0x7FFF a plain shift to that state (its need is at most the source's, so the depth
 *                       cap holds unchecked), 0x8000 | a action a.
 * State 0 is dead.  A schema row is a tl_constraint_row exactly like a JSON row (num_states 1, its own uint32
 * [2, ceil(vocab / 32)] mask buffer, the all-zero dfa).  Its automaton state is TL_SCHEMA_STATE_WORDS int64 words:
 *   word 0         the row's table blob (0: not a schema row);
 *   word 1         bits 0-14 state, 16-21 depth (stack entries), 24-29 current whitespace run, 32 the row is in schema
 *                  mode, 33 terminal (after EOS);
 *   words 2-9      the stack of return states, 16 bits each, entry k at word 2 + k / 4, bits 16 (k % 4); entries at
 *                  or above the depth are 0.
 * A byte in a state: look up the entry; a reprocess entry pops the return state and looks the byte up there.  In a
 * whitespace state the run grows on whitespace (at most TL_JSON_MAX_WS_RUN); any other byte resets it.  A checked
 * shift to t needs depth + need(t) <= TL_SCHEMA_MAX_DEPTH, a call (t, r) depth + 1 + need(t) and depth + need(r)
 * within it. */
#define TL_SCHEMA_MAX_DEPTH 32
#define TL_SCHEMA_MAX_ITEMS 64
#define TL_SCHEMA_MAX_STATES 32767
#define TL_SCHEMA_MAX_TABLE_BYTES (1 << 22)
#define TL_SCHEMA_SMEM_BYTES (47 * 1024)
#define TL_SCHEMA_STATE_WORDS 10
/* Row 0 of every schema row's mask (rows with bit 32 of word 1 set and bit 33 clear; others are not touched), in one
 * launch: bit t iff token t has bytes and walking them from the row's state stays in the language, or t has no bytes,
 * the text is complete (accepting state, depth 0) and bit t of the row's mask row 1 is set.  smem_bytes (a multiple of
 * 16, at most TL_SCHEMA_SMEM_BYTES) is the dynamic shared memory of each CTA: a row's blob is staged there when it
 * fits and read through L1/L2 otherwise, with the same result (size it to the largest blob that fits, or 0).
 * Deterministic, no atomics. */
int tl_schema_token_masks(const tl_constraint_row *constraints, const int64_t *schema_states, int rows, int vocab, int smem_bytes,
                          void *stream);
/* After the draw: for schema rows with positions[r] > 0 and not terminal, the state becomes the walk of tokens[r]'s
 * bytes (the dead state when it leaves the language), or terminal when the token has no bytes (EOS). */
int tl_schema_advance(const tl_constraint_row *constraints, int64_t *schema_states, const int32_t *tokens, const int32_t *positions,
                      int rows, void *stream);
/* Grammar-constrained generation (DESIGN.md section 23): a byte-level pushdown automaton compiled from a GBNF grammar
 * into one table blob per grammar (grammar.py writes it; 16-byte aligned):
 *   int32 num_states S (ids 0..S-1, 0 dead), num_classes C, blob bytes, action words A;  uint8 class_of[256];
 *   uint32 info[S]      bit 0 the state's rule may end here, bits 8-15 need (stack entries the cheapest completion
 *                       from the state still pushes);
 *   uint32 trans[S, C]  0 no action, else bits 0-23 the first action word in acts, bits 24-31 the action count;
 *   uint32 acts[A]      per action one word (bits 0-14 target, 16-21 pushes k, 24-31 peak: the most stack entries the
 *                       chain's cheapest completion holds above the current depth), then ceil(k / 2) words of 16-bit
 *                       return states, bottom first, low half first.
 * A grammar row is a tl_constraint_row exactly like a JSON row (num_states 1, its own uint32 [2, ceil(vocab / 32)] mask
 * buffer, the all-zero dfa).  Its state is a set of at most TL_GRAMMAR_MAX_PARSES parses in TL_GRAMMAR_STATE_WORDS
 * int64 words:
 *   word 0         the row's table blob (0: not a grammar row);
 *   word 1         bits 0-3 the parse count n, 32 the row is in grammar mode, 33 terminal (after EOS), 34 failed (a
 *                  drawn token was not allowed);
 *   words 2-9      parse p < n: bits 0-14 state, 16-21 depth; others 0;
 *   words 10-73    the return stacks, 16 bits each: entry k of parse p at uint16 index p * TL_GRAMMAR_MAX_DEPTH + k;
 *                  entries at or above a parse's depth are 0.
 * A byte over the set: for each parse in order, each action of its state on the byte's class (in table order) whose
 * depth + peak <= TL_GRAMMAR_MAX_DEPTH makes a parse (target, stack + pushes), kept unless an equal (state, depth,
 * stack) parse was made before; then, while the state's rule may end and the depth is above 0, the return state is
 * popped and its actions are taken the same way.  The byte fails when no parse is made or when a parse beyond
 * TL_GRAMMAR_MAX_PARSES would be kept.  The text is complete when some parse, popping through states whose rule may
 * end, reaches depth 0 in such a state. */
#define TL_GRAMMAR_MAX_STATES 32767
#define TL_GRAMMAR_MAX_DEPTH 32
#define TL_GRAMMAR_MAX_PARSES 8
#define TL_GRAMMAR_MAX_TABLE_BYTES (1 << 22)
#define TL_GRAMMAR_SMEM_BYTES (46 * 1024)
#define TL_GRAMMAR_STATE_WORDS 74
/* Row 0 of every grammar row's mask (rows with bit 32 of word 1 set and bit 33 clear; others are not touched), in one
 * launch: bit t iff token t has bytes and walking them from the row's parse set never fails, or t has no bytes, the
 * text is complete and bit t of the row's mask row 1 is set.  smem_bytes (a multiple of 16, at most
 * TL_GRAMMAR_SMEM_BYTES) is the dynamic shared memory of each CTA: a row's blob is staged there when it fits and read
 * through L1/L2 otherwise, with the same result.  Deterministic, no atomics. */
int tl_grammar_token_masks(const tl_constraint_row *constraints, const int64_t *grammar_states, int rows, int vocab, int smem_bytes,
                           void *stream);
/* After the draw: for grammar rows with positions[r] > 0, neither terminal nor failed, the parse set becomes the walk of
 * tokens[r]'s bytes, or terminal when the token has no bytes, is an EOS id (bit set in the row's mask row 1) and the
 * text is complete.  A token that is not allowed (drawn only when the row allows none) leaves n = 0, every parse and
 * stack word 0 and the failed bit set; callers must refuse such a row. */
int tl_grammar_advance(const tl_constraint_row *constraints, int64_t *grammar_states, const int32_t *tokens, const int32_t *positions,
                       int rows, int vocab, void *stream);
/* Log-probabilities of logits [rows, vocab] (rows <= 65535, vocab <= 409,600; fp32, fp16 or bf16 read as fp32), one
 * launch, one cluster of CTAs per row (DESIGN.md section 8a).
 *
 * The distribution reported is the raw model distribution, lp_i = x_i - m - log S with m the row maximum and
 * S = sum_i exp(x_i - m): the reference's logits - logsumexp(logits).  Temperature, top-k and top-p do not enter it;
 * a sampled token reports its raw log-probability.  Rounding points, in order:
 *   d_i = fl32(x_i - m);  e_i = expf(d_i);  E_i = round-to-nearest(e_i * 2^40) as a 64-bit integer;
 *   S_fx = sum_i E_i over the non-NaN entries (exact, so the same bits in any order, row count, row index or graph);
 *   log_s = logf(fl32(S_fx) * 2^-40)  (the conversion rounds, the scaling is exact: S >= 1);
 *   lp(x) = fl32(fl32(x - m) - log_s),  lse = fl32(m + log_s).
 * Per row r, written at row o = r + (out_index ? *out_index * rows : 0); with out_index (device), the outputs are logs
 * of out_capacity such blocks and a launch whose *out_index is outside [0, out_capacity) writes nothing (as
 * tl_decode_advance treats its token log; out_capacity is ignored without out_index):
 *   lse[o];
 *   targets (device, may be NULL: every target -1): for t = targets[r] in [0, vocab), target_lp[o] = lp(x_t) and
 *     target_rank[o] = 1 + #{i : x_i > x_t}; t outside [0, vocab) or x_t NaN gives NaN and rank 0;
 *   top_n (device, may be NULL: max_n for every row), 0 <= max_n <= TL_LOGPROBS_MAX_N: the min(top_n[r], max_n)
 *     largest entries in top_ids[o * max_n + j] (int32) and top_lp[...] (lp(x), the target's expression: bit-identical
 *     when the target is listed), in descending order with ties to the lower id (tl_argmax's first-maximum rule);
 *     slots past the listed entries hold id -1 and -inf.  top_ids / top_lp may be NULL when max_n == 0.
 * NaN entries are never listed, never counted in S and never counted in a rank; -inf entries are ordinary entries
 * with lp -inf.  A row whose maximum is not finite (+inf, every non-NaN entry -inf, or every entry NaN) reports
 * lse = that maximum (NaN when every entry is NaN) and NaN for every lp, with ranks and top-N ids by the rules above.
 * targets and top_n are read after the programmatic-dependent-launch wait, so the previous launch may write them.
 * No workspace; deterministic. */
#define TL_LOGPROBS_MAX_N 20
int tl_logprobs(const void *logits, const int32_t *targets, const int32_t *top_n, const int32_t *out_index, float *lse, float *target_lp,
                int32_t *target_rank, int32_t *top_ids, float *top_lp, int rows, int vocab, int max_n, int out_capacity, int dtype,
                void *stream);
/* Fused W4A16 projection for the decode hot loop: the weight-streaming kernel of
 * tl_quantized_matmul with the neighbouring element-wise operator folded in.
 * Rounding points are those of the unfused call sequence, so results are
 * bit-identical to it.
 *   prologue TL_PRO_NONE    : a = p0 [M, N]
 *            TL_PRO_RMSNORM : a = rms_norm(p0 [M, N], p1 [N], eps)      (then projected)
 *            TL_PRO_SWIGLU  : a = swiglu(p0 = gate [M, N], p1 = up [M, N])
 *   epilogue TL_EPI_NONE    : out = result
 *            TL_EPI_RESIDUAL: out = residual [M, K] + result
 *            TL_EPI_SWIGLU_PAIRS: out [M, K/2]; the weight rows are gate and up rows interleaved in
 *                             blocks of 8 (rows 16c..16c+7 = gate 8c..8c+7, rows 16c+8..16c+15 = up
 *                             8c..8c+7; K % 16 == 0) and out[m, 8c+r] = swiglu(T(gate), T(up)): the
 *                             MLP activation leaves the gate|up projection already combined
 *                             (week2_kernels.metal:115-116 applied to the rounded projection outputs)
 * lda is the row stride (elements) of p0 (and of p1 for SWIGLU), so gate/up may
 * be the two halves of one [M, 2N] buffer.
 * With 9 <= M <= 128, no prologue and lda == N the launch goes to the swap-AB wgmma kernel (same
 * epilogues; weights rounded to the activation dtype like every tensor-core path) and needs
 * tl_quantized_matmul_fused_workspace() bytes of workspace. */
enum { TL_PRO_NONE = 0, TL_PRO_RMSNORM = 1, TL_PRO_SWIGLU = 2 };
enum { TL_EPI_NONE = 0, TL_EPI_RESIDUAL = 1, TL_EPI_SWIGLU_PAIRS = 2 };
size_t tl_quantized_matmul_fused_workspace(int M, int N, int K, int lda, int prologue, int dtype);
int tl_quantized_matmul_fused(const void *scales, const void *biases, const void *b, void *out, const void *p0,
                              const void *p1, const void *residual, int M, int N, int K, int lda, int prologue,
                              int epilogue, float eps, int dtype, void *workspace, size_t workspace_bytes, void *stream);
size_t tl_quantized_matmul_fused_workspace_bits(int M, int N, int K, int lda, int prologue, int dtype, int bits);
int tl_quantized_matmul_fused_bits(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *p1,
                                   const void *residual, int M, int N, int K, int lda, int prologue, int epilogue, float eps, int dtype, int bits,
                                   void *workspace, size_t workspace_bytes, void *stream);
/* out = residual + projection(p0) and, in the same call, normed_out = rms_norm(out, norm_weight, norm_eps): the
 * residual-stream projections (o, down) of qwen3_week3.py:204-206 followed by the RMSNorm that opens the next block
 * (:195-199).  Same rounding points as tl_quantized_matmul_fused(TL_EPI_RESIDUAL) then tl_rms_norm; with a split
 * reduction (9 <= M <= 128) the normalisation happens inside the kernel that adds the partial planes.  p0 is contiguous
 * [M, N]; workspace as for tl_quantized_matmul_fused(prologue TL_PRO_NONE). */
int tl_quantized_matmul_residual_norm(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *residual,
                                      const void *norm_weight, void *normed_out, int M, int N, int K, float norm_eps, int dtype, void *workspace,
                                      size_t workspace_bytes, void *stream);
int tl_quantized_matmul_residual_norm_bits(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *residual,
                                           const void *norm_weight, void *normed_out, int M, int N, int K, float norm_eps, int dtype, int bits,
                                           void *workspace, size_t workspace_bytes, void *stream);
/* q|k|v projection of `rows` activation rows (p0 [rows, N], packed weight rows = q heads | k heads | v heads) followed by
 * per-head q/k RMSNorm + RoPE + K/V append (tl_decode_qk_norm_rope_append, or its chunk form when chunk != 0).  With a
 * split reduction (9..128 rows) the partial planes feed the second kernel directly and q|k|v is never materialised;
 * otherwise qkv_scratch [rows, (Hq + 2 Hkv) * D] receives it.  Same results as the two calls.  bfloat16; workspace as
 * for tl_quantized_matmul_fused(prologue TL_PRO_NONE). */
int tl_qkv_project_rope_append(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch, const void *q_norm_weight,
                               const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table, const int32_t *context_lens, void *q_out,
                               void *key_pages, void *value_pages, int rows, int N, int num_heads, int num_kv_heads, int head_dim, float base, float eps,
                               int num_pages, int page_size, int max_pages, int chunk, int dtype, void *workspace, size_t workspace_bytes, void *stream);
int tl_qkv_project_rope_append_table(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch,
                                     const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table,
                                     const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int rows, int N, int num_heads,
                                     int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size, int max_pages, int chunk,
                                     int dtype, void *workspace, size_t workspace_bytes, void *stream, const double *inv_freq);
int tl_qkv_project_rope_append_bits(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch,
                                    const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table,
                                    const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int rows, int N, int num_heads,
                                    int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size, int max_pages, int chunk,
                                    int dtype, int bits, void *workspace, size_t workspace_bytes, void *stream);
int tl_qkv_project_rope_append_table_bits(const void *scales, const void *biases, const void *b, const void *p0, void *qkv_scratch,
                                          const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets, const int32_t *block_table,
                                          const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int rows, int N, int num_heads,
                                          int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size, int max_pages,
                                          int chunk, int dtype, int bits, void *workspace, size_t workspace_bytes, void *stream,
                                          const double *inv_freq);
/* Decode step, L == 1: per-head q/k RMSNorm + RoPE + K/V append in one launch.
 * qkv [B, (Hq + 2*Hkv) * D] (q heads | k heads | v heads); q_out [B, Hq, D];
 * K/V rows land in the page slot of token context_lens[b]-1 (rows with context
 * 0 are skipped).  Non-traditional RoPE over the full head dimension. */
int tl_decode_qk_norm_rope_append(const void *qkv, const void *q_norm_weight, const void *k_norm_weight,
                                  const int32_t *offsets, const int32_t *block_table, const int32_t *context_lens,
                                  void *q_out, void *key_pages, void *value_pages, int batch, int num_heads,
                                  int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size,
                                  int max_pages, int dtype, void *stream);
int tl_decode_qk_norm_rope_append_table(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                        const int32_t *block_table, const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages,
                                        int batch, int num_heads, int num_kv_heads, int head_dim, float base, float eps, int num_pages,
                                        int page_size, int max_pages, int dtype, void *stream, const double *inv_freq);
/* The kernel tl_decode_qk_norm_rope_append, tl_chunk_qk_norm_rope_append and the second half of
 * tl_qkv_project_rope_append run (nothing is launched), or a negative TL_E* code for arguments they reject:
 * TL_QKN_ROW, one CTA per row with 16 warps sharing the row's angles (bf16, D == 128, Hq + 2 Hkv <= 64; the only
 * kernel that reads split-reduction planes), else TL_QKN_HEAD, one CTA per (head, row). */
enum { TL_QKN_HEAD = 0, TL_QKN_ROW = 1 };
int tl_qk_norm_rope_route(int num_heads, int num_kv_heads, int head_dim, int dtype);
/* Prefill-chunk form of the same kernel: the rows of qkv [tokens, (Hq + 2*Hkv) * D] are consecutive tokens of ONE
 * request (one shared block-table row, int32 [max_pages]); offsets[t] is the RoPE position and context_lens[t]
 * the post-append length of token t (0 = padding row: nothing is appended), all DEVICE data, so a captured
 * chunk replays for any position.  q_out is [Hq, tokens, D] - the layout tl_paged_attention takes.  Replaces,
 * for one chunk, rms_norm x2 + rope x2 + the paged_cache_update calls of qwen3_week3.py:62-84. */
int tl_chunk_qk_norm_rope_append(const void *qkv, const void *q_norm_weight, const void *k_norm_weight,
                                 const int32_t *offsets, const int32_t *block_table_row, const int32_t *context_lens,
                                 void *q_out, void *key_pages, void *value_pages, int tokens, int num_heads,
                                 int num_kv_heads, int head_dim, float base, float eps, int num_pages, int page_size,
                                 int max_pages, int dtype, void *stream);
int tl_chunk_qk_norm_rope_append_table(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                       const int32_t *block_table_row, const int32_t *context_lens, void *q_out, void *key_pages,
                                       void *value_pages, int tokens, int num_heads, int num_kv_heads, int head_dim, float base, float eps,
                                       int num_pages, int page_size, int max_pages, int dtype, void *stream, const double *inv_freq);
/* Chunk append (CUDA extension of paged_cache_update, paged_attention.cpp:14-31): the rows of ONE
 * request's key/value chunk [1, H, L, D] (element strides src_head_stride / src_token_stride, unit
 * inner stride) are written into up to TL_PAGE_SPANS page slices in one launch:
 * pages[page_id[i], :, start[i]:start[i]+count[i], :] = chunk[0, :, src[i]:src[i]+count[i], :].
 * `spans` is a HOST pointer (passed by value to the kernel). */
#define TL_PAGE_SPANS 64
typedef struct tl_page_span_list {
    int32_t page_id[TL_PAGE_SPANS], start[TL_PAGE_SPANS], count[TL_PAGE_SPANS], src[TL_PAGE_SPANS];
    int32_t n;
} tl_page_span_list;
int tl_paged_cache_append_chunk(void *key_pages, void *value_pages, const void *keys, const void *values,
                                const tl_page_span_list *spans, int num_pages, int heads, int page_size, int head_dim,
                                long long src_head_stride, long long src_token_stride, int dtype, void *stream);
/* Prefix copy-on-write (prefix caching): for every record i of `copies`, in ONE launch,
 *   key_slab[layer][dst, :, 0:slots, :] = key_slab[layer][src, :, 0:slots, :]   (and the same for values)
 * over slabs [num_pages[layer], heads, page_size, head_dim] that share heads, page_size, head_dim and dtype.
 * Rows at or beyond `slots` of the destination are not written; the source is never written.  Both records are
 * HOST pointers passed by value to the kernel: together 3.3 KiB, under the 4 KiB kernel-parameter limit, so a
 * longer list goes out as several launches.  Checked before any device call: dtype, layer < slabs->n, both pages
 * inside that layer's slab, 1 <= slots <= page_size, src != dst, no destination named twice in one layer and no
 * page that is a destination and a source in one layer (the records of a launch run concurrently). */
#define TL_PREFIX_COPY_LAYERS 64
#define TL_PREFIX_COPIES 128
typedef struct tl_kv_slab_table {
    void *key[TL_PREFIX_COPY_LAYERS];
    void *value[TL_PREFIX_COPY_LAYERS];
    int32_t num_pages[TL_PREFIX_COPY_LAYERS];
    int32_t n;
} tl_kv_slab_table;
typedef struct tl_prefix_copy_list {
    int32_t layer[TL_PREFIX_COPIES], src[TL_PREFIX_COPIES], dst[TL_PREFIX_COPIES], slots[TL_PREFIX_COPIES];
    int32_t n;
} tl_prefix_copy_list;
int tl_paged_cache_copy_prefix(const tl_kv_slab_table *slabs, const tl_prefix_copy_list *copies, int heads, int page_size,
                               int head_dim, int dtype, void *stream);
/* Fused decode attention, L == 1 (bf16, head_dim 128, <= 4 query heads per KV head): per-head
 * q/k RMSNorm + RoPE, append of the newest K/V row and paged GQA attention in ONE launch (plus a
 * merge launch when the context is split over several CTAs).  Replaces, with the same rounding
 * points, the call sequence rms_norm, rms_norm, rope, rope, paged_cache_update, paged_attention
 * of src/tiny_llm_ref/qwen3_week3.py:62-105.  qkv [B, (Hq + 2 Hkv) * 128] is the
 * row-concatenated projection output; context_lens are post-append; rope_inv_freq holds the 64
 * float64 frequencies (base^(-i/64), or a scaled table as for the *_table entry points); out [B, Hq * 128]; max_context bounds every context_lens[b]
 * (it fixes the split count, so a captured launch stays valid as the contexts grow);
 * workspace: tl_decode_attention_fused_workspace() floats.  A context longer than the block table
 * (max_pages * page_size) is clamped to it for the attention and for the append alike: the row's
 * K/V land in the table's last slot.  tl_decode_qk_norm_rope_append skips such a row instead. */
size_t tl_decode_attention_fused_workspace(int batch, int num_heads, int num_kv_heads);
int tl_decode_attention_fused(const void *qkv, const void *q_norm_weight, const void *k_norm_weight,
                              const int32_t *offsets, const int32_t *block_table, const int32_t *context_lens,
                              const double *rope_inv_freq, void *key_pages, void *value_pages, void *out,
                              float *workspace, int batch, int num_heads, int num_kv_heads, int head_dim, float eps,
                              float scale, int num_pages, int page_size, int max_pages, int max_context, int dtype,
                              void *stream);
/* The same with rows_per_request (1..8) consecutive query rows per request, e.g. the verify pass of
 * speculative decoding: qkv [B R, (Hq + 2 Hkv) * 128], offsets / context_lens [B R], out [B R, Hq * 128],
 * block_table [B, max_pages] shared by the rows of a request.  Row j of a request must have context
 * context_lens[row 0] + j (or all rows 0: an idle request).  Each row's output, and the K/V it appends, equal
 * bit for bit tl_decode_attention_fused run on that row alone with the rows before it already appended (the
 * split count follows B and max_context, not B R).  rows_per_request == 1 is tl_decode_attention_fused. */
size_t tl_decode_attention_fused_rows_workspace(int batch, int rows_per_request, int num_heads, int num_kv_heads);
int tl_decode_attention_fused_rows(const void *qkv, const void *q_norm_weight, const void *k_norm_weight,
                                   const int32_t *offsets, const int32_t *block_table, const int32_t *context_lens,
                                   const double *rope_inv_freq, void *key_pages, void *value_pages, void *out,
                                   float *workspace, int batch, int rows_per_request, int num_heads, int num_kv_heads,
                                   int head_dim, float eps, float scale, int num_pages, int page_size, int max_pages,
                                   int max_context, int dtype, void *stream);
/* ---- Qwen3-MoE sparse block (moe.py:36-89 of the reference) ----------------
 * One layer runs: router projection (tl_quantized_matmul*, or tl_moe_router for 8-bit group-64 routers), tl_moe_topk, tl_moe_group, tl_moe_gather,
 * tl_moe_grouped_matmul (gate|up, EPI_SWIGLU_PAIRS, sorted output), tl_moe_grouped_matmul (down, scattered back to
 * the original row order with out_index = perm), tl_moe_combine.  All are capture-safe: outputs are sized by
 * R = T * k rows and E experts, nothing synchronises and no count is read by the host.  Rounding (DESIGN.md):
 *   probs = T(softmax_fp32(logits)); ids = the k largest probs, descending, ties to the lower id; scores = probs[ids],
 *   with norm: T(score / T(sum_fp32 scores in slot order)); expert outputs rounded to T; SwiGLU rounded once;
 *   r = T(sum_fp32 over slots of T(y_j * score_j)); x' = T(x + r).
 * A row's result depends only on that row. */
#define TL_MOE_MAX_EXPERTS 256
#define TL_MOE_MAX_TOPK 8
/* logits [T, E] -> probs [T, E] (dtype of logits), ids int32 [T, k], scores [T, k].  E <= 256, 1 <= k <= min(8, E).
 * A NaN probability ranks below every number: a row whose softmax is NaN (a NaN or +inf logit, every logit -inf) gives
 * ids 0..k-1 and NaN scores. */
int tl_moe_topk(const void *logits, void *probs, int32_t *ids, void *scores, int T, int E, int k, int norm_topk_prob, int dtype, void *stream);
/* ids int32 [R] (each in [0, E); others are clamped) -> offsets int32 [E + 1] (segment of expert e in sorted order),
 * perm int32 [R] (sorted position -> row, stable within an expert) and, with nt > 0, the tile table of the grouped
 * GEMM: tiles int32 [tl_moe_tile_table_size(R, E, nt)] = {count, (expert, first sorted row) x count}, one entry per
 * nt-row piece of each expert's segment, experts in order. */
int tl_moe_group(const int32_t *ids, int R, int E, int nt, int32_t *offsets, int32_t *perm, int32_t *tiles, void *stream);
int tl_moe_tile_table_size(int R, int E, int nt);
/* xs[j] = x[perm[j] / rows_per_source] for j < R; x [R / rows_per_source, H].  With norm_weight: the row's RMSNorm
 * T(x * rsqrt(mean(x^2) + eps) * w). */
int tl_moe_gather(const void *x, const int32_t *perm, const void *norm_weight, float eps, void *xs, int R, int rows_per_source, int H, int dtype,
                  void *stream);
/* Grouped W4A16 projection of R = T * k expert-sorted rows a [R, N] by the experts b [E K, N / 8], scales / biases
 * [E K, N / 128]: row j uses expert e with offsets[e] <= j < offsets[e + 1].  out [R, K] (EPI_NONE) or [R, K / 2]
 * (EPI_SWIGLU_PAIRS over each expert's interleaved gate|up rows), row j stored at out_index[j] when out_index is given,
 * else at j.  tiles: tl_moe_group's table for the nt tl_moe_grouped_matmul_route reports (unused on the control route). */
int tl_moe_grouped_matmul(const void *scales, const void *biases, const void *b, const void *a, void *out, const int32_t *offsets,
                          const int32_t *tiles, const int32_t *out_index, int T, int k, int E, int N, int K, int epilogue, int dtype, void *stream);
/* The kernel tl_moe_grouped_matmul runs (nothing is launched or read; a and b only count for their alignment):
 *   TL_MOE_WGMMA   : the swap-AB wgmma kernel, one CTA = 128 features of one expert x nt sorted rows, no split;
 *                    16-bit dtype, K % 128 == 0, a and b 16-byte aligned.  nt = the smallest of 16 / 32 / 64 / 128 at
 *                    least ceil(T k / E); *max_tiles = the CTA rows launched;
 *   TL_MOE_CONTROL : the scalar control kernel (one thread per output); *nt = *max_tiles = 0.
 * or a negative TL_E* code for arguments the launch rejects. */
enum { TL_MOE_CONTROL = 0, TL_MOE_WGMMA = 1 };
int tl_moe_grouped_matmul_route(int T, int k, int E, int N, int K, int epilogue, int dtype, const void *a, const void *b, int *nt, int *max_tiles);
/* Router projection of a router stored as MLX affine 8-bit codes at group 64 (the group-128 projection entries take
 * the others): w uint32 [E, H / 4] (code j of a word in bits [8 j, 8 j + 8)), scales / biases [E, H / 64] and x [T, H]
 * of one 16-bit dtype, logits [T, E]:
 *   logits[t, e] = T(sum over groups g, in a fixed order, of fp32 scale[e, g] * sum_k code[e, k] a[t, k]
 *                                                             + bias[e, g] * sum_k a[t, k])      (k in group g)
 * i.e. sum_k (scale * code + bias) * a in fp32, rounded once.  With norm_weight [H] (else NULL) a = the row's RMSNorm
 * T(x * rsqrt(mean(x^2) + eps) * w), bit for bit tl_rms_norm's output; without it a = x.  E <= 256, H % 64 == 0,
 * 0 <= T <= TL_MOE_ROUTER_MAX_ROWS; x, w and norm_weight 16-byte aligned.  A row's logits depend only on that row.
 * Other arguments: TL_EINVAL. */
#define TL_MOE_ROUTER_MAX_ROWS (1 << 19)
int tl_moe_router(const void *x, const void *norm_weight, float eps, const void *w, const void *scales, const void *biases, void *logits, int T,
                  int E, int H, int dtype, void *stream);
/* out [T, H] = T(residual + T(sum_fp32 over j < k of T(y[t k + j] * scores[t, j]))) (no residual: the sum alone);
 * y [T k, H] in original row order.  With norm_weight, normed_out = the RMSNorm of out (H <= 4096). */
int tl_moe_combine(const void *y, const void *scores, const void *residual, const void *norm_weight, float eps, void *out, void *normed_out,
                   int T, int k, int H, int dtype, void *stream);

/* ---- Multi-LoRA: per-row bf16 low-rank adapters over a projection's output (DESIGN.md section 12) ----------------
 * A SITE is one projection input x [M, N] with up to three output SEGMENTS (q|k|v: 3, o: 1, gate|up: 2, down: 1).
 * Segment s of row m is the K_s elements at y[s] + m * ldy[s] (host arrays of nseg entries): the segments of one packed
 * projection side by side (y[s] = base + K_0 + .. + K_{s-1}, ldy[s] = their sum) or one tensor per projection; the
 * optional residual (host array of nseg pointers, or NULL) has the layout of y.  Per adapter a and segment s there is A_s [r_a, N] and
 * B_s [K_s, r_a] in bf16 and sc_a = alpha / r_a in fp32.  For a row x (T = bf16) with adapter_ids[row] = a >= 0:
 *   t_j = T(sum_fp32_i A_s[j,i] * x_i)                 j < r_a  (the intermediate is rounded once, as PEFT's is)
 *   s_o = sum_fp32_j B_s[o,j] * float(t_j)             fp32, fmaf over j ascending from +0
 *   y_o = T(fmaf(sc_a, s_o, float(base_o)))            one fp32 rounding of base_o + sc_a * s_o, then T; base_o: y as the
 *                                                      projection left it (already rounded)
 * and, with a residual: y_o = T(float(residual_o) + float(y_o)), the operator sequence add(x, lora(proj(h))).
 * A row with adapter_ids[row] < 0 keeps base's bits (with a residual: T(residual + base)), and so does a segment the
 * adapter's seg_mask does not name; nothing outside rows [0, M) of y is written.
 * The i-sum runs in an order fixed by N alone: each of 8 CTAs takes ceil(N / 64) whole 8-element chunks, a lane its
 * chunks 32 apart in ascending order with one fmaf per element, then the xor butterfly over the lanes, then the CTAs in
 * order.  A row's result is therefore a pure function of that row and its adapter: the same bits alone, at any index of
 * any launch, on either route and under graph replay.
 * Storage is padded to the set's r_max with zeros: a [n_adapters, nseg * r_max, N] (segment s at rows s * r_max ..),
 * b[s] [n_adapters, K_s, r_max]; rows / columns >= ranks[a] are never read, which equals adding their exact zeros.
 * ranks[a] in {8, 16, 32, 64}; N % 8 == 0, N <= 12288; a, b[s], x 16-byte aligned.  Capture-safe: nothing is
 * allocated or synchronised, adapter_ids is device data read after griddepcontrol.wait.
 * Routes (tl_lora_apply_route; nothing is launched or read):
 *   TL_LORA_ROWS  (M <= 64)  one 8-CTA cluster per row;
 *   TL_LORA_TILES (M > 64)   one cluster per 8 consecutive rows: when they name one adapter (a prefill chunk) they share
 *                            every load of A and B, each row still summed as above, so the bits are those of
 *                            TL_LORA_ROWS; otherwise the cluster runs its rows one after the other.
 * Both routes run on CUDA cores; there is no tensor-core route yet. */
#define TL_LORA_MAX_SEGMENTS 3
#define TL_LORA_MAX_RANK 64
#define TL_LORA_MAX_ADAPTERS 32
typedef struct tl_lora_site {
    const void *a;           /* bf16 [n_adapters, nseg * r_max, N] */
    const void *b[3];        /* bf16 [n_adapters, K_s, r_max] per segment */
    const float *scales;     /* [n_adapters] alpha / r */
    const int32_t *ranks;    /* [n_adapters] */
    const int32_t *seg_mask; /* [n_adapters] bit s: the adapter targets segment s */
    int32_t n_adapters, nseg, r_max, N;
    int32_t K[3];
} tl_lora_site;
enum { TL_LORA_ROWS = 0, TL_LORA_TILES = 1 };
int tl_lora_apply_route(int M, int dtype, const tl_lora_site *site);
int tl_lora_apply(const void *x, void *const *y, const void *const *residual, const long long *ldy, const int32_t *adapter_ids,
                  const tl_lora_site *site, int M, int dtype, void *stream);

/* Programmatic dependent launch for the streaming kernels (on by default; 0 turns it off,
 * TL_PDL=0 in the environment does the same). */
int tl_set_pdl(int enabled);
/* Device-side bookkeeping between two decode steps of a CUDA-graph loop (the
 * per-request `req.decode_done(token)` + `offset += 1` of batch.py:241-247 done
 * without a host round trip): for every ACTIVE row (context_lens > 0)
 *   tokens[b] = next_tokens[b]; offsets[b] += 1; context_lens[b] += 1;
 * and the sampled row is logged at out_log[*step_counter * batch + b]
 * (idle rows log -1); *step_counter is then incremented. */
int tl_decode_advance(int32_t *tokens, const int32_t *next_tokens, int32_t *offsets, int32_t *context_lens,
                      int32_t *out_log, int32_t *step_counter, int batch, int log_capacity, void *stream);

/* Prompt-lookup proposals (DESIGN.md section 14).  history (int32, device, `capacity` entries) holds s[0..length);
 * the call first appends the n_appended (0..TL_NGRAM_MAX_APPEND) ids at `appended` (HOST memory: they travel as
 * kernel arguments, no copy) so that s = s[0..L), L = length + n_appended <= capacity, then searches it:
 *   c(e), e in [0, L-2]: the largest t <= min(n_max, e + 1) with s[e-t+1..e] == s[L-t..L-1] (0 if s[e] != s[L-1]);
 *   e* maximises (c(e), e) over the e with c(e) >= n_min (the longest match, then the latest);
 *   p_t = s'[e* + 1 + t], t < k, s' = s followed by p (a continuation past s repeats the matched period).
 * out (int32, device, [2 + k]) receives c(e*), e*, p_0..p_{k-1}; with no match 0, -1 and k times -1.
 * state (int32, device, TL_NGRAM_STATE_WORDS, 8-byte aligned, zeroed once by the caller) carries the cross-CTA
 * reduction, which the call leaves zeroed, and the one-hot rows last written.  onehot (optional, dtype [k, vocab],
 * device, filled with -inf once by the caller, used with one state only): the previous call's rows are cleared to
 * -inf and row t gets 0 at p_t, so it holds exactly the current proposals as point masses (all -inf with no match),
 * in O(k) writes.  1 <= k <= TL_NGRAM_MAX_K, 1 <= n_min <= n_max <= TL_NGRAM_MAX_N, and with onehot
 * 1 <= vocab <= TL_NGRAM_MAX_VOCAB (the vocabularies tl_speculative_sample takes).  grid: the number of CTAs, 0 for
 * ceil((L - 1) / TL_NGRAM_TILE); the outputs do not depend on it.  One launch, no synchronisation: graph-capturable. */
#define TL_NGRAM_MAX_K 7
#define TL_NGRAM_MAX_N 8
#define TL_NGRAM_MAX_APPEND 8
#define TL_NGRAM_TILE 1024
#define TL_NGRAM_STATE_WORDS 12
#define TL_NGRAM_MAX_VOCAB TL_SPECULATIVE_SAMPLE_MAX_VOCAB
int tl_ngram_propose(int32_t *history, int capacity, int length, const int32_t *appended, int n_appended, int k, int n_min,
                     int n_max, int32_t *out, int32_t *state, void *onehot, int vocab, int dtype, int grid, void *stream);

/* Beam search's cross-beam selection (DESIGN.md section 15).  top_lp (float32) and top_ids (int32), device, [rows, n],
 * are tl_logprobs' top-n lists of `rows` logits rows, n = num_beams + num_eos; cum (float32, device, num_beams
 * entries) holds the rows' cumulative log-probabilities.  Candidate (r, k) scores s = fl(cum[r] + top_lp[r, k]); one
 * with id -1, or whose s is -inf or NaN, is never taken.  The takeable candidates are walked in the order (s
 * descending, r ascending, k ascending), p their position: an EOS id (eos_ids, HOST memory, passed by value) at
 * p < num_beams finishes a hypothesis, one at p >= num_beams is skipped, and any other id becomes a live beam while
 * fewer than num_beams are live.  result (int32, device, TL_BEAM_RESULT_WORDS) receives
 *   [0] live count, [1] finished count,
 *   [2 + j], [10 + j], [18 + j]: live beam j's parent row, token and new cum (float32 bits), in walk order,
 *   [26 + f], [34 + f], [42 + f], [50 + f]: finished f's parent row, EOS id, sum (float32 bits) and walk position.
 * cum is rewritten in place after every input is read: [0, live) the live beams' sums, [live, num_beams) -inf (an
 * idle row of a later step is then never taken).  1 <= num_beams <= TL_BEAM_MAX_WIDTH, 1 <= rows <= num_beams,
 * 0 <= num_eos <= TL_BEAM_MAX_EOS distinct non-negative ids, n == num_beams + num_eos.  One launch, no
 * synchronisation: graph-capturable. */
#define TL_BEAM_MAX_WIDTH 8
#define TL_BEAM_MAX_EOS 4
#define TL_BEAM_MAX_N (TL_BEAM_MAX_WIDTH + TL_BEAM_MAX_EOS)
#define TL_BEAM_RESULT_WORDS (2 + 7 * TL_BEAM_MAX_WIDTH)
int tl_beam_select(const float *top_lp, const int32_t *top_ids, float *cum, int rows, int n, int num_beams, const int32_t *eos_ids,
                   int num_eos, int32_t *result, void *stream);

/* Logits controls (DESIGN.md section 22): logit_bias, allowed_token_ids, bad_words_ids and min_tokens of a request.
 * One descriptor per row, in device memory (48 bytes):
 *   data        the row's packed int32 words (NULL with flags 0):
 *                 data[bias_off + j], j < num_bias: a biased token id; data[bias_off + num_bias + j]: its bias (f32 bits);
 *                 data[bad_off + TL_CONTROL_BAD_WORD_WORDS * s]: length L (1..16) of banned sequence s, then its L ids;
 *                 data[eos_off + j], j < num_eos: the EOS ids min_tokens holds back;
 *                 data[allow_off ..]: ceil(vocab / 32) words, bit t set iff token t is allowed (flags & TL_CONTROL_ALLOW);
 *   flags       TL_CONTROL_ON for a controlled row (0: the row is copied and its tail left alone), | TL_CONTROL_ALLOW;
 *   prompt_len  the request's prompt length; the generated count at a launch is positions[r] - prompt_len;
 *   min_tokens  while the generated count is below it, the EOS ids are banned. */
#define TL_CONTROL_ON 1
#define TL_CONTROL_ALLOW 2
#define TL_CONTROL_MAX_BIAS 1024
#define TL_CONTROL_MAX_BAD_WORDS 64
#define TL_CONTROL_MAX_BAD_WORD_LEN 16
#define TL_CONTROL_BAD_WORD_WORDS (1 + TL_CONTROL_MAX_BAD_WORD_LEN)
#define TL_CONTROL_MAX_EOS 8
#define TL_CONTROL_TAIL (TL_CONTROL_MAX_BAD_WORD_LEN - 1)
typedef struct tl_control_row {
    const int32_t *data;
    int32_t flags;
    int32_t prompt_len;
    int32_t min_tokens;
    int32_t num_bias;
    int32_t bias_off;
    int32_t num_bad;
    int32_t bad_off;
    int32_t num_eos;
    int32_t eos_off;
    int32_t allow_off;
} tl_control_row;
/* The controlled rows y (fp32 [rows, vocab]) of logits [rows, vocab] (fp32, fp16 or bf16; rows <= 65535), one launch,
 * one cluster of CTAs per row, each CTA owning a slice of the row:
 *   y_i = float(x_i), or -inf where the allow mask clears bit i;
 *   then y_i = fl32(y_i + b_i) for every biased id (one IEEE round-to-nearest add: NaN stays NaN, -inf stays -inf);
 *   then y_i = -inf for the last id of every banned sequence whose other L - 1 ids equal the row's last L - 1 tokens,
 *   and for the EOS ids while positions[r] - prompt_len < min_tokens.
 * tails (int32 [rows, TL_CONTROL_TAIL], read and written) holds each controlled row's most recent tokens before this
 * step's input token, oldest first, -1 where the history is shorter.  For controlled rows with positions[r] > 0 the
 * launch appends tokens[r] (the step's input token: the previously drawn one, or the prompt's last token at the first
 * draw) before matching and writes the new tail back; rows at position 0 (idle slots, capture warm-ups) match on the
 * tail as it is and leave it alone.  Uncontrolled rows are copied exactly.  No atomics, no workspace, no host
 * synchronisation; a row's y does not depend on its index or on the row count.  Out-of-range ids in data are ignored. */
int tl_logit_controls(const void *logits, const tl_control_row *controls, const int32_t *positions, const int32_t *tokens,
                      int32_t *tails, float *out, int rows, int vocab, int dtype, void *stream);

/* DRY, "don't repeat yourself" (DESIGN.md section 24).  One descriptor per row, in device memory (528 bytes):
 *   flags           TL_DRY_ON for a DRY row (0: the row is left alone);
 *   allowed_length  a >= 1, the longest repeat that goes unpenalised;
 *   last_n          N: the window is h_lo .. h_{n-1}, lo = 0 for N = 0, else max(0, n - N);
 *   num_breakers    the count of ids in breakers (sorted ascending, at most TL_DRY_MAX_BREAKERS);
 *   penalty         P[k] = fl32(m b^k) for k = 0 .. TL_DRY_MAX_MATCH - a, computed in double by the host.
 * TL_DRY_MAX_MATCH caps the match length: at b = 1.75 and m = 1 the penalty passes 10^15 at k = 62 already, so a
 * longer match changes nothing a sampler could see; the cap bounds a match's reads at 64 ids per end. */
#define TL_DRY_ON 1
#define TL_DRY_MAX_MATCH 64
#define TL_DRY_MAX_BREAKERS 64
typedef struct tl_dry_row {
    int32_t flags;
    int32_t allowed_length;
    int32_t last_n;
    int32_t num_breakers;
    int32_t breakers[TL_DRY_MAX_BREAKERS];
    float penalty[TL_DRY_MAX_MATCH];
} tl_dry_row;
/* The DRY penalty on the fp32 rows x [rows, vocab] (in place; tl_logit_controls' output), one launch, one cluster of
 * CTAs per row splitting the row's history ends.  For a DRY row with 1 <= n = positions[r] <= capacity the history is
 * h_0 .. h_{n-2} = history[r, 0 .. n-2] and h_{n-1} = tokens[r] (the step's input token).  Unless h_{n-1} is a breaker,
 * for every end lo <= e <= n - 2 whose next id t = h_{e+1} is not a breaker, l(e) is the largest l <= TL_DRY_MAX_MATCH
 * with e - i >= lo, h_{e-i} = h_{n-1-i} and h_{n-1-i} not a breaker for every i < l; l*(t) the maximum over the ends
 * followed by t.  Every t with l*(t) >= a becomes fl32(x_t - P[l*(t) - a]), or -inf when that P is +inf (NaN stays).
 * The launch then writes history[r, n - 1] = tokens[r].  Rows at position 0 (idle slots, capture warm-ups), rows past
 * capacity and rows with flags 0 are left alone.  scratch (fp32 [rows, capacity]) holds each end's candidate between
 * the read and the write phases; every candidate is computed from the unpenalised row and the row keeps the least of
 * them, so the result is deterministic.  No host synchronisation. */
int tl_dry_penalty(float *x, const tl_dry_row *dry, const int32_t *positions, const int32_t *tokens, int32_t *history, float *scratch,
                   int rows, int vocab, int capacity, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* TINY_LLM_B200_H */
