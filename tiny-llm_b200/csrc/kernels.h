// Internal launcher declarations (one translation unit per kernel family);
// c_abi.cu validates arguments and forwards here.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/tiny_llm_b200.h"

namespace tl {

// elementwise.cu
// Kernel selection, shared by the launches and the tl_*_route exports: rms_norm's threads per row (32 | 256, *vec: 16-byte
// accesses) and whether rope runs the per-(token, pair) kernel.  q/k norm: qkv_planes_rope_supported (the row kernel).
int rms_norm_path(int dim, int dtype, const void *x, const void *w, const void *out, bool *vec);
bool rope_heads_path(int B, int L, int H, int D, int dims);
int launch_rms_norm(const void *x, const void *w, void *out, int rows, int dim, float eps, int dtype, cudaStream_t st);
int launch_rope(const void *x, const int32_t *off, void *out, int B, int L, int H, int D, int dims, float base,
                int traditional, int dtype, cudaStream_t st);
int launch_swiglu(const void *gate, const void *up, void *out, long long n, int dtype, cudaStream_t st);
int launch_add(const void *a, const void *b, void *out, long long n, int dtype, cudaStream_t st);
int launch_quantized_embedding(const void *indices, const void *scales, const void *biases, const void *weight,
                               void *out, int tokens, int vocab, int dim, int dtype, cudaStream_t st);
int launch_paged_cache_update(void *pages, const void *values, int heads, int page_size, int head_dim, int length,
                              int page_id, int start, int dtype, cudaStream_t st);
int launch_paged_cache_append_chunk(void *key_pages, void *value_pages, const void *keys, const void *values,
                                    const tl_page_span_list &spans, int heads, int page_size, int head_dim, long long src_head_stride,
                                    long long src_token_stride, int dtype, cudaStream_t st);
int launch_paged_cache_append_decode(void *key_pages, void *value_pages, const void *keys, const void *values,
                                     const int32_t *block_table, const int32_t *context_lens, int batch,
                                     int num_pages, int heads, int page_size, int head_dim, int max_pages, int dtype,
                                     cudaStream_t st);
size_t argmax_workspace(int rows, int vocab);
int launch_argmax(const void *logits, int32_t *out, int rows, int vocab, int dtype, void *ws, size_t ws_bytes,
                  cudaStream_t st);

// sampling.cu: cluster size and fp32 entries per CTA for a row of `vocab` (TL_EINVAL beyond the staging limit)
int sample_plan(int vocab, int *cluster, int *slice);
int launch_sample(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                  const int32_t *positions, int32_t *out, int rows, int vocab, int dtype, cudaStream_t st);
int launch_sample_penalized(const void *logits, const float *temperature, const int32_t *top_k, const float *top_p, const int64_t *seed,
                            const int32_t *positions, const float *repetition, const float *presence, const float *frequency,
                            const float *min_p, int32_t *state, int32_t *out, int rows, int vocab, int dtype, cudaStream_t st);
// logprobs.cu: same cluster plan as sampling.cu
constexpr int LOGPROBS_MAX_N = TL_LOGPROBS_MAX_N;
int launch_logprobs(const void *logits, const int32_t *targets, const int32_t *top_n, const int32_t *out_index, float *lse, float *lp,
                    int32_t *rank, int32_t *top_ids, float *top_lp, int rows, int vocab, int max_n, int out_capacity, int dtype,
                    cudaStream_t st);

int launch_decode_advance(int32_t *tokens, const int32_t *next_tokens, int32_t *offsets, int32_t *context_lens,
                          int32_t *out_log, int32_t *step_counter, int batch, int log_capacity, cudaStream_t st);

int launch_decode_qk_norm_rope_append(const void *qkv, const void *q_norm_w, const void *k_norm_w, const int32_t *offsets,
                                      const int32_t *block_table, const int32_t *context_lens, void *q_out, void *key_pages,
                                      void *value_pages, int batch, int Hq, int Hkv, int D, float base, float eps,
                                      int num_pages, int page_size, int max_pages, int dtype, cudaStream_t st, bool chunk = false);

// w4a16_matvec.cu
// Weight-streaming tensor-core kernel, up to 32 rows per pass (larger M is processed in passes), with optional fused
// prologue (0 none: p0 = a; 1 rms_norm: p0 = x, p1 = norm weight; 2 swiglu: p0 = gate, p1 = up; lda = row stride of
// p0/p1 in elements) and epilogue (0 none; 1 out = residual + result); and the scalar control kernel.
int launch_w4a16_fused(const void *scales, const void *biases, const void *b, void *out, const void *p0, const void *p1,
                       const void *residual, int M, int N, int K, int lda, int prologue, int epilogue, float eps, int dtype,
                       cudaStream_t st);
void set_use_pdl(bool on);
bool use_pdl();
int launch_w4a16_vanilla(const void *scales, const void *biases, const void *a, const void *b, void *out, int M,
                         int N, int K, int dtype, cudaStream_t st);
// Rows per pass and 128-column groups per unit of the streaming kernel, or TL_EINVAL for operands it cannot take.
int w4a16_stream_plan(int M, int N, int K, int lda, const void *p0, const void *p1, const void *b, const void *scales, const void *biases,
                      int *rows_per_pass, int *units);

// w4a16_skinny.cu (swap-AB wgmma GEMM: split reduction for 9 <= M <= 128, 128-token tiles for prefill)
// Split count of the reduction; *gb_per_split (optional) receives the 128-wide group blocks of each split.
int w4a16_skinny_splits(int M, int N, int K, int *gb_per_split = nullptr);
size_t w4a16_skinny_workspace(int M, int N, int K);
// norm_w / normed (optional, residual epilogue): also write normed = rms_norm(out, norm_w, norm_eps); *norm_done tells
// whether the launch did it (split reduction, K <= 4096) or the caller still has to run rms_norm
int launch_w4a16_skinny(const void *scales, const void *biases, const void *a, const void *b, void *out, const void *residual, int M, int N,
                        int K, int epilogue, int dtype, void *ws, size_t ws_bytes, cudaStream_t st, const void *norm_w = nullptr,
                        float norm_eps = 0.f, void *normed = nullptr, bool *norm_done = nullptr, int *planes_out = nullptr);
// planes_out (optional): with a split reduction the launch stops after the GEMM (partial planes [splits][M][K] fp32 in the
// workspace, *planes_out = splits) and the caller's fused kernel adds them; *planes_out = 1 means `out` is complete
int launch_w4a16_tiles(const void *scales, const void *biases, const void *a, const void *b, void *out, int M, int N, int K, int dtype,
                       cudaStream_t st);
// Grouped expert GEMM over expert-sorted rows (MoE; tl_moe_grouped_matmul): K % 128 == 0, splits == 1
int launch_w4a16_grouped(const void *scales, const void *biases, const void *a, const void *b, void *out, const int32_t *offsets, const int32_t *tiles,
                         const int32_t *out_index, int R, int E, int N, int K, int epilogue, int nt, int max_tiles, int dtype, cudaStream_t st);
bool qkv_planes_rope_supported(int Hq, int Hkv, int D, int dtype);
int launch_qkv_planes_rope_append(const float *part, int splits, const void *q_norm_w, const void *k_norm_w, const int32_t *offsets,
                                  const int32_t *block_table, const int32_t *context_lens, void *q_out, void *key_pages, void *value_pages, int batch,
                                  int Hq, int Hkv, float base, float eps, int num_pages, int page_size, int max_pages, cudaStream_t st, bool chunk);

// moe.cu (Qwen3-MoE routing, grouping, gather, combine and the grouped control kernel)
int launch_moe_topk(const void *logits, void *probs, int32_t *ids, void *scores, int rows, int E, int k, int norm, int dtype, cudaStream_t st);
int launch_moe_group(const int32_t *ids, int R, int E, int nt, int32_t *offsets, int32_t *perm, int32_t *tiles, cudaStream_t st);
int launch_moe_gather(const void *x, const int32_t *perm, const void *norm_w, float eps, void *xs, int R, int rows_per_source, int H, int dtype,
                      cudaStream_t st);
int launch_moe_combine(const void *y, const void *scores, const void *residual, const void *norm_w, float eps, void *out, void *normed, int T,
                       int k, int H, int dtype, cudaStream_t st);
int launch_moe_grouped_vanilla(const void *scales, const void *biases, const void *a, const void *b, void *out, const int32_t *offsets,
                               const int32_t *out_index, int R, int E, int N, int K, int epilogue, int dtype, cudaStream_t st);

// decode_attention_fused.cu
#if defined(TL_TRACE) && TL_TRACE
void trace_bind_matvec(unsigned long long *buf, unsigned int *n, unsigned int cap);
void trace_bind_attention(unsigned long long *buf, unsigned int *n, unsigned int cap);
void trace_bind_skinny(unsigned long long *buf, unsigned int *n, unsigned int cap);
#endif
// batch = requests; each carries rows_per_request (1..8) consecutive query rows (qkv / out / offsets / context_lens
// have batch * rows_per_request rows, the block table has batch rows)
size_t decode_attention_fused_workspace(int batch, int rows_per_request, int num_heads, int num_kv_heads);
int launch_decode_attention_fused(const void *qkv, const void *q_norm_weight, const void *k_norm_weight, const int32_t *offsets,
                                  const int32_t *block_table, const int32_t *context_lens, const double *rope_inv_freq,
                                  void *key_pages, void *value_pages, void *out, float *workspace, int batch, int rows_per_request,
                                  int num_heads, int num_kv_heads, int head_dim, float eps, float scale, int num_pages,
                                  int page_size, int max_pages, int max_context, int dtype, cudaStream_t st);

// attention_decode.cu
int launch_decode_attention(const void *q, const void *k, const void *v, const float *mask, void *out, int q_rows,
                            int L, int S, int D, int num_heads, int num_kv_heads, float scale, int is_causal,
                            int has_mask, int dtype, cudaStream_t st);
// Any dtype / head size / page size: one CTA per query row.
int launch_paged_rowwise(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl, void *out, int rows, int L,
                         int D, int num_pages, int page_size, int max_pages, float scale, int is_causal, int num_kv_heads, int num_heads,
                         int dtype, cudaStream_t st);
// bf16, D = 128, 16-byte aligned q / K / V: the CUDA-core GQA-grouped kernel; allow_split cuts the key range into up to
// PAGED_MAX_SPLITS pieces (partials in ws) so that a small batch still fills the GPU.
int launch_paged_gqa(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl, void *out, int rows, int L,
                     int num_pages, int page_size, int max_pages, float scale, int is_causal, int num_kv_heads, int num_heads, bool allow_split,
                     void *ws, size_t ws_bytes, cudaStream_t st);
// Split-KV decode cuts a request's key range into at most this many pieces: the merge kernel then reads the scalars
// of all splits in one load per lane of a warp.  The workspace of tl_paged_attention is sized for it.
constexpr int PAGED_MAX_SPLITS = 32;

// attention_prefill_tc.cu (wgmma + TMA flash prefill; page_size % 64 == 0, Hq/Hkv divides 128)
bool paged_prefill_tc_supported(int L, int num_pages, int page_size, int num_kv_heads, int num_heads);
int launch_paged_prefill_tc(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl, void *out, int rows,
                            int L, int num_pages, int page_size, int max_pages, float scale, int is_causal, int num_kv_heads,
                            int num_heads, bool allow_split, void *ws, size_t ws_bytes, cudaStream_t st, bool out_token_major = false);
int launch_paged_gqa_merge(const float *ws_o, const float *ws_m, const float *ws_l, void *out, int rows_total, int splits, cudaStream_t st);

// attention_prefill.cu (mma.sync flash prefill: fallback for page sizes / head ratios the wgmma kernel does not take)
int launch_paged_prefill_fa(const void *q, const void *kp, const void *vp, const int32_t *bt, const int32_t *cl, void *out, int rows,
                            int L, int num_pages, int page_size, int max_pages, float scale, int is_causal, int num_kv_heads,
                            int num_heads, cudaStream_t st);

}  // namespace tl
