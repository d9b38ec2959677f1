/* sr_b200_testhooks.h -- hooks for the parity tests and profiling tools.  NOT exported by the product libraries
 * (lib/libcandle_semantic_router.so, lib/libonnx_semantic_router.so): the same objects plus these entry points are linked
 * into lib/lib{candle,onnx}_semantic_router_testhooks.so (built with -DSRB_TEST_HOOKS), which only tests/ and tools/ load.
 */
#ifndef SR_B200_TESTHOOKS_H
#define SR_B200_TESTHOOKS_H
#include <stddef.h>
#include "sr_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* ---- host-logic test hooks (no GPU): the span logic the text ABI runs after the token classifiers ------------ */
/* BIO decoding of per-token predictions (offsets [n,2] = byte spans, (0,0) = special token).  In
 * libcandle_semantic_router: traditional/modernbert.rs:1478-1567; in libonnx_semantic_router:
 * mmbert_classifier.rs:952-1050 (other I- handling, spans clipped at text_len).  labels[i] = name of class i.
 * Writes up to cap entities and their types as "TYPE\n..." into types_out; returns the entity count. */
SR_API int sr_test_bio_decode(const int32_t* pred, const float* conf, const int32_t* offsets, int n, const char* const* labels,
                       int n_labels, int text_len, int32_t* ent_start, int32_t* ent_end, float* ent_conf, char* types_out,
                       int types_cap, int cap);
/* detect_hallucinations after the token classifier (ffi/classify.rs:1536-1660); -1 in the ONNX library. */
SR_API int sr_test_hallucination_spans(const int32_t* pred, const float* conf, const int32_t* offsets, int n, int answer_start,
                                int answer_len, float threshold, int32_t* span_start, int32_t* span_end, float* span_conf,
                                int cap, int* has_hallucination, float* overall_confidence);

/* ---- unit-op hooks for the parity tests (device pointers, legacy default stream) --------------------- */
SR_API int sr_test_gemm(const void* a_f16, const void* w_f16, void* out, int m, int n, int k, int epi, int ldo,
                 const float* bias, const float* resid, const int32_t* pos, const float* rope_cos,
                 const float* rope_sin, int rope_cols);
/* EPI_RESID_HL (gemm.h): the residual stream as an fp16 pair, in place.  (hi + lo) holds x - pivot_in; after the call it holds
 * x + a w^T (+bias) - pivot_out with pivot_out = pivot_in + (row mean of the old pair, from pivot_in_stats; 0 without), and
 * row_stats [n/128][m][2] the (sum, sum of squares) partials of the new pair. */
SR_API int sr_test_gemm_resid_hl(const void* a_f16, const void* w_f16, void* hi_f16, void* lo_f16, int m, int n, int k,
                                 const float* bias, float* row_stats, float* pivot_out, const float* pivot_in,
                                 const float* pivot_in_stats);
/* The thread-block cluster the GEMM launches for (epilogue, N, K): cluster_n CTAs on neighbouring column tiles of one row
 * block share each A k-block (1: no clusters); workers = clusters of its persistent grid on this device (null: only
 * cluster_n, which needs no device). */
SR_API int sr_test_gemm_cluster(int epi, int n, int k, int* cluster_n, int* workers);
/* Every field of the GEMM descriptor (csrc/gemm.h GemmDesc, same names and meaning; epi = GemmEpilogue value).  Zeroed
 * fields take GemmDesc's defaults.  EPI_ROPE / EPI_GEGLU with fold_stats (weights: W diag(gamma) with zero-sum rows)
 * scale the accumulator rows by the rstd computed from fold_stats over rows of length fold_h; the EPI_RESID_HL fields
 * mean what they mean for sr_test_gemm_resid_hl (out = hi).  bias_per_group (with w_groups > 1): bias holds w_groups
 * vectors of n, and rows of group g add bias[g * n, (g + 1) * n). */
typedef struct sr_gemm_desc {
  int m, n, k;
  const void* a;
  int a_rows;
  const void* w;
  void* out;
  int ldo;
  int epi;
  const float* bias;
  const float* resid;
  int ldr;
  const int32_t* pos;
  const float* rope_cos;
  const float* rope_sin;
  int rope_cols;
  int32_t* topk_idx;
  float* topk_score;
  const uint8_t* topk_valid;
  int topk_n;
  float* row_stats;
  void* lo16;
  float* pivot_out;
  const float* pivot_in;
  const float* pivot_in_stats;
  const float* fold_stats;
  float fold_eps;
  int fold_h;
  int w_groups, w_group_rows;
  int bias_per_group;
} sr_gemm_desc;
/* gemm_f16 on the legacy default stream with every descriptor field; EPI_TOPK's list count goes to *topk_lists. */
SR_API int sr_test_gemm_desc(const sr_gemm_desc* d, int* topk_lists);
/* The route sr_cache_topk takes for b queries over n stored rows of dimension dim (csrc/kernels.h cache_topk_plan):
 * route 0 the empty store, 1 the GEMM's fused top-8 epilogue, 2 GEMV scores + two-stage selection, 3 GEMM scores +
 * two-stage selection; chunks = score chunks of the two-stage routes (0 otherwise); candidates = stage-2 candidates per
 * query (fused: the upper bound).  Returns -1 (route -1) wherever sr_cache_topk refuses the shape. */
SR_API int sr_test_cache_plan(int b, int n, int dim, int k, int* route, int* chunks, int* candidates);
/* The last scan of an exact cache (sr_cache_create_exact) over b queries, per query: path 0 when its band of possible
 * winners was certified inside the candidates of the fp16 scan, 1 when it fell back to the exhaustive exact scan, 2 when
 * the device refused it (a component out of range; band and eps 0); band = the candidates at or above s16_(k) - 2 eps (for
 * a fallback query: all of them); eps = the bound on |fp16-operand score - Go score| (csrc/cache_scan.cu exact_eps).
 * candidates = k' of that scan, fallback = its fallback queries, read from the device at this call (either may be null).
 * After a device-resident scan, call it once the scan's stream has reached its results.  -1 for a cache that is not exact
 * or whose last scan had another b. */
SR_API int sr_test_cache_exact_stats(sr_cache* c, int b, int32_t* path, int32_t* band, double* eps, int* candidates,
                                     int* fallback);
SR_API int sr_test_hl_to_f32(const void* hi_f16, const void* lo_f16, const float* pivot, int t, int hdim, float* x);
/* attention_wgmma_fwd (csrc/kernels.h: same arguments and meaning; window 0 = global, kv_lens [batch] or null) */
SR_API int sr_test_attention_wgmma(const void* qkv_f16, void* out_f16, const int32_t* cu_seqlens, int batch, int max_len,
                                   int num_heads, int head_dim, int window, const int32_t* kv_lens);
/* ---- the precise path's row kernels (csrc/precise.cu), one hook per launcher (csrc/engine.h: same arguments and meaning) */
/* x [t, h] fp32 -> out [t, 3h] fp16 rows [hi | lo | hi]; gamma non-null: the no-bias LayerNorm with eps first */
SR_API int sr_test_precise_split(const float* x, int t, int h, const float* gamma, float eps, void* out_f16);
/* rotate-half RoPE in place on the q and k thirds of qkv [t, 3 * heads * 64] fp32 with the [*, 32] tables at pos[t] */
SR_API int sr_test_precise_rope(float* qkv, const int32_t* pos, int t, int heads, const float* cos_t, const float* sin_t);
/* out [t, i] = gelu_erf(a) * b, ab [t, 2i] fp32 */
SR_API int sr_test_precise_geglu(const float* ab, int t, int i, float* out);
/* fp32 attention over packed qkv [T, 3 * heads * 64] -> out [T, heads * 64]; window 0 = global */
SR_API int sr_test_precise_attention(const float* qkv, float* out, const int32_t* cu_seqlens, int batch, int max_len,
                                     int heads, int window);
/* the same over heads of head_dim 32 or 64 (qkv [T, 3 * heads * head_dim] -> out [T, heads * head_dim], scores scaled by
 * head_dim^-1/2); kv_lens [batch] or null (global attention only): keys >= kv_lens[b] are masked for every query row of
 * sequence b, and every row stays a query */
SR_API int sr_test_precise_attention_kv(const float* qkv, float* out, const int32_t* cu_seqlens, int batch, int max_len,
                                        int heads, int head_dim, int window, const int32_t* kv_lens);
/* x = gelu_erf(x) in place over fp32 [t, i] */
SR_API int sr_test_precise_gelu(float* x, int t, int i);
SR_API int sr_test_layernorm(const float* x, int t, int h, const float* w, const float* b, float eps, float* y32,
                      void* y16);

/* ---- the row kernels of csrc/elementwise.cu, one hook per launcher (csrc/kernels.h: same arguments and meaning) -- */
SR_API int sr_test_embed_ln_modernbert(const int32_t* ids, int t, int h, int vocab, const float* table, const float* ln_w,
                                       float eps, float* x, void* h16, void* lo16);
SR_API int sr_test_embed_ln_bert(const int32_t* ids, const int32_t* pos, int t, int h, int vocab, int max_pos,
                                 const float* word, const float* pos_emb, const float* type0, const float* ln_w,
                                 const float* ln_b, float eps, float* x, void* h16);
SR_API int sr_test_positions(const int32_t* cu_seqlens, int batch, int32_t* pos);
SR_API int sr_test_cast_f16(const float* x, size_t n, void* y16);
/* mode: 0 mean, 1 first token; part [batch, 8, h] and arrived [batch] (zero on entry) are the caller's scratch */
SR_API int sr_test_pool_rows(const float* x, const int32_t* cu_seqlens, int batch, int h, int mode, const float* ln_w,
                             const float* ln_b, float eps, float* pooled, float* part, int32_t* arrived,
                             const int32_t* div_lens);
SR_API int sr_test_l2_normalize(const float* pooled, int batch, int h, int dim, float norm_eps, float* emb);
/* Every field of the sequence-head weights (csrc/kernels.h SeqHeadWeights, same names and meaning). */
typedef struct sr_seq_head_weights {
  const float* dense_w;
  const float* dense_b;
  const float* norm_w;
  int dense_mode;
  const float* cls_w;
  const float* cls_b;
  int num_classes;
  int argmax_last;
  int gelu_erf;
  float head_eps;
} sr_seq_head_weights;
SR_API int sr_test_seq_head(const float* pooled, int batch, int h, const sr_seq_head_weights* w, float* logits,
                            float* probs, int32_t* cls, float* conf);
SR_API int sr_test_token_head(const float* hidden32, const void* dense16, int t, int h, const float* norm_w,
                              const float* pre_ln_w, float pre_ln_eps, const float* cls_w, const float* cls_b, int c,
                              int argmax_last, float* logits, float* probs, int32_t* pred, float* conf, int gelu_erf,
                              float head_eps);

#ifdef __cplusplus
}
#endif
#endif
