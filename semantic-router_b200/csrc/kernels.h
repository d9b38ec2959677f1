// Host-callable launchers of the HBM-bound kernels (elementwise.cu), attention (attention_wgmma.cu) and the
// cache scan (cache_scan.cu).  All pointers are device pointers; all launches are asynchronous on `stream`.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace srb {

// kernel-launch accounting (engine.cu): every launcher below bumps it; bench.py reports it as gpu_launches
void note_launch(int n = 1);
// SRB_PDL=1 turns programmatic dependent launch on for the GEMM kernels (default off)
bool pdl_enabled();
long long launches_total();
// SMs of the current device (gemm_wgmma.cu), asked once: the devices of one process are taken to be alike.  -1 when
// the runtime cannot tell.
int device_sms();

// Sequences one attention launch takes: they sit in gridDim.z, whose limit is 65 535; the attention launchers (here and in
// precise.cu) run larger packs as slices of at most this many sequences.
constexpr int kMaxGridZ = 65535;

// ---- attention_wgmma.cu (wgmma flash attention, head dim 64, optional sliding window |i - j| <= window; every layer)
// kv_lens [batch] (optional, global attention only): keys >= kv_lens[b] of sequence b are masked for EVERY query row while
// all rows stay queries -- right-padded sequences whose pads are queries, as candle's BertModel sees them under a
// fixed-padding tokenizer (core/similarity.rs:189-222)
int attention_wgmma_fwd(cudaStream_t stream, const __half* qkv, __half* out, const int* cu_seqlens, int batch,
                        int max_len, int num_heads, int head_dim, int window, const int* kv_lens = nullptr);

// ---- elementwise.cu
// Per-row parameters of a grouped pass (engine.h: Grouped): rows [g * rows, (g + 1) * rows) read p[g]; rows == 0: every
// row reads p[0].  A tensor every group shares is the same pointer in every slot.  Passed by value to the kernels.
constexpr int kMaxRowGroups = 8;
struct RowGroups {
  const float* p[kMaxRowGroups] = {};
  static RowGroups one(const float* q) { RowGroups r; r.p[0] = q; return r; }
};

// pos[t] = t - cu_seqlens[seq(t)]
int compute_positions(cudaStream_t stream, const int* cu_seqlens, int batch, int* pos);
// ModernBERT embeddings: x = LN_nobias(E[ids]); writes fp32 residual stream and its fp16 copy.
// lo (optional): fp16(x - fp16(x)), the low half of the fp16-pair form of the residual stream; x may be null then
int embed_ln_modernbert(cudaStream_t stream, const int* ids, int T, int H, int vocab, const float* table,
                        const float* ln_w, float eps, float* x, __half* h, __half* lo = nullptr);
// the same with the table and LayerNorm weight of row r's group (group_rows > 0: g = r / group_rows)
int embed_ln_modernbert(cudaStream_t stream, const int* ids, int T, int H, int vocab, const RowGroups& table,
                        const RowGroups& ln_w, int group_rows, float eps, float* x, __half* h, __half* lo);
// x[r, :] = pivot[r] + hi[r, :] + lo[r, :]  (pivot null: 0)
int hl_to_f32(cudaStream_t stream, const __half* hi, const __half* lo, const float* pivot, int T, int H, float* x);
// BERT embeddings: x = LN(word[id] + pos[p] + type[0]).
int embed_ln_bert(cudaStream_t stream, const int* ids, const int* pos, int T, int H, int vocab, int max_pos,
                  const float* word, const float* pos_emb, const float* type0, const float* ln_w,
                  const float* ln_b, float eps, float* x, __half* h);
int embed_ln_bert(cudaStream_t stream, const int* ids, const int* pos, int T, int H, int vocab, int max_pos,
                  const RowGroups& word, const RowGroups& pos_emb, const RowGroups& type0, const RowGroups& ln_w,
                  const RowGroups& ln_b, int group_rows, float eps, float* x, __half* h);
// Row LayerNorm of fp32 x[T,H]; optional outputs: y32 (may alias x) and y16.
int layernorm_rows(cudaStream_t stream, const float* x, int T, int H, const float* w, const float* b, float eps,
                   float* y32, __half* y16);
// the same with the weight and bias (null slots: no bias) of row r's group
int layernorm_rows(cudaStream_t stream, const float* x, int T, int H, const RowGroups& w, const RowGroups& b,
                   int group_rows, float eps, float* y32, __half* y16);
// fp32 -> fp16 copy of n elements, any n (x 16-byte and y 8-byte aligned)
int cast_rows_f16(cudaStream_t stream, const float* x, size_t n, __half* y);

enum PoolMode { POOL_MEAN = 0, POOL_CLS = 1 };
// pooled[b,:] = mean_t / first-token of (optionally LayerNorm'ed) x rows of sequence b.
// `part` [batch, kPoolParts, H] and `arrived` [batch] (zero on entry, zero again on exit) are scratch.
constexpr int kPoolParts = 8;
int pool_rows(cudaStream_t stream, const float* x, const int* cu_seqlens, int batch, int H, PoolMode mode,
              const float* ln_w, const float* ln_b, float eps, float* pooled, float* part, int* arrived,
              const int* div_lens = nullptr);   // div_lens [batch]: divide the sums by these instead of the row counts
// emb[b, :dim] = pooled[b, :dim] / (||pooled[b,:dim]||_2 + norm_eps)
int l2_normalize_rows(cudaStream_t stream, const float* pooled, int batch, int H, int dim, float norm_eps,
                      float* emb);

struct SeqHeadWeights {
  // ModernBERT: dense [H,H] (no bias) -> gelu_tanh -> LN(norm_w, 0, 1e-12); BERT: pooler [H,H]+bias -> tanh
  const float* dense_w = nullptr;
  const float* dense_b = nullptr;
  const float* norm_w = nullptr;
  int dense_mode = 0;  // 0 none, 1 ModernBERT head, 2 BERT pooler y = x @ P^T (+b), 3 BERT pooler y = x @ P (+b)
  const float* cls_w = nullptr;  // [C,H]
  const float* cls_b = nullptr;  // [C]
  int num_classes = 0;
  int argmax_last = 0;  // 0: first max wins (strict > from 0.0), 1: last max wins (max_by)
  // HF/ONNX-export flavour of the ModernBERT head (onnx-binding twin): erf GELU and eps = config.norm_eps
  int gelu_erf = 0;
  float head_eps = 1e-12f;
};
// logits/probs [B,C], cls int32 [B], conf fp32 [B]
int seq_head(cudaStream_t stream, const float* pooled, int batch, int H, const SeqHeadWeights& w, float* logits,
             float* probs, int* cls, float* conf);

// Token head tail: (optional: gelu_tanh + LN(norm_w, 0, 1e-12) of the fp16 dense output) -> classifier ->
// logits/probs [T,C], pred int32 [T] (argmax over logits; first max unless argmax_last), conf [T].
// hidden32 path: optional LayerNorm(pre_ln_w, no bias, pre_ln_eps) first (ModernBERT final_norm).
int token_head(cudaStream_t stream, const float* hidden32, const __half* dense16, int T, int H,
               const float* norm_w, const float* pre_ln_w, float pre_ln_eps, const float* cls_w,
               const float* cls_b, int C, int argmax_last, float* logits, float* probs, int* pred, float* conf,
               int gelu_erf = 0, float head_eps = 1e-12f);

// ---- cache_scan.cu
// The route cache_topk takes for (B queries, N stored rows, dimension D, k): the empty store; the GEMM's fused top-8
// epilogue (B > 4, k <= 8); or scores in chunks of at most 1 GiB followed by the two-stage selection, the scores coming
// from a GEMV (B <= 4 and B * D * 4 <= 48 KB) or from the GEMM.  Refused (route CACHE_REFUSED): B or k <= 0, k > 64,
// or more than 200 KB of stage-2 candidates (ceil(N / 8192) * k > 25600).
enum CacheRoute { CACHE_REFUSED = -1, CACHE_EMPTY = 0, CACHE_FUSED = 1, CACHE_GEMV = 2, CACHE_GEMM = 3 };
struct CachePlan {
  int route = CACHE_REFUSED;
  int chunk_rows = 0;          // two-pass: stored rows per score chunk, a multiple of the 8192-row stage-1 segment
  int chunks = 0;              // two-pass: score chunks (one score GEMV / GEMM and one stage-1 launch each)
  int segments = 0;            // two-pass: stage-1 segments over the whole store, ceil(N / 8192)
  int candidates = 0;          // stage-2 candidates per query (fused: the upper bound, 8 per list)
  size_t stage2_smem = 0;      // two-pass: dynamic shared memory of stage 2, candidates x 8 bytes
  size_t workspace_bytes = 0;  // what cache_topk needs for this route
};
CachePlan cache_topk_plan(int B, int N, int D, int k);
// scores = Q[B,D] . C[N,D]^T (fp16 operands, fp32 accumulate); per query top-k (descending score, lower
// index wins ties); rows with valid[i]==0 are skipped.  out_idx int32 [B,k] (global id = row + id_offset,
// -1 when fewer than k valid rows), out_score fp32 [B,k].  Returns -1 where cache_topk_plan refuses.
int cache_topk(cudaStream_t stream, const __half* queries, int B, const __half* cache, const uint8_t* valid,
               int N, int D, int k, int id_offset, int* out_idx, float* out_score, void* workspace,
               size_t workspace_bytes);
size_t cache_topk_workspace_bytes(int B, int N, int D, int k);

// Exact caches: the same top-k with scores bitwise the reference's sequential fp32 dot product of the fp32 query
// (queries32 [B,D]) and the fp32 rows (cache32 [N,D]), sum_rule 0 (product rounded, then added) or 1 (one fma per term).
// The scan rounds the queries to fp16 into queries16 [B,D] (its own scratch) and the fp16 scan (queries16, cache) picks
// k' candidates per query; queries whose band of possible winners is not certified within them are scanned exhaustively
// in Go order.  A query with a non-finite component or one above 65504 in magnitude is refused on the device: its k
// results are (-1, -inf).  rmax >= every stored row's L2 norm.  path / band / eps [B]: per query 0 certified, 1 fallback
// or 2 refused, the candidates in its band, its bound eps.  Nothing waits on the host: the number of fallback queries
// stays on the device (cache_exact_fallback_count points at it).  Refused (-1) where the two-stage selection at k is
// (ceil(N / 8192) * k > 25600) and for D % 8 != 0.
int cache_exact_candidates(int B, int N, int D, int k);   // k'; 0 where refused
size_t cache_topk_exact_workspace_bytes(int B, int N, int D, int k);
const int* cache_exact_fallback_count(const void* workspace, int B, int N, int D, int k);   // device int; null where refused
int cache_topk_exact(cudaStream_t stream, const float* queries32, __half* queries16, int B, const __half* cache,
                     const float* cache32, const uint8_t* valid, int N, int D, double rmax, int k, int sum_rule,
                     int id_offset, int* out_idx, float* out_score, void* workspace, size_t workspace_bytes, int* path,
                     int* band, double* eps);

// sharded-cache exchange format: 8-byte entries {fp32 score, int32 global id}
int cache_pack_pairs(cudaStream_t stream, const int* idx, const float* score, int n, void* pairs_out);
// merge of G gathered lists in that format, pairs [G][B][k] -> [B,k]; refused (-1) for G * k > 6144
int cache_merge_packed(cudaStream_t stream, const void* pairs, int G, int B, int k, int* out_idx, float* out_score);

}  // namespace srb
