/* sr_b200.h -- additive "side door" C ABI of the H100 (sm_90a) signal-extraction library.
 *
 * NOT part of the reference's Go surface: these entry points take pre-tokenised ids (the reference's text ABI
 * tokenises inside the call, SURVEY.md section 8b "Side-door for measurement") so that parity tests and the
 * throughput harness can drive the encoder without the host tokeniser in the way.  They sit beside the
 * drop-in ABI declared in include/candle_semantic_router.h and share the same engine.
 *
 * Conventions: plain C, no torch types; `ids` / `cu_seqlens` are int32; sequences are packed back to back,
 * cu_seqlens has batch+1 entries (cu[0] = 0, cu[batch] = total tokens).  Return 0 on success, -1 on error
 * (message on stderr and via sr_last_error()).  There is no CPU fallback: loading fails without an sm_90 GPU.
 */
#ifndef SR_B200_H
#define SR_B200_H
#include <stdint.h>
#if defined(__GNUC__)
#define SR_API __attribute__((visibility("default")))
#else
#define SR_API
#endif
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sr_model sr_model;

typedef struct {
  int arch;          /* 0 = ModernBERT/mmBERT, 1 = BERT */
  int hidden, layers, heads, intermediate, vocab, max_pos;
  int num_heads_loaded;   /* classification heads attached to this encoder */
  int device;
} sr_model_info_t;

SR_API const char* sr_last_error(void);
SR_API int sr_device_count(void);

/* Load <dir>/config.json + <dir>/model.safetensors onto CUDA device `device`; a classifier found in the
 * checkpoint becomes head 0.  Replaces init_* of the reference (candle-binding/src/ffi/init.rs:154-877). */
SR_API int sr_model_load(const char* model_dir, int device, sr_model** out);
/* Attach another head (head.*, classifier.*) from a second checkpoint sharing this encoder (BASELINE cfg 3).
 * token_level: 1 token classifier, 0 sequence classifier, -1 from config.json "architectures".  Returns head id. */
SR_API int sr_model_add_head(sr_model* m, const char* model_dir, int token_level);
SR_API void sr_model_free(sr_model* m);
SR_API int sr_model_info(const sr_model* m, sr_model_info_t* out);
SR_API int sr_head_num_classes(const sr_model* m, int head);
/* ModernBERT head semantics.  0 (default): candle (traditional/modernbert.rs:303-329,818,1184-1192 -- MEAN pooling
 * always, tanh GELU, LayerNorm eps 1e-12, first max).  1: the HF graph an ONNX export carries, which onnx-binding
 * runs (mmbert_classifier.rs:796-830 -- pooling per config "classifier_pooling", erf GELU, eps = norm_eps, last max). */
SR_API int sr_model_set_head_flavor(sr_model* m, int flavor);
/* Encoder arithmetic of a ModernBERT / mmBERT model.  0 (default): the production path -- fp16 operands on the tensor cores,
 * fp32 accumulation, residual stream and statistics (logits of the x8-scaled synthetic heads within ~3e-4 RELATIVE of the
 * fp32 reference).  1: the "precise" path -- every GEMM operand as an fp16 hi + lo pair (three wgmma passes in one GEMM of
 * triple depth, fp32-equivalent products), fp32 LayerNorm / RoPE / GeGLU / attention in between: logits and embeddings
 * within the 1e-3 ABSOLUTE bound of BASELINE's north star, at about five times the cost.  Parity mode, not a serving mode.
 * Returns -1 for other architectures. */
SR_API int sr_model_set_precise(sr_model* m, int on);

/* ---- host-buffer entries (synchronous; H2D of ids and D2H of results inside the call) ---------------- */
/* classify_modernbert_text_with_probabilities / classify_candle_bert_text on ids
 * (ffi/classify.rs:757,1023; traditional/modernbert.rs:1125-1203; traditional/bert.rs:222-255).
 * probs/logits [batch, C] (nullable), cls int32 [batch], conf float [batch].
 * pooler_mode (BERT only): 0 = traditional/bert.rs:107 (x @ P), 1 = lora/bert_lora.rs:534 (x @ P^T). */
SR_API int sr_classify_ids(sr_model* m, int head, const int32_t* ids, const int32_t* cu_seqlens, int batch,
                    int pooler_mode, float* probs, float* logits, int32_t* cls, float* conf);
/* classify_modernbert_pii_tokens / classify_candle_bert_tokens on ids (ffi/classify.rs:1355,629):
 * probs/logits [T, C] (nullable), pred int32 [T], conf float [T]. */
SR_API int sr_classify_tokens_ids(sr_model* m, int head, const int32_t* ids, const int32_t* cu_seqlens, int batch,
                           float* probs, float* logits, int32_t* pred, float* conf);
/* get_embedding_2d_matryoshka / get_text_embedding on ids (ffi/embedding.rs:1068, ffi/similarity.rs:12):
 * encoder to target_layer (<=0: all), pool, narrow to target_dim (<=0: hidden), L2 normalise.
 * emb [batch, dim]. */
SR_API int sr_embed_ids(sr_model* m, const int32_t* ids, const int32_t* cu_seqlens, int batch, int target_layer,
                 int target_dim, float* emb);
/* BertSimilarity::get_embedding under a tokenizer.json that carries fixed-length padding (core/similarity.rs:189-222; the
 * sentence-transformers MiniLM checkpoints ship "padding": {"strategy": {"Fixed": 128}}): sequence b holds cu[b+1]-cu[b]
 * positions of which the first real_lens[b] are text and the rest pad tokens.  The pads are masked as KEYS only -- they run
 * through the encoder as queries -- and the pooled vector is the sum over EVERY position divided by the number of real
 * tokens, then L2-normalised without epsilon.  BERT-family models; emb [batch, hidden]. */
SR_API int sr_embed_ids_padded(sr_model* m, const int32_t* ids, const int32_t* cu_seqlens, const int32_t* real_lens, int batch,
                               float* emb);
/* One encoder pass, several heads (BASELINE cfg 3).  For each i < n_heads: sequence heads write
 * probs_out[i] [batch,C_i], cls_out[i] [batch]; token heads write probs_out[i] [T,C_i], cls_out[i] [T]. */
SR_API int sr_classify_multi_ids(sr_model* m, const int* heads, int n_heads, const int32_t* ids,
                          const int32_t* cu_seqlens, int batch, float** probs_out, int32_t** cls_out);

/* ---- shared-base multi-task serving from UNMERGED LoRA checkpoints (SURVEY section 8 f3) ----------------
 * The reference's LoRA path computes x W^T + (alpha / r) (x A^T) B^T per adapted Linear (candle-binding/src/
 * model_architectures/lora/lora_adapter.rs:136-144) and its stated direction is one shared encoder for the intent / PII /
 * security tasks (src/semantic-router/pkg/classification/unified_classifier.go:113).  task_dirs[t] is a complete checkpoint
 * of task t: the SAME base tensors in every directory (checked bit for bit), `X.lora_A.weight` / `X.lora_B.weight` next to
 * the adapted `X.weight`s, its own classifier head, lora_config.json {"rank", "alpha"}.  ONE copy of the base is loaded;
 * a batch then runs ONCE through the encoder as n_tasks copies of its rows, every copy with its own task's rank-r term added
 * inside the projection GEMMs' accumulators (a K extension of the wgmma mainloop), instead of n_tasks forwards over
 * n_tasks merged models.  token_level[t]: 1 token head, 0 sequence head, -1 from config.json.
 * mode SR_LORA_LOWRANK: as described (one copy of the base: the memory form).  mode SR_LORA_GROUPED: every task's adapters are
 * folded into its own copy of the projection weights at load, the copies are stacked, and each 256-row block of a projection
 * GEMM picks its task's matrix in the TMA producer -- still ONE pass over n_tasks copies of the rows, no rank-r GEMMs and no
 * extra k-blocks, the arithmetic of n_tasks separately loaded models (the latency / throughput form). */
enum { SR_LORA_LOWRANK = 0, SR_LORA_GROUPED = 1 };
SR_API int sr_model_load_lora_shared(const char* const* task_dirs, const int* token_level, int n_tasks, int mode, int device,
                                     sr_model** out);
SR_API int sr_lora_shared_mode(const sr_model* m);    /* SR_LORA_LOWRANK / SR_LORA_GROUPED, -1 for an ordinary model */
SR_API int sr_lora_shared_tasks(const sr_model* m);   /* 0 for an ordinary model */
/* 1: <model_dir>/model.safetensors carries lora_A / lora_B tensors, 0: it does not (a merged checkpoint), -1: unreadable */
SR_API int sr_checkpoint_has_adapters(const char* model_dir);
/* For each task t: sequence heads write probs_out[t] [batch, C_t], cls_out[t] / conf_out[t] [batch]; token heads write
 * probs_out[t] [T, C_t], cls_out[t] / conf_out[t] [T] (T = cu_seqlens[batch]).  Any of the pointers may be NULL. */
SR_API int sr_classify_lora_shared_ids(sr_model* m, const int32_t* ids, const int32_t* cu_seqlens, int batch, int pooler_mode,
                                       float** probs_out, int32_t** cls_out, float** conf_out);

/* ---- device-resident entries (asynchronous on the model's stream; for kernel-only timing) ------------- */
SR_API int sr_model_set_stream(sr_model* m, void* cuda_stream);   /* cudaStream_t; NULL restores the private stream */
SR_API int sr_reserve(sr_model* m, int total_tokens, int batch, int max_classes_rows);
SR_API int sr_forward_dev(sr_model* m, const int32_t* d_ids, const int32_t* d_cu_seqlens, int batch, int total_tokens,
                   int max_len, int num_layers);
SR_API int sr_head_seq_dev(sr_model* m, int head, const int32_t* d_cu_seqlens, int batch, int pooler_mode);
SR_API int sr_head_tokens_dev(sr_model* m, int head, int batch, int total_tokens);
SR_API int sr_head_embed_dev(sr_model* m, const int32_t* d_cu_seqlens, int batch, int dim);
SR_API int sr_sync(sr_model* m);
/* Per-category device timing for the roofline report.  Categories: 0 embed, 1 norm/cast, 2 gemm Wqkv,
 * 3 attention, 4 gemm attn-out, 5 gemm MLP-in (GeGLU/GELU), 6 gemm MLP-out, 7 heads.  sr_profile_read
 * synchronises, returns accumulated milliseconds and launch counts since sr_profile_enable(m, 1). */
SR_API int sr_profile_enable(sr_model* m, int on);
SR_API int sr_profile_read(sr_model* m, float* ms8, int* count8);
/* total kernels launched by this library in this process (all models/caches) */
SR_API long long sr_launch_count(void);
/* device pointers of the last results (valid until the next call) */
SR_API const float* sr_dev_probs(const sr_model* m);
SR_API const float* sr_dev_logits(const sr_model* m);
SR_API const int32_t* sr_dev_cls(const sr_model* m);
SR_API const float* sr_dev_conf(const sr_model* m);
SR_API const float* sr_dev_emb(const sr_model* m);
SR_API const float* sr_dev_hidden(const sr_model* m);   /* fp32 residual stream [T, hidden] after the last forward */

/* ---- semantic cache (cosine top-k over device-resident fp16 unit vectors) ---------------------------- */
typedef struct sr_cache sr_cache;
/* capacity rows of dimension dim on `device`; id_offset = global id of local row 0 (sharded caches). */
SR_API int sr_cache_create(int device, int capacity, int dim, int id_offset, sr_cache** out);
SR_API void sr_cache_free(sr_cache* c);
/* Append n rows (float32 host, rounded to fp16 on upload); returns first local row index or -1. */
SR_API int sr_cache_add(sr_cache* c, const float* rows, int n);
SR_API int sr_cache_invalidate(sr_cache* c, int local_row);   /* expired / evicted entry: skipped by the scan */
/* Lifecycle mirror of the reference's entries slice (device row i == entries[i]; pkg/cache/inmemory_cache_lifecycle.go):
 * set_valid: pending entry completed / entry expired (0 = skipped by the scan, as ResponseBody == nil / isExpired are);
 * move: evictOne's "swap with the last entry" (:296-303) -- copies row and validity src -> dst;
 * truncate: shrink to new_size rows (dropped rows become invalid);
 * compact: stable removal of the rows with keep[i] == 0 (cleanupExpiredEntriesInternal :120-137); returns the new size. */
SR_API int sr_cache_set_valid(sr_cache* c, int local_row, int valid);
SR_API int sr_cache_move(sr_cache* c, int dst_row, int src_row);
SR_API int sr_cache_truncate(sr_cache* c, int new_size);
SR_API int sr_cache_compact(sr_cache* c, const uint8_t* keep, int n);
SR_API int sr_cache_size(const sr_cache* c);
SR_API int sr_cache_dim(const sr_cache* c);
/* queries float32 host [b, dim]; out_idx int32 [b,k] (global ids, -1 = none), out_score float [b,k].
 * Semantics: pkg/cache/inmemory_cache_search.go:65-89 (k = 1) and ffi/embedding.rs:1640-1681 (top-k):
 * descending score, lower index wins ties. */
SR_API int sr_cache_topk(sr_cache* c, const float* queries, int b, int k, int32_t* out_idx, float* out_score);
/* device-resident variant: d_queries fp16 [b, dim]; results in device buffers owned by the cache, valid until the next
 * scan of this cache.  Asynchronous on `cuda_stream`: growing the scratch and queueing the scan are locked, but callers
 * that share one cache through this entry serialise "scan, then read the results" themselves (sr_cache_topk and
 * sr_cache_lookup_ids do it under the cache's lock). */
SR_API int sr_cache_topk_dev(sr_cache* c, const void* d_queries_f16, int b, int k, void* cuda_stream);
SR_API const int32_t* sr_cache_dev_idx(const sr_cache* c);
/* Sharded cache (SURVEY 8e): every rank scans its row shard for the whole query batch, the per-rank [b,k] lists travel
 * as 8-byte entries {float score, int32 GLOBAL id} (b * k * 8 bytes per rank through ONE all-gather over NVLink), and
 * the g gathered lists are merged on the device with the reference tie rule (descending score, lower global id first;
 * pkg/cache/inmemory_cache_search.go:65-89, ffi/embedding.rs:1640-1681).
 * sr_cache_topk_packed_dev: scan + pack into d_pairs_out [b,k] entries (device memory of the caller, e.g. the send buffer
 * of the collective).  sr_cache_merge_packed_dev: d_pairs_parts [g][b,k] entries -> d_out_idx / d_out_score [b,k]. */
SR_API int sr_cache_topk_packed_dev(sr_cache* c, const void* d_queries_f16, int b, int k, void* d_pairs_out, void* cuda_stream);
SR_API int sr_cache_merge_packed_dev(int device, const void* d_pairs_parts, int g, int b, int k, int32_t* d_out_idx,
                                     float* d_out_score, void* cuda_stream);
SR_API const float* sr_cache_dev_score(const sr_cache* c);
/* The whole lookup of pkg/cache/inmemory_cache_search.go:27-176 (embed the query, scan, best matches) in one call with
 * the embedding never leaving the device: encoder to target_layer (<= 0: all) -> pool -> narrow to the cache's dim ->
 * L2 normalise -> fp16 -> scan.  ids/cu_seqlens host, out_idx/out_score host [batch, k].  The cache must live on the
 * model's device.  Thread-safe: holds the model's and the cache's locks until the results have landed on the host. */
SR_API int sr_cache_lookup_ids(sr_model* m, sr_cache* c, const int32_t* ids, const int32_t* cu_seqlens, int batch,
                        int target_layer, int k, int32_t* out_idx, float* out_score);
/* merge G per-shard result lists (host): idx/score [G][b,k] -> [b,k] */
SR_API int sr_cache_merge_topk(const int32_t* idx_parts, const float* score_parts, int g, int b, int k,
                        int32_t* out_idx, float* out_score);

/* ---- host tokenizer (tokenizer.json -> ids + byte offsets; replaces the `tokenizers` crate behind
 * candle-binding/src/core/tokenization.rs:196-395) ------------------------------------------------------ */
typedef struct sr_tokenizer sr_tokenizer;
SR_API int sr_tokenizer_load(const char* tokenizer_json_path, sr_tokenizer** out);
SR_API void sr_tokenizer_free(sr_tokenizer* t);
/* encode(text, add_special_tokens) with truncation to max_length (<= 0: none).  Writes up to cap ids and
 * 2*cap byte offsets (start, end); returns the token count (call again with a larger cap if it exceeds cap),
 * -1 on error. */
SR_API int sr_tokenizer_encode(const sr_tokenizer* t, const char* text, int add_special_tokens, int max_length,
                               int32_t* ids, int32_t* offsets, int cap);

/* request coalescing statistics of the text ABI: batches executed / requests served by them (process-wide) */
SR_API void sr_abi_batch_stats(long long* batches, long long* requests);
/* Multi-GPU dispatch of the text ABI: the library replicates every slot on the devices SR_B200_DEVICES names ("all" or
 * "0,2,5"; unset: SR_B200_DEVICE if set, else every visible GPU) and hands each call -- and each piece of a batch call
 * -- to the least-loaded replica.  Returns the number of requests (texts) handed to `device` so far, -1 if out of range. */
SR_API long long sr_abi_device_requests(int device);

#ifdef __cplusplus
}
#endif
#endif
