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
 * checkpoint becomes head 0.  Replaces init_* of the reference (candle-binding/src/ffi/init.rs:154-877).
 * The directory is checked before the device: one that cannot be served is refused from its config.json and
 * safetensors header alone, so on a host without a usable device its own error is reported, not the device's.  A
 * servable directory still needs an sm_90 device ("no CUDA device available" without one). */
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
/* Encoder arithmetic of a model.  0 (default): the production path -- fp16 operands on the tensor cores, fp32
 * accumulation, residual stream and statistics (logits of the x8-scaled synthetic heads within ~3e-4 RELATIVE of the
 * fp32 reference).  1: the "precise" path -- every GEMM operand as an fp16 hi + lo pair (three wgmma passes in one GEMM of
 * triple depth, fp32-equivalent products), fp32 LayerNorm / RoPE / GeGLU / attention in between: logits and embeddings
 * within the 1e-3 ABSOLUTE bound of BASELINE's north star, at several times the cost.  Parity mode, not a serving mode.
 * ModernBERT / mmBERT and BERT / MiniLM encoders: for BERT the post-LN layers run with fp32 biases added in the GEMM
 * epilogue, fp32 erf GELU and fp32 attention over the model's own heads (64, or MiniLM's 32: no zero-padded heads), and
 * every entry that runs the encoder (sr_classify_ids under both pooler modes, sr_classify_tokens_ids,
 * sr_classify_multi_ids, sr_embed_ids, sr_embed_ids_padded with its key lengths) takes it.  Returns -1 for grouped
 * models (sr_model_load_grouped / sr_model_load_lora_shared). */
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

/* ---- several task checkpoints of one encoder in ONE pass ---------------------------------------------------
 * task_dirs[t] (1 <= n_tasks <= 8) is a complete checkpoint of task t with its own classifier head: merged LoRA models
 * (the reference publishes its LoRA classifiers merged, lora_*_model), full fine-tunes of one base, or anything else of
 * one encoder shape.  Every config.json field that shapes the encoder (architecture, hidden_size, num_hidden_layers,
 * num_attention_heads, intermediate_size, vocab_size, max_position_embeddings, global_attn_every_n_layers,
 * local_attention, both rope thetas, layer_norm_eps, classifier_pooling) must be equal, padded-head (MiniLM) encoders
 * are refused, and so are two or more BERT tasks whose intermediate_size is not a multiple of 128; these refusals name
 * the field and the directory and come before any device is touched.  A tensor that
 * is bitwise the same in every task is loaded once; one that differs gets a device copy per task.  Each task's
 * projection weights (its own LayerNorm gamma folded in, adapters a checkpoint still carries merged as sr_model_load
 * merges them) are stacked.  A batch then runs ONCE through the encoder as n_tasks copies of its rows, each padded to
 * whole 256-row blocks by pad sequences of at most min(255, max_position_embeddings) rows: each 256-row block
 * of a projection GEMM picks its task's matrix and bias, every embedding and LayerNorm row its task's weights, every
 * task's head its task's final norm -- bitwise what n_tasks separately loaded models give.  The ordinary entries above
 * run task 0's encoder on such a model; sr_model_set_precise refuses it.  token_level[t]: 1 token head, 0 sequence head, -1
 * from config.json. */
SR_API int sr_model_load_grouped(const char* const* task_dirs, const int* token_level, int n_tasks, int device,
                                 sr_model** out);
/* sr_model_load_grouped for UNMERGED LoRA checkpoints over one base (SURVEY section 8 f3): the reference's LoRA path
 * computes x W^T + (alpha / r) (x A^T) B^T per adapted Linear (candle-binding/src/model_architectures/lora/
 * lora_adapter.rs:136-144).  Every directory carries the SAME base tensors (checked bit for bit; refused otherwise),
 * `X.lora_A.weight` / `X.lora_B.weight` next to the adapted `X.weight`s and lora_config.json {"rank", "alpha"}; a set
 * without adapters is refused (load it with sr_model_load_grouped).  Each task's adapters are folded into its own copy
 * of the projection weights at load. */
SR_API int sr_model_load_lora_shared(const char* const* task_dirs, const int* token_level, int n_tasks, int device,
                                     sr_model** out);
/* tasks of a model from sr_model_load_grouped or sr_model_load_lora_shared; 0 for an ordinary model */
SR_API int sr_lora_shared_tasks(const sr_model* m);
/* 1: <model_dir>/model.safetensors carries lora_A / lora_B tensors, 0: it does not (a merged checkpoint), -1: unreadable */
SR_API int sr_checkpoint_has_adapters(const char* model_dir);
/* One pass of a grouped model (sr_model_load_grouped or sr_model_load_lora_shared) over a batch, every task's head.
 * For each task t: sequence heads write probs_out[t] [batch, C_t], cls_out[t] / conf_out[t] [batch]; token heads write
 * probs_out[t] [T, C_t], cls_out[t] / conf_out[t] [T] (T = cu_seqlens[batch]).  Any of the pointers may be NULL. */
SR_API int sr_classify_lora_shared_ids(sr_model* m, const int32_t* ids, const int32_t* cu_seqlens, int batch, int pooler_mode,
                                       float** probs_out, int32_t** cls_out, float** conf_out);
/* device bytes of the tensors a model holds (weights, heads, rotary tables; not the per-call workspace) */
SR_API long long sr_model_device_bytes(const sr_model* m);

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
/* An exact cache: sr_cache_topk and sr_cache_lookup_ids return, per query, the scores of the reference's
 * embeddingDotProduct (pkg/cache/inmemory_cache_search.go:14-20: dot = 0, dot += q[i] * c[i] in index order) on the fp32
 * query and the fp32 rows exactly as passed to sr_cache_add, bit for bit, and the ids in descending score order, lower
 * index first on ties, with the same -1 / -inf padding.  sum_rule picks how each term is accumulated: 0 rounds the product
 * to fp32, then adds (Go on amd64 at the default GOAMD64=v1); 1 is one fused multiply-add (Go on arm64, ppc64le, s390x and
 * on amd64 at GOAMD64=v3 or higher); any other value is refused.  The store keeps every row twice, fp32 beside the fp16
 * copy (6 bytes per element instead of 2).  The fp16 scan stays the filter: it picks k' candidates per query (k' = 32 for
 * k <= 32 and 64 above, where the two-stage selection takes that many, else 16 or k), a certified band of them is rescored in Go order, and a query
 * whose band does not fit in k' is scanned exhaustively in Go order on the CUDA cores.  Limits: 1 <= k <= 64 and
 * ceil(size / 8192) * k <= 25600 for every b (the fallback selects through the two-stage selection; there is no fused
 * route).  No scan waits on the host: how many queries fell back stays on the device.  Refused (-1, outputs untouched):
 * rows (sr_cache_add) or queries (sr_cache_topk) with a non-finite component or one of magnitude above 65504;
 * sr_cache_topk_dev and sr_cache_topk_packed_dev, which see only fp16 queries -- device-resident queries of an exact cache
 * go through sr_cache_topk_f32_dev and sr_cache_topk_packed_f32_dev, and a sharded exact cache merges its shards' lists
 * with sr_cache_merge_packed_dev or sr_cache_merge_topk, which are exact on exact scores.  Lifecycle calls keep both
 * stores in step. */
SR_API int sr_cache_create_exact(int device, int capacity, int dim, int id_offset, int sum_rule, sr_cache** out);
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
 * descending score, lower index wins ties.  Limits: 1 <= k <= 64, and ceil(size / 8192) * k <= 25600 (the candidates
 * of the two-stage selection, 200 KB of shared memory per query; the fused route, b > 4 and k <= 8, has no size limit).
 * Returns -1 outside them, with out_idx / out_score untouched.  sr_cache_topk_dev and sr_cache_topk_packed_dev share
 * these limits. */
SR_API int sr_cache_topk(sr_cache* c, const float* queries, int b, int k, int32_t* out_idx, float* out_score);
/* device-resident variant: d_queries fp16 [b, dim]; results in device buffers owned by the cache, valid until the next
 * scan of this cache.  Asynchronous on `cuda_stream`: growing the scratch and queueing the scan are locked, but callers
 * that share one cache through this entry serialise "scan, then read the results" themselves (sr_cache_topk and
 * sr_cache_lookup_ids do it under the cache's lock).  Refused (-1) for exact caches: use sr_cache_topk_f32_dev. */
SR_API int sr_cache_topk_dev(sr_cache* c, const void* d_queries_f16, int b, int k, void* cuda_stream);
/* device-resident variant for fp32 queries, and the one for exact caches: d_queries_f32 device [b, dim] fp32, rounded to
 * fp16 into the cache's own query buffer for the candidate scan; results where sr_cache_topk_dev puts them, with its
 * limits and its rule that callers of one cache serialise "scan, then read".  Default cache: bitwise sr_cache_topk on the
 * same queries.  Exact cache: bitwise sr_cache_topk on the same queries under the cache's sum rule; a query with a
 * non-finite component or one above 65504 in magnitude, which sr_cache_topk refuses on the host, is refused here on the
 * device: its k results are (-1, -inf) and the batch's other queries are unaffected.  Asynchronous: nothing waits on the
 * host between the call and the stream reaching its results, except the scratch growth of the first call at a larger
 * (b, k) or after the store grew (it synchronises the device).  So the scan can be captured into a CUDA graph after one
 * eager call at the same (b, k).  A captured scan stays valid across sr_cache_set_valid / sr_cache_invalidate /
 * sr_cache_move; after sr_cache_add, sr_cache_truncate or sr_cache_compact capture again: the row count, the largest row
 * norm and the scratch are arguments of the captured launches. */
SR_API int sr_cache_topk_f32_dev(sr_cache* c, const float* d_queries_f32, int b, int k, void* cuda_stream);
SR_API const int32_t* sr_cache_dev_idx(const sr_cache* c);
/* Sharded cache (SURVEY 8e): every rank scans its row shard for the whole query batch, the per-rank [b,k] lists travel
 * as 8-byte entries {float score, int32 GLOBAL id} (b * k * 8 bytes per rank through ONE all-gather over NVLink), and
 * the g gathered lists are merged on the device with the reference tie rule (descending score, lower global id first;
 * pkg/cache/inmemory_cache_search.go:65-89, ffi/embedding.rs:1640-1681).
 * sr_cache_topk_packed_dev: scan + pack into d_pairs_out [b,k] entries (device memory of the caller, e.g. the send buffer
 * of the collective).  sr_cache_merge_packed_dev: d_pairs_parts [g][b,k] entries -> d_out_idx / d_out_score [b,k];
 * g * k <= 6144 (every entry of a query in 48 KB of shared memory), -1 with the outputs untouched beyond that. */
SR_API int sr_cache_topk_packed_dev(sr_cache* c, const void* d_queries_f16, int b, int k, void* d_pairs_out, void* cuda_stream);
/* sr_cache_topk_f32_dev + pack into d_pairs_out [b,k]: the sharded scan of exact caches (and of default caches fed fp32
 * queries).  Each exact shard's list holds the exact scores of its own rows, so sr_cache_merge_packed_dev of the shards'
 * lists is the unsharded exact cache's result; a query refused on the device is (-1, -inf) in every shard and merges to
 * (-1, -inf).  sr_cache_topk_packed_dev refuses exact caches. */
SR_API int sr_cache_topk_packed_f32_dev(sr_cache* c, const float* d_queries_f32, int b, int k, void* d_pairs_out,
                                        void* cuda_stream);
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
