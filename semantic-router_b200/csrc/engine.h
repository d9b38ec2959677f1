// Encoder engine: model loading (config.json + model.safetensors), device-resident weights, workspace,
// and the forward orchestration of the kernels (one CUDA stream per model instance).
//
// Replaces L1+L0 of the reference (SURVEY.md section 1): candle-binding/src/model_architectures/traditional/
// {bert.rs, modernbert.rs, candle_models/modernbert.rs}, embedding/mmbert_embedding.rs and the candle crates.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "kernels.h"

namespace srb {

enum Arch { ARCH_MODERNBERT = 0, ARCH_BERT = 1 };

struct EncoderConfig {
  Arch arch = ARCH_MODERNBERT;
  int vocab = 0, H = 0, L = 0, heads = 0, I = 0, max_pos = 0;
  float ln_eps = 1e-5f;
  int pad_id = 0;
  int global_every = 3;
  double theta_global = 160000.0, theta_local = 10000.0;
  int local_attention = 128;
  int type_vocab = 2;
  int cls_pooling = 0;  // config.json "classifier_pooling": 0 = "cls", 1 = "mean" (read by the HF head flavour only)
  // width of the q / k / v and attention-output rows: heads * 64.  Equals H except for MiniLM-class BERT encoders
  // (12 heads x 32, all-MiniLM-L6/L12): their heads are zero-padded to 64 at load time so the head_dim-64 attention
  // kernels serve them unchanged (the padding contributes exact zeros to q.k and to the context rows).
  int attn_w = 0;
  std::map<int, std::string> id2label;
};

struct LayerWeights {     // one layer's projections (its norms are per task: TaskNorms)
  __half* wqkv = nullptr;        // [3H, H]
  float* bqkv = nullptr;         // BERT only
  __half* wo = nullptr;          // [H, H]
  float* bo = nullptr;
  __half* wi = nullptr;          // ModernBERT [2I, H] (GeGLU-interleaved) / BERT [I, H]
  float* bi = nullptr;
  __half* wo2 = nullptr;         // [H, I]
  float* bo2 = nullptr;
  // LayerNorm fold (pre-LN models, gemm.h): W diag(gamma) with zero-sum rows, fp16, for the two projections that
  // consume a LayerNorm output; null when the fold is off or the layer has no such norm
  __half* wqkv_f = nullptr;      // Wqkv diag(attn_norm), rows centred
  __half* wi_f = nullptr;        // Wi (GeGLU-interleaved) diag(mlp_norm), rows centred
};

struct Head {
  bool token_level = false;
  int num_classes = 0;
  bool has_dense = false;          // ModernBERT head.dense / BERT pooler
  float* dense_w32 = nullptr;      // [H,H] fp32 (sequence heads)
  __half* dense_w16 = nullptr;     // [H,H] fp16 (token heads: dense runs on the wgmma GEMM)
  float* dense_b = nullptr;
  float* norm_w = nullptr;
  float* cls_w = nullptr;
  float* cls_b = nullptr;
  float* final_norm_w = nullptr;   // ModernBERT: the final_norm of this head's task (Model::task)
  std::map<int, std::string> id2label;
};

struct Workspace {
  int cap_tokens = 0, cap_seqs = 0;
  uint64_t generation = 0;   // bumped whenever a device buffer is reallocated (captured graphs hold the old pointers)
  float* x = nullptr;       // fp32 residual stream [T,H]
  __half* h = nullptr;      // fp16 GEMM A operand [T,H]
  __half* lo = nullptr;     // [T,H] low halves of the fp16-pair residual stream (gemm.h: EPI_RESID_HL; w.h holds the high halves)
  __half* qkv = nullptr;    // [T,3H]
  __half* ctx = nullptr;    // [T,H]
  __half* mid = nullptr;    // [T, I]
  int* ids = nullptr;       // [T]
  int* pos = nullptr;       // [T]
  // LayerNorm fold: two ping-pong records, each [H/128][T][2] partial (sum, sum of squares) + [T] row pivots
  float* row_stats = nullptr;
  int* cu = nullptr;        // [B+1]
  int* kv_lens = nullptr;   // [B] valid keys per sequence (sr_embed_ids_padded: right-padded BERT rows whose pads stay queries)
  float* pooled = nullptr;  // [B,H]
  float* pool_part = nullptr;   // [B, kPoolParts, H] partial sums of the split pooling
  int* pool_arrived = nullptr;  // [B] arrival counters (zero between calls)
  float* logits = nullptr;  // [max(B,T), Cmax] (sized lazily)
  float* probs = nullptr;
  int* cls = nullptr;
  float* conf = nullptr;
  float* emb = nullptr;     // [B,H]
  size_t out_elems = 0;
  // precise path (precise.cu), sized for cap_tokens rows while Model::precise.on
  int cap_precise = 0;      // rows the buffers below hold
  __half* split = nullptr;  // [T, 3 * max(H, I)]  A operand [hi | lo | hi]
  float* qkv32 = nullptr;   // [T, 3H]
  float* ctx32 = nullptr;   // [T, H]
  float* mid32 = nullptr;   // ModernBERT [T, 2I] / BERT [T, I]
  float* act32 = nullptr;   // ModernBERT [T, I]
  // pinned host staging
  int* h_ids = nullptr;
  int* h_cu = nullptr;
  float* h_out = nullptr;
  int* h_cls = nullptr;
  float* h_conf = nullptr;
  size_t h_out_elems = 0;
  int h_cap_tokens = 0, h_cap_seqs = 0;
};

enum ProfCat { PC_EMBED = 0, PC_NORM, PC_GEMM_QKV, PC_ATTN, PC_GEMM_WO, PC_GEMM_WI, PC_GEMM_WO2, PC_HEAD, PC_COUNT };

// Optional per-category device timing (cudaEvent pairs on the model stream) for the roofline report.
struct Profiler {
  bool on = false;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  struct Rec { int cat; cudaEvent_t a, b; };
  std::vector<Rec> recs;
  float ms[PC_COUNT] = {0};
  int count[PC_COUNT] = {0};
};

// "Precise" path (precise.cu): split-fp16 weights [W_hi | W_hi | W_lo] per projection, in source order (BERT / MiniLM:
// no padded heads, no scaled query rows) and their fp32 biases (BERT; null for ModernBERT).  Its fp32 intermediates are
// workspace buffers (Workspace::split ... act32).
struct PreciseLayer {
  __half* wqkv = nullptr;   // [3H, 3H]
  __half* wo = nullptr;     // [H, 3H]
  __half* wi = nullptr;     // ModernBERT [2I, 3H] (original row order: a rows, then b rows) / BERT [I, 3H]
  __half* wo2 = nullptr;    // [H, 3I]
  float *bqkv = nullptr, *bo = nullptr, *bi = nullptr, *bo2 = nullptr;
};
struct PreciseState {
  bool on = false;
  std::vector<PreciseLayer> layers;
};

// Several task checkpoints of one encoder served in ONE pass (model_load_grouped): merged or fully fine-tuned
// checkpoints, or unmerged LoRA adapters over one base (model_load_lora_shared).  The T tasks' projection matrices are
// stacked along N in Model::layers, each task's own LayerNorm gamma folded into its slice and BERT's biases stacked the
// same way; every task's embeddings and norms are Model::task[t].  A batch runs ONCE as T copies of its rows (task-major,
// each copy padded to whole 256-row blocks): every row block of a projection GEMM picks its task's matrix and bias
// (gemm.h: w_groups), every row kernel its task's embeddings and norms (kernels.h: RowGroups), every task's head its
// task's final_norm -- the numerics of T separately loaded models in one pass.  Outside such a pass the model is task 0;
// a model from model_load is a model of that one task.
struct TaskNorms {      // one layer's norms of one task (null where the architecture has none)
  float* attn_w = nullptr;   // ModernBERT pre-attention LN (null on layer 0 and wherever the checkpoint has none)
  float* mid_w = nullptr;    // ModernBERT mlp_norm / BERT attention.output.LayerNorm
  float* mid_b = nullptr;
  float *out_w = nullptr, *out_b = nullptr;   // BERT output.LayerNorm
};
struct TaskTensors {    // one task's tensors outside the projections; a tensor equal in every task is ONE allocation
  float *emb_word = nullptr, *emb_pos = nullptr, *emb_type0 = nullptr, *emb_ln_w = nullptr, *emb_ln_b = nullptr;
  float* final_norm_w = nullptr;
  std::vector<TaskNorms> layers;
};
struct Grouped {        // what describes a grouped pass
  int tasks = 0;        // 0: a model from model_load
  std::vector<int> head_of_task;
  int rows_per_task = 0;   // set (under mu) for one forward: rows [t * rows_per_task, (t + 1) * rows_per_task) belong to task t
};

struct Model {
  int device = 0;
  PreciseState precise;
  Grouped group;
  Profiler prof;
  EncoderConfig cfg;
  std::string dir;
  std::vector<TaskTensors> task;   // at least one; task[0] outside a grouped pass
  std::vector<LayerWeights> layers;
  float *rope_cos_g = nullptr, *rope_sin_g = nullptr, *rope_cos_l = nullptr, *rope_sin_l = nullptr;   // cfg.max_pos rows
  std::vector<Head> heads;
  // 0: candle semantics (MEAN pooling always, tanh GELU, eps 1e-12, first-max; traditional/modernbert.rs:303-329,818)
  // 1: HF / ONNX-export semantics (pooling per config, erf GELU, eps = norm_eps, last-max;
  //    onnx-binding/src/model_architectures/classification/mmbert_classifier.rs:796-830 consumes that graph)
  int head_flavor = 0;
  Workspace ws;
  // set (under mu) for one forward by sr_embed_ids_padded: device [B] real lengths; null otherwise
  const int* cur_kv_lens = nullptr;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  std::vector<void*> allocs;  // everything to cudaFree
  size_t weight_bytes = 0;    // bytes of those allocations (the loaded tensors)
};

// The loaders read every directory on the host first: a checkpoint that cannot be served is refused before a device is
// touched.  Adapters a checkpoint carries are merged (lora_config.json alpha).
// One checkpoint as a model of one task (Grouped::tasks stays 0); its classifier, when there is one of width H, is head 0
// (token_level from config.json).
Model* model_load(const std::string& dir, int device, std::string* err);
// 1..8 task checkpoints of one encoder shape (every EncoderConfig field equal, no padded heads), each with its own head,
// as one grouped model (engine.h: Grouped).  token_level[t]: 1 / 0 / -1 (from config.json).
Model* model_load_grouped(const std::vector<std::string>& dirs, const std::vector<int>& token_level, int device,
                          std::string* err);
// model_load_grouped for unmerged LoRA checkpoints over ONE base: refuses directories whose base tensors differ or that
// carry no adapters.
Model* model_load_lora_shared(const std::vector<std::string>& dirs, const std::vector<int>& token_level, int device,
                              std::string* err);
int checkpoint_has_adapters(const std::string& dir);
// The precise path's split weights (PreciseLayer), built once from <m.dir>/model.safetensors opened afresh: every layer's
// four projections in source order, adapters merged as model_load merges them.  Not counted in m.weight_bytes.
int precise_prepare(Model& m, std::string* err);
int model_add_head(Model* m, const std::string& dir, int force_token_level, std::string* err);
void model_free(Model* m);

int workspace_reserve(Model& m, int tokens, int seqs, size_t out_elems);
// The precise path's workspace buffers for ws.cap_tokens rows (workspace_reserve calls it while m.precise.on).  On
// failure ws.cap_tokens drops to 0, so no forward runs until a reservation succeeds.
int precise_reserve(Model& m);
void profile_enable(Model& m, bool on);
// synchronises the stream, folds the recorded event pairs into prof.ms / prof.count
int profile_collect(Model& m);

// All of the following enqueue on m.stream and do NOT synchronise.
// ids/cu are device pointers (int32); T = cu[B]; max_len = longest sequence.
int encoder_forward(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int num_layers);
// precise.cu: encoder_forward's embedding and first L layers while m.precise.on (encoder_forward has checked the
// capacity and the positions and computed ws.pos)
int encoder_forward_precise(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int L);
// The precise path's row kernels, one launcher each (device pointers, asynchronous on s; note_launch per launch):
// x [T, H] fp32 -> out [T, 3H] fp16 rows [hi | lo | hi], hi = fp16(v), lo = fp16(v - hi), v = x or (gamma non-null) the
// no-bias LayerNorm (x - mean) rsqrt(var + eps) gamma
int precise_split_rows(cudaStream_t s, const float* x, int T, int H, const float* gamma, float eps, __half* out);
// rotate-half RoPE in place on the q and k thirds of qkv [T, 3 * heads * 64] fp32, row pos[t] of the [*, 32] tables
int precise_rope(cudaStream_t s, float* qkv, const int* pos, int T, int heads, const float* cos_t, const float* sin_t);
// out [T, I] = gelu_erf(a) * b over ab [T, 2I] fp32 (a = the first I columns, b = the last I)
int precise_geglu(cudaStream_t s, const float* ab, int T, int I, float* out);
// x = gelu_erf(x) in place over fp32 [T, I]
int precise_gelu(cudaStream_t s, float* x, int T, int I);
// fp32 softmax(D^-1/2 q k^T) v per head of D = head_dim (32 or 64) over packed qkv [T, 3 * heads * D] -> out
// [T, heads * D]; window 0: global, else |i - j| <= window; kv_lens [batch] (optional, global attention only): keys
// >= kv_lens[b] of sequence b are masked for every query row while all rows stay queries (attention_wgmma_fwd's kv_lens);
// any batch (slices of kMaxGridZ sequences)
int precise_attention(cudaStream_t s, const float* qkv, float* out, const int* cu_seqlens, int batch, int max_len, int heads,
                      int head_dim, int window, const int* kv_lens = nullptr);
// Sequence classification with head `head`: writes ws.logits/probs [B,C], ws.cls, ws.conf.
int head_sequence(Model& m, int head, const int* d_cu, int B, int pooler_mode);
// Token classification with head `head`: writes ws.logits/probs [T,C], ws.cls [T], ws.conf [T].
// row0: first row of the hidden states this head reads (grouped passes hold one copy of the batch per task)
int head_tokens(Model& m, int head, int B, int T, int row0 = 0);
// Embedding: mean/CLS pool (+final norm for ModernBERT) -> narrow(dim) -> L2 normalise into ws.emb [B,dim].
int head_embedding(Model& m, const int* d_cu, int B, int dim, float norm_eps);

}  // namespace srb
