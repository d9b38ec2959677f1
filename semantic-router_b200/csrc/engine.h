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

struct LayerWeights {
  float* attn_norm_w = nullptr;  // ModernBERT pre-attention LN (null on layer 0)
  __half* wqkv = nullptr;        // [3H, H]
  float* bqkv = nullptr;         // BERT only
  __half* wo = nullptr;          // [H, H]
  float* bo = nullptr;
  float* mid_norm_w = nullptr;   // ModernBERT mlp_norm / BERT attention.output.LayerNorm
  float* mid_norm_b = nullptr;
  __half* wi = nullptr;          // ModernBERT [2I, H] (GeGLU-interleaved) / BERT [I, H]
  float* bi = nullptr;
  __half* wo2 = nullptr;         // [H, I]
  float* bo2 = nullptr;
  float* out_norm_w = nullptr;   // BERT output.LayerNorm
  float* out_norm_b = nullptr;
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
  __half* lora_u = nullptr; // [T, lora.max_R] rank-r projections of the current GEMM's input (shared-LoRA models)
  float* pooled = nullptr;  // [B,H]
  float* pool_part = nullptr;   // [B, kPoolParts, H] partial sums of the split pooling
  int* pool_arrived = nullptr;  // [B] arrival counters (zero between calls)
  float* logits = nullptr;  // [max(B,T), Cmax] (sized lazily)
  float* probs = nullptr;
  int* cls = nullptr;
  float* conf = nullptr;
  float* emb = nullptr;     // [B,H]
  size_t out_elems = 0;
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

// "Precise" path (precise.cu): split-fp16 weights [W_hi | W_hi | W_lo] per projection and fp32 intermediates.
struct PreciseLayer {
  __half* wqkv = nullptr;   // [3H, 3H]
  __half* wo = nullptr;     // [H, 3H]
  __half* wi = nullptr;     // [2I, 3H] (original row order: a rows, then b rows)
  __half* wo2 = nullptr;    // [H, 3I]
};
struct PreciseState {
  bool on = false;
  std::vector<PreciseLayer> layers;
  __half* split = nullptr;  // [T, 3 * max(H, I)]  A operand [hi | lo | hi]
  float* qkv32 = nullptr;   // [T, 3H]
  float* ctx32 = nullptr;   // [T, H]
  float* mid32 = nullptr;   // [T, 2I]
  float* act32 = nullptr;   // [T, I]
  size_t split_cap = 0, qkv_cap = 0, ctx_cap = 0, mid_cap = 0, act_cap = 0;
};

// Shared-base multi-task serving from UNMERGED LoRA checkpoints (SURVEY section 8 f3; lora_adapter.rs:136-144): T task
// checkpoints over one base load ONE copy of the base weights plus, per projection, the tasks' rank-r factors stacked:
//   a [R, K]   rows t * block + j = A_t[j, :]            (down-projections of all tasks, one skinny GEMM: U = x a^T)
//   b [N, R]   columns t * block + j = (alpha_t / r_t) B_t[:, j]
// A batch is run as T copies of its rows (task-major); copy t keeps only its own column block of U (EPI_F16 mask) and
// the projection GEMM takes U b^T into its accumulator as a K extension (gemm.h) -- base weights read once, three
// tasks in one pass.  BERT's fused QKV has three segments per task (query / key / value adapters): block = 3 * rp.
struct LoraProj {
  __half* a = nullptr;
  __half* a_f = nullptr;   // LayerNorm-fold form of `a` (A diag(gamma), rows centred) where the projection runs folded
  __half* b = nullptr;
  int R = 0;               // padded to a multiple of 64
  int block = 0;           // columns of U per task
};
struct LoraLayer { LoraProj qkv, wo, wi, wo2; };
struct LoraShared {
  int tasks = 0;
  int max_R = 0;
  std::vector<LoraLayer> layers;
  // GROUPED form (the latency / throughput form; the low-rank form above is the memory form): every task's adapters folded
  // into its own copy of the projection weights at load (W_t = W + (alpha_t / r_t) B_t A_t), the T copies stacked along N; the
  // batch still runs ONCE as T copies of its rows, and every row block of a projection GEMM picks its task's matrix in the TMA
  // producer (gemm.h: w_groups) -- no rank-r GEMMs, no extra k-blocks, the numerics of T separately loaded models.
  bool grouped = false;
  std::vector<LayerWeights> glayers;   // per layer: the base layer's norms / biases + the stacked projection weights
  std::vector<int> head_of_task;
  int rows_per_task = 0;   // set (under mu) for one forward: rows [t * rows_per_task, (t + 1) * rows_per_task) belong to task t
};

struct Model {
  int device = 0;
  PreciseState precise;
  LoraShared lora;
  Profiler prof;
  EncoderConfig cfg;
  std::string dir;
  float* emb_word = nullptr;
  float* emb_pos = nullptr;
  float* emb_type0 = nullptr;
  float* emb_ln_w = nullptr;
  float* emb_ln_b = nullptr;
  std::vector<LayerWeights> layers;
  float* final_norm_w = nullptr;
  float *rope_cos_g = nullptr, *rope_sin_g = nullptr, *rope_cos_l = nullptr, *rope_sin_l = nullptr;
  int rope_len = 0;
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
};

// flags: kLoadKeepAdapters = leave `lora_A / lora_B` tensors unmerged (the base weights load as they are),
// kLoadNoHead = do not load <dir>'s classifier
enum { kLoadKeepAdapters = 1, kLoadNoHead = 2 };
Model* model_load(const std::string& dir, int device, std::string* err, int flags = 0);
// One base + n task checkpoints (each a full unmerged-LoRA checkpoint over the SAME base weights, with its own head);
// token_level[t]: 1 / 0 / -1 (from config.json).  Fails when the base tensors differ between the directories.
Model* model_load_lora_shared(const std::vector<std::string>& dirs, const std::vector<int>& token_level, int device,
                              bool grouped, std::string* err);
int checkpoint_has_adapters(const std::string& dir);
int model_add_head(Model* m, const std::string& dir, int force_token_level, std::string* err);
void model_free(Model* m);

int workspace_reserve(Model& m, int tokens, int seqs, size_t out_elems);
void profile_enable(Model& m, bool on);
// synchronises the stream, folds the recorded event pairs into prof.ms / prof.count
int profile_collect(Model& m);

// All of the following enqueue on m.stream and do NOT synchronise.
// ids/cu are device pointers (int32); T = cu[B]; max_len = longest sequence.
int encoder_forward(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int num_layers);
// precise.cu: builds the split weights (re-reads <dir>/model.safetensors), the fp32-equivalent forward, buffer release
int precise_prepare(Model& m, std::string* err);
int encoder_forward_precise(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int num_layers);
void precise_free(Model& m);
// Sequence classification with head `head`: writes ws.logits/probs [B,C], ws.cls, ws.conf.
int head_sequence(Model& m, int head, const int* d_cu, int B, int pooler_mode);
// Token classification with head `head`: writes ws.logits/probs [T,C], ws.cls [T], ws.conf [T].
// row0: first row of the hidden states this head reads (shared-LoRA passes hold one copy of the batch per task)
int head_tokens(Model& m, int head, int B, int T, int row0 = 0);
// Embedding: mean/CLS pool (+final norm for ModernBERT) -> narrow(dim) -> L2 normalise into ws.emb [B,dim].
int head_embedding(Model& m, const int* d_cu, int B, int dim, float norm_eps);

}  // namespace srb
