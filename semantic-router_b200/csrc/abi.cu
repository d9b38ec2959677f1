// Drop-in C ABI (include/candle_semantic_router.h): the symbol table candle-binding/semantic-router.go links,
// implemented over the CUDA engine.  Replaces candle-binding/src/ffi/{init,classify,embedding,similarity,
// tokenization,memory}.rs.  One global slot per reference OnceLock (ffi/init.rs:19-60,431-456); every result
// buffer is malloc'd here and released by the matching free_* (free(3)).
#include "../../include/candle_semantic_router.h"
#include "../../include/sr_b200_testhooks.h"
#include "abi_core.h"

#define SRB_ABI_HEAD_FLAVOR 0   // candle head semantics (sr_b200.h: sr_model_set_head_flavor)

namespace {
Slot g_similarity, g_classifier, g_pii, g_jailbreak, g_candle_bert, g_candle_bert_tok, g_bert_tok;
Slot g_mb_cls, g_mb_pii, g_mb_jb, g_mb_pii_tok, g_factcheck, g_feedback;
Slot g_mm32k_intent, g_mm32k_factcheck, g_mm32k_jailbreak, g_mm32k_feedback, g_mm32k_pii, g_mm32k_modality;
Slot g_mm_embed;
Slot g_halluc, g_nli;
EmbeddingResult emb_error() { return EmbeddingResult{nullptr, 0, true, -1, 0, 0.0f}; }
}  // namespace

extern "C" {

void sr_abi_batch_stats(long long* batches, long long* requests) {
  if (batches) *batches = g_batches.load();
  if (requests) *requests = g_batched_requests.load();
}
long long sr_abi_device_requests(int device) { return device >= 0 && device < 64 ? g_dev_requests[device].load() : -1; }

// ================================================================================================
// similarity model
// ================================================================================================
bool init_similarity_model(const char* model_id, bool use_cpu) {
  note_use_cpu(use_cpu);
  return slot_init(g_similarity, model_id, -2, false);
}
bool is_similarity_model_initialized(void) { return g_similarity.ready(); }

EmbeddingResult get_text_embedding(const char* text, int max_length) {
  std::vector<float> e;
  if (!embed_text_similarity(g_similarity, text, max_length <= 0 ? 512 : max_length, e)) return emb_error();
  return EmbeddingResult{dup_floats(e), static_cast<int>(e.size()), false, -1, 0, 0.0f};
}
float calculate_similarity(const char* text1, const char* text2, int max_length) {
  std::vector<float> a, b;
  const int ml = max_length <= 0 ? 512 : max_length;
  if (!embed_text_similarity(g_similarity, text1, ml, a) || !embed_text_similarity(g_similarity, text2, ml, b)) return -1.0f;
  return dot(a, b);
}
SimilarityResult find_most_similar(const char* query, const char** candidates, int num_candidates, int max_length) {
  SimilarityResult r{-1, -1.0f};
  if (!query || !candidates || num_candidates <= 0) return r;
  const int ml = max_length <= 0 ? 512 : max_length;
  std::vector<float> q, c;
  if (!embed_text_similarity(g_similarity, query, ml, q)) return r;
  for (int i = 0; i < num_candidates; ++i) {   // core/similarity.rs:278-308: best = -1.0, strict >
    if (!embed_text_similarity(g_similarity, candidates[i], ml, c)) return SimilarityResult{-1, -1.0f};
    const float s = dot(q, c);
    if (s > r.score) { r.score = s; r.index = i; }
  }
  return r;
}
TokenizationResult tokenize_text(const char* text, int max_length) {
  TokenizationResult r{nullptr, 0, nullptr, true};
  if (!text || !g_similarity.ready()) return r;
  const Tokens t = tokenize(g_similarity, text, max_length <= 0 ? 512 : max_length);
  const int n = static_cast<int>(t.ids.size());
  r.token_ids = static_cast<int*>(malloc(sizeof(int) * (n ? n : 1)));
  r.tokens = static_cast<char**>(malloc(sizeof(char*) * (n ? n : 1)));
  if (!r.token_ids || !r.tokens) { free(r.token_ids); free(r.tokens); return TokenizationResult{nullptr, 0, nullptr, true}; }
  for (int i = 0; i < n; ++i) { r.token_ids[i] = t.ids[i]; r.tokens[i] = dup_cstr(t.tokens[i]); }
  r.token_count = n;
  r.error = false;
  return r;
}
void free_tokenization_result(TokenizationResult result) {
  if (result.tokens) for (int i = 0; i < result.token_count; ++i) free(result.tokens[i]);
  free(result.tokens);
  free(result.token_ids);
}
void free_embedding(float* data, int) { free(data); }

// ================================================================================================
// BERT classifiers
// ================================================================================================
#define CSR_SEQ_INIT_N(fn, slot, reinit)                                    \
  bool fn(const char* model_id, int num_classes, bool use_cpu) {            \
    (void)num_classes;                                                      \
    note_use_cpu(use_cpu);                                                  \
    return slot_init(slot, model_id, 0, reinit);                            \
  }
#define CSR_SEQ_INIT(fn, slot, reinit)                                      \
  bool fn(const char* model_id, bool use_cpu) {                             \
    note_use_cpu(use_cpu);                                                  \
    return slot_init(slot, model_id, 0, reinit);                            \
  }
#define CSR_TOK_INIT(fn, slot)                                              \
  bool fn(const char* model_id, bool use_cpu) {                             \
    note_use_cpu(use_cpu);                                                  \
    return slot_init(slot, model_id, 1, true);                              \
  }
#define CSR_CLASSIFY(ret, fn, slot)                                         \
  ret fn(const char* text) {                                                \
    float conf = 0.f;                                                       \
    const int c = run_seq(slot, text, &conf, nullptr);                      \
    if (c < 0) return ret{-1, 0.0f};                                        \
    return ret{c, conf};                                                    \
  }

// NOTE (documented divergence, SURVEY section 0 fact 9): in the reference init_classifier/init_pii_classifier set
// statics that classify_text/classify_pii_text never read, so those always return -1.  Here init -> classify works.
CSR_SEQ_INIT_N(init_classifier, g_classifier, false)
CSR_SEQ_INIT_N(init_pii_classifier, g_pii, false)
CSR_SEQ_INIT_N(init_jailbreak_classifier, g_jailbreak, false)
CSR_SEQ_INIT_N(init_candle_bert_classifier, g_candle_bert, true)
CSR_CLASSIFY(ClassificationResult, classify_text, g_classifier)
CSR_CLASSIFY(ClassificationResult, classify_pii_text, g_pii)
CSR_CLASSIFY(ClassificationResult, classify_jailbreak_text, g_jailbreak)
CSR_CLASSIFY(ClassificationResult, classify_bert_text, g_classifier)
CSR_CLASSIFY(ClassificationResult, classify_candle_bert_text, g_candle_bert)

ClassificationResultWithProbs classify_text_with_probabilities(const char* text) {
  float conf = 0.f;
  std::vector<float> p;
  const int c = run_seq(g_classifier, text, &conf, &p);
  if (c < 0) return ClassificationResultWithProbs{-1, 0.0f, nullptr, 0};
  return ClassificationResultWithProbs{c, conf, dup_floats(p), static_cast<int>(p.size())};
}
void free_probabilities(float* probabilities, int) { free(probabilities); }

bool init_candle_bert_token_classifier(const char* model_path, int, bool use_cpu) {
  note_use_cpu(use_cpu);
  return slot_init(g_candle_bert_tok, model_path, 1, true);
}
bool init_bert_token_classifier(const char* model_path, int, bool use_cpu) {
  note_use_cpu(use_cpu);
  return slot_init(g_bert_tok, model_path, 1, true);
}

static BertTokenClassificationResult bert_tokens(Slot& s, const char* text, const char* id2label_json) {
  BertTokenClassificationResult none{nullptr, 0};
  std::vector<TokenPred> toks;
  if (!run_tokens(s, text, toks)) return none;
  std::map<int, std::string> id2label = s.id2label;
  if (id2label_json && *id2label_json) {
    Json j;
    srb::JsonParser jp(id2label_json, strlen(id2label_json));
    if (jp.parse(j) && j.is_obj()) {
      id2label.clear();
      for (const auto& kv : j.obj) if (kv.second.is_str()) id2label[atoi(kv.first.c_str())] = kv.second.str;
    }
  }
  // per-token entities for non-"O" predictions (ffi/classify.rs:560-578)
  std::vector<Entity> ents;
  std::vector<std::string> types;
  for (const auto& t : toks) {
    if (t.start == 0 && t.end == 0) continue;
    auto it = id2label.find(t.pred);
    const std::string label = it == id2label.end() ? "label_" + std::to_string(t.pred) : it->second;
    if (t.pred == 0 || label == "O") continue;
    ents.push_back(Entity{label, t.pred, t.start, t.end, t.conf});
    types.push_back(label);
  }
  return pack_entities<BertTokenEntity, BertTokenClassificationResult>(text, ents, types);
}
BertTokenClassificationResult classify_candle_bert_tokens(const char* text) { return bert_tokens(g_candle_bert_tok, text, nullptr); }
BertTokenClassificationResult classify_candle_bert_tokens_with_labels(const char* text, const char* id2label_json) {
  return bert_tokens(g_candle_bert_tok, text, id2label_json);
}
BertTokenClassificationResult classify_bert_pii_tokens(const char* text, const char* id2label_json) {
  return bert_tokens(g_bert_tok.ready() ? g_bert_tok : g_candle_bert_tok, text, id2label_json);
}
void free_bert_token_classification_result(BertTokenClassificationResult result) {
  if (result.entities)
    for (int i = 0; i < result.num_entities; ++i) { free(result.entities[i].entity_type); free(result.entities[i].text); }
  free(result.entities);
}

// ================================================================================================
// ModernBERT / mmBERT classifiers
// ================================================================================================
CSR_SEQ_INIT(init_modernbert_classifier, g_mb_cls, false)
CSR_SEQ_INIT(init_modernbert_pii_classifier, g_mb_pii, false)
CSR_SEQ_INIT(init_modernbert_jailbreak_classifier, g_mb_jb, false)
CSR_SEQ_INIT(init_fact_check_classifier, g_factcheck, false)
CSR_SEQ_INIT(init_feedback_detector, g_feedback, false)
CSR_TOK_INIT(init_modernbert_pii_token_classifier, g_mb_pii_tok)
CSR_SEQ_INIT(init_mmbert_classifier, g_mb_cls, false)
CSR_SEQ_INIT(init_mmbert_classifier_auto, g_mb_cls, false)
CSR_TOK_INIT(init_mmbert_token_classifier, g_mb_pii_tok)
CSR_SEQ_INIT(init_mmbert_32k_intent_classifier, g_mm32k_intent, false)
CSR_SEQ_INIT(init_mmbert_32k_factcheck_classifier, g_mm32k_factcheck, false)
CSR_SEQ_INIT(init_mmbert_32k_jailbreak_classifier, g_mm32k_jailbreak, false)
CSR_SEQ_INIT(init_mmbert_32k_feedback_classifier, g_mm32k_feedback, false)
CSR_SEQ_INIT(init_mmbert_32k_modality_classifier, g_mm32k_modality, false)
CSR_TOK_INIT(init_mmbert_32k_pii_classifier, g_mm32k_pii)
CSR_CLASSIFY(ModernBertClassificationResult, classify_modernbert_text, g_mb_cls)
CSR_CLASSIFY(ModernBertClassificationResult, classify_modernbert_pii_text, g_mb_pii)
CSR_CLASSIFY(ModernBertClassificationResult, classify_modernbert_jailbreak_text, g_mb_jb)
CSR_CLASSIFY(ModernBertClassificationResult, classify_fact_check_text, g_factcheck)
CSR_CLASSIFY(ModernBertClassificationResult, classify_feedback_text, g_feedback)
CSR_CLASSIFY(ModernBertClassificationResult, classify_mmbert_32k_intent, g_mm32k_intent)
CSR_CLASSIFY(ModernBertClassificationResult, classify_mmbert_32k_factcheck, g_mm32k_factcheck)
CSR_CLASSIFY(ModernBertClassificationResult, classify_mmbert_32k_jailbreak, g_mm32k_jailbreak)
CSR_CLASSIFY(ModernBertClassificationResult, classify_mmbert_32k_feedback, g_mm32k_feedback)
CSR_CLASSIFY(ModernBertClassificationResult, classify_mmbert_32k_modality, g_mm32k_modality)

ModernBertClassificationResultWithProbs classify_modernbert_text_with_probabilities(const char* text) {
  float conf = 0.f;
  std::vector<float> p;
  const int c = run_seq(g_mb_cls, text, &conf, &p);
  if (c < 0) return ModernBertClassificationResultWithProbs{-1, 0.0f, nullptr, 0};
  return ModernBertClassificationResultWithProbs{c, conf, dup_floats(p), static_cast<int>(p.size())};
}
void free_modernbert_probabilities(float* probabilities, int) { free(probabilities); }

ModernBertTokenClassificationResult classify_modernbert_pii_tokens(const char* text, const char* model_config_path) {
  ModernBertTokenClassificationResult none{nullptr, 0};
  std::vector<TokenPred> toks;
  if (!model_config_path || !run_tokens(g_mb_pii_tok, text, toks)) return none;
  std::map<int, std::string> id2label;
  load_id2label(model_config_path, id2label);
  if (id2label.empty()) return ModernBertTokenClassificationResult{nullptr, -1};   // ffi/classify.rs:1391-1400
  std::vector<Entity> all = bio_decode(toks, id2label), ents;
  std::vector<std::string> types;
  for (const auto& e : all)
    if (e.conf > 0.5f && e.cls > 0) {   // ffi/classify.rs:1404-1411
      ents.push_back(e);
      auto it = id2label.find(e.cls);
      types.push_back(it == id2label.end() ? "UNKNOWN_PII" : it->second);
    }
  return pack_entities<ModernBertTokenEntity, ModernBertTokenClassificationResult>(text, ents, types);
}
ModernBertTokenClassificationResult classify_mmbert_32k_pii_tokens(const char* text) {
  ModernBertTokenClassificationResult none{nullptr, 0};
  std::vector<TokenPred> toks;
  if (!run_tokens(g_mm32k_pii, text, toks)) return none;
  const std::vector<Entity> ents = bio_decode(toks, g_mm32k_pii.id2label);
  std::vector<std::string> types;
  for (const auto& e : ents) types.push_back("LABEL_" + std::to_string(e.cls));   // ffi/classify.rs:2282
  return pack_entities<ModernBertTokenEntity, ModernBertTokenClassificationResult>(text, ents, types);
}
void free_modernbert_token_result(ModernBertTokenClassificationResult result) {
  if (result.entities)
    for (int i = 0; i < result.num_entities; ++i) { free(result.entities[i].entity_type); free(result.entities[i].text); }
  free(result.entities);
}

static bool config_says(const char* config_path, bool want_32k) {
  if (!config_path) return false;
  Json cfg;
  if (!srb::parse_json_file(config_path, cfg)) return false;
  const double vocab = cfg.num_or("vocab_size", 0), maxpos = cfg.num_or("max_position_embeddings", 0);
  const bool mm = cfg.str_or("model_type", "") == "modernbert" && vocab >= 200000;   // traditional/modernbert.rs:42-55
  return want_32k ? (mm && maxpos >= 32768) : mm;
}
bool is_mmbert_model(const char* config_path) { return config_says(config_path, false); }
bool is_mmbert_32k_model(const char* config_path) { return config_says(config_path, true); }

// ================================================================================================
// embeddings
// ================================================================================================
bool init_mmbert_embedding_model(const char* model_path, bool use_cpu) {
  note_use_cpu(use_cpu);
  const bool ok = slot_init(g_mm_embed, model_path, -2, true);
  if (ok) g_mm_embed.max_len = g_mm_embed.max_pos;   // no truncation besides the position table (ffi/embedding.rs:720)
  return ok;
}
bool init_embedding_models_with_mmbert(const char* qwen3, const char* gemma, const char* mmbert, bool use_cpu) {
  const bool want_other = (qwen3 && *qwen3) || (gemma && *gemma);
  if (want_other) fprintf(stderr, "[srb200] qwen3/gemma embedding models are out of scope (SURVEY 2 row 7): ignored\n");
  if (mmbert && *mmbert) return init_mmbert_embedding_model(mmbert, use_cpu);
  return false;
}
bool init_embedding_models(const char* qwen3, const char* gemma, bool use_cpu) {
  return init_embedding_models_with_mmbert(qwen3, gemma, nullptr, use_cpu);
}
bool init_embedding_models_batched(const char*, int, unsigned long long, bool) { return false; }   // Qwen3 only

static int embed_into(const char* text, const char* model_type, int layer, int dim, EmbeddingResult* result) {
  if (!text || !result) return -1;
  if (model_type && strcmp(model_type, "mmbert") != 0 && strcmp(model_type, "auto") != 0) { *result = emb_error(); return -1; }
  const double t0 = now_ms();
  std::vector<float> e;
  if (!embed_text(g_mm_embed, text, g_mm_embed.max_len, layer > 0 ? layer : 0, dim > 0 ? dim : 0, e)) { *result = emb_error(); return -1; }
  *result = EmbeddingResult{dup_floats(e), static_cast<int>(e.size()), false, 2, word_count(text), static_cast<float>(now_ms() - t0)};
  return 0;
}
int get_embedding_2d_matryoshka(const char* text, const char* model_type, int target_layer, int target_dim, EmbeddingResult* result) {
  if (!model_type) return -1;
  return embed_into(text, model_type, target_layer, target_dim, result);
}
int get_embedding_with_model_type(const char* text, const char* model_type, int target_dim, EmbeddingResult* result) {
  return embed_into(text, model_type, 0, target_dim, result);
}
int get_embedding_batched(const char* text, const char* model_type, int target_dim, EmbeddingResult* result) {
  return embed_into(text, model_type, 0, target_dim, result);
}
int get_embedding_smart(const char* text, float, float, EmbeddingResult* result) { return embed_into(text, "mmbert", 0, 0, result); }
int get_embedding_with_dim(const char* text, float, float, int target_dim, EmbeddingResult* result) {
  return embed_into(text, "mmbert", 0, target_dim, result);
}
int calculate_embedding_similarity(const char* text1, const char* text2, const char* model_type, int target_dim,
                                   EmbeddingSimilarityResult* result) {
  if (!result) return -1;
  *result = EmbeddingSimilarityResult{-1.0f, -1, 0.0f, true};
  if (model_type && strcmp(model_type, "mmbert") != 0 && strcmp(model_type, "auto") != 0) return -1;
  const double t0 = now_ms();
  std::vector<float> a, b;
  if (!embed_text(g_mm_embed, text1, g_mm_embed.max_len, 0, target_dim, a) ||
      !embed_text(g_mm_embed, text2, g_mm_embed.max_len, 0, target_dim, b))
    return -1;
  const float na = std::sqrt(dot(a, a)), nb = std::sqrt(dot(b, b));
  *result = EmbeddingSimilarityResult{(na > 0 && nb > 0) ? dot(a, b) / (na * nb) : 0.0f, 2, static_cast<float>(now_ms() - t0), false};
  return 0;
}
int calculate_similarity_batch(const char* query, const char** candidates, int num_candidates, int top_k, const char* model_type,
                               int target_dim, BatchSimilarityResult* result) {
  if (!result) return -1;
  *result = BatchSimilarityResult{nullptr, 0, -1, 0.0f, true};
  if (!query || !candidates || num_candidates <= 0) return -1;
  if (model_type && strcmp(model_type, "mmbert") != 0 && strcmp(model_type, "auto") != 0) return -1;
  const double t0 = now_ms();
  // query + candidates as ONE packed varlen batch (the reference embeds them one forward at a time,
  // ffi/embedding.rs:1600-1659); cosine and the stable sort stay on the host
  std::vector<const char*> all{query};
  for (int i = 0; i < num_candidates; ++i) {
    if (!candidates[i]) return -1;
    all.push_back(candidates[i]);
  }
  std::vector<float> e;
  int d = 0;
  if (!embed_packed(g_mm_embed, all.data(), static_cast<int>(all.size()), g_mm_embed.max_len, 0, target_dim, e, d)) return -1;
  auto row_dot = [&](const float* a, const float* b) { float acc = 0.f; for (int j = 0; j < d; ++j) acc += a[j] * b[j]; return acc; };
  const float* q = e.data();
  std::vector<std::pair<int, float>> sims;
  const float nq = std::sqrt(row_dot(q, q));
  for (int i = 0; i < num_candidates; ++i) {
    const float* c = e.data() + static_cast<size_t>(i + 1) * d;
    const float nc = std::sqrt(row_dot(c, c));
    sims.push_back({i, (nq > 0 && nc > 0) ? row_dot(q, c) / (nq * nc) : 0.0f});   // ffi/embedding.rs:1640-1659
  }
  std::stable_sort(sims.begin(), sims.end(), [](const std::pair<int, float>& a, const std::pair<int, float>& b) { return a.second > b.second; });
  const int k = (top_k <= 0 || top_k > num_candidates) ? num_candidates : top_k;
  SimilarityMatch* m = static_cast<SimilarityMatch*>(malloc(sizeof(SimilarityMatch) * k));
  if (!m) return -1;
  for (int i = 0; i < k; ++i) m[i] = SimilarityMatch{sims[i].first, sims[i].second};
  *result = BatchSimilarityResult{m, k, 2, static_cast<float>(now_ms() - t0), false};
  return 0;
}
void free_batch_similarity_result(BatchSimilarityResult* result) {
  if (!result) return;
  free(result->matches);
  result->matches = nullptr;
  result->num_matches = 0;
}
int get_embedding_models_info(EmbeddingModelsInfoResult* result) {
  if (!result) return -1;
  EmbeddingModelInfo* m = static_cast<EmbeddingModelInfo*>(malloc(sizeof(EmbeddingModelInfo)));
  if (!m) { *result = EmbeddingModelsInfoResult{nullptr, 0, true}; return -1; }
  sr_model_info_t info{};
  if (g_mm_embed.ready()) sr_model_info(g_mm_embed.model, &info);
  m[0] = EmbeddingModelInfo{dup_cstr("mmbert"), g_mm_embed.ready(), g_mm_embed.ready() ? info.max_pos : 0,
                            g_mm_embed.ready() ? info.hidden : 768, g_mm_embed.ready() ? dup_cstr(g_mm_embed.dir) : nullptr};
  *result = EmbeddingModelsInfoResult{m, 1, false};
  return 0;
}
void free_embedding_models_info(EmbeddingModelsInfoResult* result) {
  if (!result || !result->models) return;
  for (int i = 0; i < result->num_models; ++i) { free(result->models[i].model_name); free(result->models[i].model_path); }
  free(result->models);
  result->models = nullptr;
  result->num_models = 0;
}

// batch entries (init_lora_unified_classifier ... free_unified_batch_result): abi_unified.h, shared with the ONNX twin
#include "abi_unified.h"

#ifdef SRB_TEST_HOOKS
// ================================================================================================
// host-logic test hooks (include/sr_b200.h): no GPU involved
// ================================================================================================
static std::vector<TokenPred> hook_tokens(const int32_t* pred, const float* conf, const int32_t* offsets, int n) {
  std::vector<TokenPred> toks(static_cast<size_t>(n > 0 ? n : 0));
  for (int i = 0; i < n; ++i) toks[i] = TokenPred{pred[i], conf[i], offsets[2 * i], offsets[2 * i + 1], std::string()};
  return toks;
}
int sr_test_bio_decode(const int32_t* pred, const float* conf, const int32_t* offsets, int n, const char* const* labels,
                       int n_labels, int text_len, int32_t* ent_start, int32_t* ent_end, float* ent_conf, char* types_out,
                       int types_cap, int cap) {
  (void)text_len;   // the candle rules do not clip against the text (traditional/modernbert.rs:1478-1567)
  if (!pred || !conf || !offsets || n < 0 || !labels || n_labels < 0) return -1;
  std::map<int, std::string> id2label;
  for (int i = 0; i < n_labels; ++i) if (labels[i]) id2label[i] = labels[i];
  const std::vector<Entity> ents = bio_decode(hook_tokens(pred, conf, offsets, n), id2label);
  std::string types;
  for (size_t i = 0; i < ents.size() && static_cast<int>(i) < cap; ++i) {
    if (ent_start) ent_start[i] = ents[i].start;
    if (ent_end) ent_end[i] = ents[i].end;
    if (ent_conf) ent_conf[i] = ents[i].conf;
    types += ents[i].type;
    types += '\n';
  }
  if (types_out && types_cap > 0) snprintf(types_out, static_cast<size_t>(types_cap), "%s", types.c_str());
  return static_cast<int>(ents.size());
}
int sr_test_hallucination_spans(const int32_t* pred, const float* conf, const int32_t* offsets, int n, int answer_start,
                                int answer_len, float threshold, int32_t* span_start, int32_t* span_end, float* span_conf,
                                int cap, int* has_hallucination, float* overall_confidence) {
  if (!pred || !conf || !offsets || n < 0) return -1;
  const HallucSummary hs = hallucination_spans(hook_tokens(pred, conf, offsets, n), answer_start, answer_len, threshold);
  for (size_t i = 0; i < hs.spans.size() && static_cast<int>(i) < cap; ++i) {
    if (span_start) span_start[i] = hs.spans[i].start;
    if (span_end) span_end[i] = hs.spans[i].end;
    if (span_conf) span_conf[i] = hs.spans[i].conf;
  }
  // the same summary detect_hallucinations reports (classify.rs:1620-1640)
  if (has_hallucination) *has_hallucination = hs.spans.empty() ? 0 : 1;
  if (overall_confidence)
    *overall_confidence = !hs.spans.empty() ? hs.max_conf
                          : (hs.n_answer > 0 ? 1.0f - static_cast<float>(hs.n_hall) / static_cast<float>(hs.n_answer) : 1.0f);
  return static_cast<int>(hs.spans.size());
}

#endif  // SRB_TEST_HOOKS
// ================================================================================================
// STUBS (out of scope; documented failure values)
// ================================================================================================
bool init_deberta_jailbreak_classifier(const char*, bool) { return false; }
ClassificationResult classify_deberta_jailbreak_text(const char*) { return ClassificationResult{-1, 0.0f}; }
bool init_multimodal_embedding_model(const char*, bool) { return false; }
static int mm_fail(MultiModalEmbeddingResult* r) { if (r) *r = MultiModalEmbeddingResult{nullptr, 0, true, -1, 0.0f}; return -1; }
int multimodal_encode_text(const char*, int, MultiModalEmbeddingResult* r) { return mm_fail(r); }
int multimodal_encode_image(const float*, int, int, int, MultiModalEmbeddingResult* r) { return mm_fail(r); }
int multimodal_encode_audio(const float*, int, int, int, MultiModalEmbeddingResult* r) { return mm_fail(r); }
void free_multimodal_embedding(float* data, int) { free(data); }
void free_generative_classification_result(GenerativeClassificationResult* r) {
  if (!r) return;
  free(r->category_name); free(r->probabilities); free(r->error_message);
  r->category_name = nullptr; r->probabilities = nullptr; r->error_message = nullptr;
}
void free_categories(char** categories, int n) {
  if (!categories) return;
  for (int i = 0; i < n; ++i) free(categories[i]);
  free(categories);
}
int init_qwen3_multi_lora_classifier(const char*) { return -1; }
int load_qwen3_lora_adapter(const char*, const char*) { return -1; }
static int gen_fail(GenerativeClassificationResult* r) {
  if (r) *r = GenerativeClassificationResult{-1, 0.0f, nullptr, nullptr, 0, true, dup_cstr("Qwen3 generative classifier is out of scope of the B200 library")};
  return -1;
}
int classify_with_qwen3_adapter(const char*, const char*, GenerativeClassificationResult* r) { return gen_fail(r); }
int get_qwen3_loaded_adapters(char*** adapters_out, int* num) { if (adapters_out) *adapters_out = nullptr; if (num) *num = 0; return -1; }
int classify_zero_shot_qwen3(const char*, const char**, int, GenerativeClassificationResult* r) { return gen_fail(r); }
int init_qwen3_guard(const char*) { return -1; }
int classify_with_qwen3_guard(const char*, const char*, GuardResult* r) {
  if (r) *r = GuardResult{nullptr, true, dup_cstr("Qwen3Guard is out of scope of the B200 library")};
  return -1;
}
void free_guard_result(GuardResult* r) { if (!r) return; free(r->raw_output); free(r->error_message); r->raw_output = nullptr; r->error_message = nullptr; }
int is_qwen3_guard_initialized(void) { return 0; }
int is_qwen3_multi_lora_initialized(void) { return 0; }
// ================================================================================================
// hallucination detection + NLI (ffi/classify.rs:1459-2040, ffi/init.rs:1483-1574): a ModernBERT token classifier
// over "<context>[ Question: <question>] [SEP] <answer>" and a ModernBERT sequence classifier over
// "<premise> [SEP] <hypothesis>"; the span / severity logic around them is host code.
// ================================================================================================
bool init_hallucination_model(const char* model_path, bool use_cpu) {   // init.rs:1483: a second init returns true
  note_use_cpu(use_cpu);
  return slot_init(g_halluc, model_path, 1, true);
}
bool init_nli_model(const char* model_path, bool use_cpu) {             // init.rs:1522
  note_use_cpu(use_cpu);
  return slot_init(g_nli, model_path, 0, true);
}
bool is_nli_model_initialized(void) { return g_nli.ready(); }

static HallucinationDetectionResult halluc_error(const char* msg) {
  return HallucinationDetectionResult{false, 0.0f, nullptr, 0, true, dup_cstr(msg)};
}
HallucinationDetectionResult detect_hallucinations(const char* context, const char* question, const char* answer, float threshold) {
  if (!context) return halluc_error("Invalid context string");
  if (!question) return halluc_error("Invalid question string");
  if (!answer) return halluc_error("Invalid answer string");
  if (!g_halluc.ready()) return halluc_error("Hallucination detection model not initialized");
  // classify.rs:1520-1531
  std::string full_context = context;
  if (*question) { full_context += " Question: "; full_context += question; }
  const std::string input = full_context + " [SEP] " + answer;
  const int answer_start = static_cast<int>(full_context.size()) + 7;   // " [SEP] ".len()
  const int answer_len = static_cast<int>(strlen(answer));
  std::vector<TokenPred> toks;
  if (!run_tokens(g_halluc, input.c_str(), toks)) return halluc_error("Classification failed: inference error");
  const HallucSummary hs = hallucination_spans(toks, answer_start, answer_len, threshold);
  const std::vector<HallucSpan>& spans = hs.spans;
  const int n_hall = hs.n_hall, n_answer = hs.n_answer;
  const float max_conf = hs.max_conf;
  HallucinationDetectionResult r{!spans.empty(), 1.0f, nullptr, static_cast<int>(spans.size()), false, nullptr};
  if (r.has_hallucination) r.confidence = max_conf;
  else if (n_answer > 0) r.confidence = 1.0f - static_cast<float>(n_hall) / static_cast<float>(n_answer);
  if (!spans.empty()) {
    r.spans = static_cast<HallucinationSpan*>(malloc(sizeof(HallucinationSpan) * spans.size()));
    if (!r.spans) return halluc_error("out of memory");
    for (size_t i = 0; i < spans.size(); ++i)
      r.spans[i] = HallucinationSpan{dup_cstr(std::string(answer + spans[i].start, answer + spans[i].end)), spans[i].start,
                                     spans[i].end, spans[i].conf, dup_cstr("HALLUCINATED")};
  }
  return r;
}

NLIResult classify_nli(const char* premise, const char* hypothesis) {   // classify.rs:1723-1810
  auto fail = [](const char* msg) { return NLIResult{NLI_ERROR, 0.0f, 0.0f, 0.0f, 0.0f, true, dup_cstr(msg)}; };
  if (!premise) return fail("Invalid premise string");
  if (!hypothesis) return fail("Invalid hypothesis string");
  if (!g_nli.ready()) return fail("NLI model not initialized");
  const std::string input = std::string(premise) + " [SEP] " + hypothesis;
  float conf = 0.f;
  const int c = run_seq(g_nli, input.c_str(), &conf, nullptr);
  if (c < 0) return fail("NLI classification failed: inference error");
  const float rest = (1.0f - conf) / 2.0f;   // the reference reports the two other classes as an even split
  NLIResult r{NLI_ERROR, conf, 0.0f, 0.0f, 0.0f, false, nullptr};
  if (c == 0) { r.label = NLI_ENTAILMENT; r.entailment_prob = conf; r.neutral_prob = rest; r.contradiction_prob = rest; }
  else if (c == 1) { r.label = NLI_NEUTRAL; r.entailment_prob = rest; r.neutral_prob = conf; r.contradiction_prob = rest; }
  else if (c == 2) { r.label = NLI_CONTRADICTION; r.entailment_prob = rest; r.neutral_prob = rest; r.contradiction_prob = conf; }
  return r;
}

EnhancedHallucinationDetectionResult detect_hallucinations_with_nli(const char* context, const char* question, const char* answer,
                                                                    float threshold) {   // classify.rs:1840-2040
  auto fail = [](char* msg) { return EnhancedHallucinationDetectionResult{false, 0.0f, nullptr, 0, true, msg}; };
  if (!context) return fail(dup_cstr("Invalid context string"));
  if (!question) return fail(dup_cstr("Invalid question string"));
  if (!answer) return fail(dup_cstr("Invalid answer string"));
  HallucinationDetectionResult h = detect_hallucinations(context, question, answer, threshold);
  if (h.error) return fail(h.error_message);   // the message moves to the caller
  if (!h.has_hallucination || h.num_spans == 0) {
    free_hallucination_detection_result(h);
    return EnhancedHallucinationDetectionResult{false, 1.0f, nullptr, 0, false, nullptr};
  }
  const bool nli = g_nli.ready();
  std::vector<EnhancedHallucinationSpan> out;
  char buf[256];
  for (int i = 0; i < h.num_spans; ++i) {
    const HallucinationSpan& sp = h.spans[i];
    if (!sp.text || !*sp.text) continue;
    NLILabel label = NLI_NEUTRAL;
    float nconf = 0.f;
    int severity = 2;
    if (nli) {
      const std::string premise = std::string(context) + " " + question;
      NLIResult n = classify_nli(premise.c_str(), sp.text);
      if (n.error) {
        snprintf(buf, sizeof buf, "NLI classification failed, based on hallucination detector only");
      } else {
        label = n.label;
        nconf = n.confidence;
        const double pct = static_cast<double>(n.confidence) * 100.0;
        if (n.label == NLI_CONTRADICTION) { severity = 4; snprintf(buf, sizeof buf, "CONTRADICTION: This claim directly conflicts with the provided context (confidence: %.1f%%)", pct); }
        else if (n.label == NLI_NEUTRAL) { severity = 2; snprintf(buf, sizeof buf, "FABRICATION: This claim is not supported by the provided context (confidence: %.1f%%)", pct); }
        else if (n.label == NLI_ENTAILMENT) { severity = 1; snprintf(buf, sizeof buf, "UNCERTAIN: Hallucination detector flagged this but NLI suggests it may be supported (confidence: %.1f%%)", pct); }
        else { severity = 2; snprintf(buf, sizeof buf, "Unable to determine relationship with context"); }
      }
      free_nli_result(n);
    } else {
      severity = sp.confidence > 0.8f ? 3 : 2;
      snprintf(buf, sizeof buf, "Unsupported claim detected (confidence: %.1f%%)", static_cast<double>(sp.confidence) * 100.0);
    }
    out.push_back(EnhancedHallucinationSpan{dup_cstr(sp.text), sp.start, sp.end, sp.confidence, label, nconf, severity, dup_cstr(buf)});
  }
  free_hallucination_detection_result(h);
  EnhancedHallucinationDetectionResult r{!out.empty(), 0.0f, nullptr, static_cast<int>(out.size()), false, nullptr};
  for (const auto& e : out) r.confidence = std::max(r.confidence, std::max(e.hallucination_confidence, e.nli_confidence));
  if (!out.empty()) {
    r.spans = static_cast<EnhancedHallucinationSpan*>(malloc(sizeof(EnhancedHallucinationSpan) * out.size()));
    if (r.spans) memcpy(r.spans, out.data(), sizeof(EnhancedHallucinationSpan) * out.size());
  }
  return r;
}
void free_hallucination_detection_result(HallucinationDetectionResult r) {
  for (int i = 0; i < r.num_spans && r.spans; ++i) { free(r.spans[i].text); free(r.spans[i].label); }
  free(r.spans); free(r.error_message);
}
void free_enhanced_hallucination_detection_result(EnhancedHallucinationDetectionResult r) {
  for (int i = 0; i < r.num_spans && r.spans; ++i) { free(r.spans[i].text); free(r.spans[i].explanation); }
  free(r.spans); free(r.error_message);
}
void free_nli_result(NLIResult r) { free(r.error_message); }
void* candle_mlp_new(void) { return nullptr; }
void* candle_mlp_new_with_device(int) { return nullptr; }
void* candle_mlp_new_with_device_and_dtype(int, int) { return nullptr; }
void candle_mlp_free(void*) {}
char* candle_mlp_select(void*, double*, size_t) { return nullptr; }
int candle_mlp_is_trained(void*) { return 0; }
char* candle_mlp_to_json(void*) { return nullptr; }
void* candle_mlp_from_json(char*) { return nullptr; }
void* candle_mlp_from_json_with_device(char*, int) { return nullptr; }
void* candle_mlp_from_json_with_device_and_dtype(char*, int, int) { return nullptr; }
void candle_mlp_free_string(char* p) { free(p); }

}  // extern "C"
