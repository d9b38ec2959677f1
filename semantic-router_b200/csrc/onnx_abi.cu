// Drop-in C ABI #2 (include/onnx_semantic_router.h): the symbol table onnx-binding/semantic-router.go links
// (-lonnx_semantic_router), implemented over the same CUDA engine as abi.cu.  Replaces
// onnx-binding/src/ffi/{classification,embedding,memory,multimodal}.rs and the ONNX Runtime sessions behind them
// (model_architectures/classification/mmbert_classifier.rs, embedding/mmbert_embedding.rs).
//
// Differences that matter for parity (each is the ONNX side's behaviour, not candle's):
//   * named classifier slots in a map; re-init replaces the entry (classification.rs:183,245)
//   * the head is the exported HF graph: pooling per config "classifier_pooling", erf GELU, LayerNorm eps = norm_eps
//     -> every model loaded here runs with sr_model_set_head_flavor(m, 1)
//   * softmax on the host side of the reference + max_by (last max wins, NaN -> Less) (mmbert_classifier.rs:796-830)
//   * BIO decode ignores an I- tag whose type differs from the open entity (mmbert_classifier.rs:1006-1019),
//     where candle's closes it
//   * classify_batch / get_embeddings_batch / calculate_similarity_batch are TRUE batches: one packed varlen pass
#include "../../include/onnx_semantic_router.h"
#include "../../include/sr_b200_testhooks.h"
#include "abi_core.h"

#define SRB_ABI_HEAD_FLAVOR 1   // the exported HF graph's head (sr_b200.h: sr_model_set_head_flavor)

#include <memory>

namespace {

struct NamedSlot {
  Slot s;
  ~NamedSlot() { s.destroy(); }   // every replica's model and the tokenizer
};
using SlotPtr = std::shared_ptr<NamedSlot>;

std::mutex g_reg_mu;
std::map<std::string, SlotPtr> g_seq, g_tok;
SlotPtr g_embed;

SlotPtr load_slot(const char* dir, int token_level) {
  SlotPtr p = std::make_shared<NamedSlot>();
  if (!slot_init(p->s, dir, token_level, true)) return nullptr;
  for (auto& rep : p->s.reps) sr_model_set_head_flavor(rep->model, 1);
  return p;
}
SlotPtr find(std::map<std::string, SlotPtr>& reg, const char* name) {
  std::lock_guard<std::mutex> lk(g_reg_mu);
  auto it = reg.find(name);
  return it == reg.end() ? nullptr : it->second;
}
SlotPtr embed_slot() {
  std::lock_guard<std::mutex> lk(g_reg_mu);
  return g_embed;
}

std::string label_for(const Slot& s, int id) {  // MmBertClassifierConfig::get_label (mmbert_classifier.rs:155-160)
  auto it = s.id2label.find(id);
  return it == s.id2label.end() ? "LABEL_" + std::to_string(id) : it->second;
}
// probs.iter().enumerate().max_by(|a, b| a.partial_cmp(b).unwrap_or(Less)): a later element replaces the running
// maximum unless the maximum is strictly greater (mmbert_classifier.rs:809-813)
int argmax_max_by(const float* p, int n) {
  int best = 0;
  for (int c = 1; c < n; ++c)
    if (!(p[best] > p[c])) best = c;
  return best;
}
ClassificationResultFFI cls_error() { return ClassificationResultFFI{nullptr, -1, 0.0f, 0, nullptr, 0.0f, true}; }
EmbeddingResult emb_error() { return EmbeddingResult{nullptr, 0, true, -1, 0, 0.0f}; }
PIIResultFFI pii_error(const std::string& msg) { return PIIResultFFI{nullptr, 0, 0.0f, true, dup_cstr(msg)}; }

void fill_cls(const Slot& s, const float* probs, int C, float ms, ClassificationResultFFI* out) {
  const int id = argmax_max_by(probs, C);
  float* pr = static_cast<float*>(malloc(sizeof(float) * C));
  if (pr) memcpy(pr, probs, sizeof(float) * C);
  *out = ClassificationResultFFI{dup_cstr(label_for(s, id)), id, probs[id], C, pr, ms, false};
}

float cosine(const float* a, const float* b, int d) {  // ffi/embedding.rs:405-416 / :541-560
  float dp = 0.f, na = 0.f, nb = 0.f;
  for (int i = 0; i < d; ++i) { dp += a[i] * b[i]; na += a[i] * a[i]; nb += b[i] * b[i]; }
  na = sqrtf(na);
  nb = sqrtf(nb);
  return (na > 0.f && nb > 0.f) ? dp / (na * nb) : 0.f;
}

// mmbert_classifier.rs:952-1050
struct OxEntity {
  std::string type;
  int start, end;
  float conf;
};
std::vector<OxEntity> bio_decode_onnx(const Slot& s, const std::vector<TokenPred>& toks, int text_len) {
  std::vector<OxEntity> out;
  bool open = false;
  OxEntity cur{};
  auto flush = [&] {
    if (open && cur.start < text_len && cur.end <= text_len) out.push_back(cur);
    open = false;
  };
  for (const TokenPred& t : toks) {
    if (t.start == 0 && t.end == 0) continue;  // special token
    const std::string label = label_for(s, t.pred);
    if (label.rfind("B-", 0) == 0) {
      flush();
      cur = OxEntity{label.substr(2), t.start, t.end, t.conf};
      open = true;
    } else if (label.rfind("I-", 0) == 0) {
      if (open && cur.type == label.substr(2)) {
        cur.end = t.end;
        cur.conf = (cur.conf + t.conf) / 2.0f;
      }
    } else {
      flush();
    }
  }
  flush();
  return out;
}

// CStr::to_str() of the reference: reject malformed UTF-8 (and null) before anything else
bool valid_utf8(const char* s) {
  if (!s) return false;
  const unsigned char* p = reinterpret_cast<const unsigned char*>(s);
  while (*p) {
    int n;
    unsigned cp;
    if (*p < 0x80) { ++p; continue; }
    else if ((*p & 0xE0) == 0xC0) { n = 1; cp = *p & 0x1F; }
    else if ((*p & 0xF0) == 0xE0) { n = 2; cp = *p & 0x0F; }
    else if ((*p & 0xF8) == 0xF0) { n = 3; cp = *p & 0x07; }
    else return false;
    for (int i = 1; i <= n; ++i) {
      if ((p[i] & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (p[i] & 0x3F);
    }
    static const unsigned kMin[4] = {0, 0x80, 0x800, 0x10000};
    if (cp < kMin[n] || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
    p += n + 1;
  }
  return true;
}

}  // namespace

extern "C" {

#ifdef SRB_TEST_HOOKS
// host-logic test hooks (include/sr_b200_testhooks.h): no GPU involved.  This library decodes with the ONNX binding's rules
// (mmbert_classifier.rs:952-1050): a foreign I- tag leaves the entity open, spans are clipped against the text.
int sr_test_bio_decode(const int32_t* pred, const float* conf, const int32_t* offsets, int n, const char* const* labels,
                       int n_labels, int text_len, int32_t* ent_start, int32_t* ent_end, float* ent_conf, char* types_out,
                       int types_cap, int cap) {
  if (!pred || !conf || !offsets || n < 0 || !labels || n_labels < 0) return -1;
  Slot tmp;
  for (int i = 0; i < n_labels; ++i) if (labels[i]) tmp.id2label[i] = labels[i];
  std::vector<TokenPred> toks(static_cast<size_t>(n));
  for (int i = 0; i < n; ++i) toks[i] = TokenPred{pred[i], conf[i], offsets[2 * i], offsets[2 * i + 1], std::string()};
  const std::vector<OxEntity> ents = bio_decode_onnx(tmp, toks, text_len);
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
int sr_test_hallucination_spans(const int32_t*, const float*, const int32_t*, int, int, int, float, int32_t*, int32_t*, float*,
                                int, int*, float*) {
  return -1;   // the ONNX binding has no hallucination detector
}

#endif  // SRB_TEST_HOOKS

// ================================================================================================
// classification
// ================================================================================================
static bool init_named(std::map<std::string, SlotPtr>& reg, const char* name, const char* path, int token_level) {
  if (!name || !path) {
    fprintf(stderr, "[srb200] init_%s_classifier: null argument\n", token_level ? "token" : "sequence");
    return false;
  }
  SlotPtr p = load_slot(path, token_level);
  if (!p) return false;
  std::lock_guard<std::mutex> lk(g_reg_mu);
  reg[name] = p;  // HashMap::insert: replaces
  return true;
}
bool init_sequence_classifier(const char* name, const char* model_path, bool use_gpu) {
  note_use_cpu(!use_gpu);
  return init_named(g_seq, name, model_path, 0);
}
bool init_token_classifier(const char* name, const char* model_path, bool use_gpu) {
  note_use_cpu(!use_gpu);
  return init_named(g_tok, name, model_path, 1);
}
bool is_classifier_loaded(const char* name) {
  if (!name) return false;
  std::lock_guard<std::mutex> lk(g_reg_mu);
  return g_seq.count(name) || g_tok.count(name);
}

int classify_text(const char* classifier_name, const char* text, ClassificationResultFFI* result) {
  if (!classifier_name || !text || !result) return -1;
  *result = cls_error();
  if (!valid_utf8(classifier_name) || !valid_utf8(text)) return -1;
  SlotPtr p = find(g_seq, classifier_name);
  if (!p) {
    fprintf(stderr, "[srb200] classify_text: classifier '%s' not found\n", classifier_name);
    return -1;
  }
  const double t0 = now_ms();
  std::vector<float> probs;
  float conf = 0.f;
  if (run_seq(p->s, text, &conf, &probs) < 0 || probs.empty()) return -1;  // rides the slot's coalesced batches
  fill_cls(p->s, probs.data(), static_cast<int>(probs.size()), static_cast<float>(now_ms() - t0), result);
  return 0;
}

int classify_batch(const char* classifier_name, const char** texts, int num_texts, ClassificationResultFFI* results) {
  if (!classifier_name || !texts || !results || num_texts <= 0) return -1;
  if (!valid_utf8(classifier_name)) return -1;
  for (int i = 0; i < num_texts; ++i)
    if (!valid_utf8(texts[i])) return -1;
  SlotPtr p = find(g_seq, classifier_name);
  if (!p) {
    fprintf(stderr, "[srb200] classify_batch: classifier '%s' not found\n", classifier_name);
    return -1;
  }
  const double t0 = now_ms();
  std::vector<float> probs;
  int C = 0;
  if (!classify_packed(p->s, texts, num_texts, probs, C)) {
    for (int i = 0; i < num_texts; ++i) results[i] = cls_error();
    return -1;
  }
  const float per_text = static_cast<float>(now_ms() - t0) / static_cast<float>(num_texts);
  for (int i = 0; i < num_texts; ++i) fill_cls(p->s, probs.data() + static_cast<size_t>(i) * C, C, per_text, &results[i]);
  return 0;
}

int detect_pii(const char* classifier_name, const char* text, PIIResultFFI* result) {
  if (!result) return -1;
  if (!classifier_name || !text) {
    *result = pii_error("null pointer in detect_pii arguments");
    return -1;
  }
  if (!valid_utf8(classifier_name)) { *result = pii_error("invalid UTF-8 in classifier_name"); return -1; }
  if (!valid_utf8(text)) { *result = pii_error("invalid UTF-8 in text"); return -1; }
  SlotPtr p = find(g_tok, classifier_name);
  if (!p) {
    *result = pii_error(std::string("PII classifier '") + classifier_name + "' not found");
    return -1;
  }
  const double t0 = now_ms();
  std::vector<TokenPred> toks;
  if (!run_tokens(p->s, text, toks)) {
    *result = pii_error("PII detection failed: inference error");
    return -1;
  }
  const std::vector<OxEntity> ents = bio_decode_onnx(p->s, toks, static_cast<int>(strlen(text)));
  PIIResultFFI r{nullptr, static_cast<int>(ents.size()), static_cast<float>(now_ms() - t0), false, nullptr};
  if (!ents.empty()) {
    r.entities = static_cast<PIIEntityFFI*>(malloc(sizeof(PIIEntityFFI) * ents.size()));
    if (!r.entities) { *result = pii_error("out of memory"); return -1; }
    for (size_t i = 0; i < ents.size(); ++i) {
      const OxEntity& e = ents[i];
      const std::string span = e.start < e.end ? std::string(text + e.start, text + e.end) : std::string();
      r.entities[i] = PIIEntityFFI{dup_cstr(span), dup_cstr(e.type), e.start, e.end, e.conf};
    }
  }
  *result = r;
  return 0;
}

void free_classification_result(ClassificationResultFFI* result) {
  if (!result) return;
  free(result->label);
  result->label = nullptr;
  free(result->probabilities);
  result->probabilities = nullptr;
}
void free_pii_result(PIIResultFFI* result) {
  if (!result) return;
  if (result->entities) {
    for (int i = 0; i < result->num_entities; ++i) {
      free(result->entities[i].text);
      free(result->entities[i].entity_type);
    }
    free(result->entities);
    result->entities = nullptr;
  }
  free(result->error_message);
  result->error_message = nullptr;
}

// ================================================================================================
// embeddings
// ================================================================================================
bool init_mmbert_embedding_model(const char* model_path, bool use_cpu) {
  note_use_cpu(use_cpu);
  if (!model_path || !*model_path) return false;
  {
    std::lock_guard<std::mutex> lk(g_reg_mu);
    if (g_embed) return true;  // "already initialized" (ffi/embedding.rs:55-58)
  }
  SlotPtr p = load_slot(model_path, -2);
  if (!p) return false;
  std::lock_guard<std::mutex> lk(g_reg_mu);
  if (!g_embed) g_embed = p;
  return true;
}
bool is_mmbert_model_initialized(void) { return embed_slot() != nullptr; }

int get_embedding_2d_matryoshka(const char* text, int target_layer, int target_dim, EmbeddingResult* result) {
  if (!text || !result) return -1;
  *result = emb_error();
  if (!valid_utf8(text)) return -1;
  SlotPtr p = embed_slot();
  if (!p) {
    fprintf(stderr, "[srb200] get_embedding: mmBERT model not initialized\n");
    return -1;
  }
  const double t0 = now_ms();
  std::vector<float> e;
  int d = 0;
  if (!embed_packed(p->s, &text, 1, p->s.max_pos, target_layer, target_dim, e, d)) return -1;
  *result = EmbeddingResult{dup_floats(e), d, false, 0, word_count(text), static_cast<float>(now_ms() - t0)};
  return 0;
}
int get_embedding(const char* text, EmbeddingResult* result) { return get_embedding_2d_matryoshka(text, 0, 0, result); }
int get_embedding_with_dim(const char* text, int target_dim, EmbeddingResult* result) {
  return get_embedding_2d_matryoshka(text, 0, target_dim, result);
}

int get_embeddings_batch(const char** texts, int num_texts, int target_layer, int target_dim, EmbeddingResult* results) {
  if (!texts || !results || num_texts <= 0) return -1;
  for (int i = 0; i < num_texts; ++i)
    if (!valid_utf8(texts[i])) return -1;
  SlotPtr p = embed_slot();
  if (!p) return -1;
  const double t0 = now_ms();
  std::vector<float> e;
  int d = 0;
  if (!embed_packed(p->s, texts, num_texts, p->s.max_pos, target_layer, target_dim, e, d)) {
    for (int i = 0; i < num_texts; ++i) results[i] = emb_error();
    return -1;
  }
  const float per_text = static_cast<float>(now_ms() - t0) / static_cast<float>(num_texts);
  for (int i = 0; i < num_texts; ++i) {
    float* data = static_cast<float*>(malloc(sizeof(float) * d));
    if (data) memcpy(data, e.data() + static_cast<size_t>(i) * d, sizeof(float) * d);
    results[i] = EmbeddingResult{data, d, false, 0, word_count(texts[i]), per_text};
  }
  return 0;
}

int calculate_embedding_similarity(const char* text1, const char* text2, int target_layer, int target_dim,
                                   EmbeddingSimilarityResult* result) {
  if (!text1 || !text2 || !result) return -1;
  *result = EmbeddingSimilarityResult{-1.0f, -1, 0.0f, true};
  if (!valid_utf8(text1) || !valid_utf8(text2)) return -1;
  SlotPtr p = embed_slot();
  if (!p) return -1;
  const double t0 = now_ms();
  const char* both[2] = {text1, text2};
  std::vector<float> e;
  int d = 0;
  if (!embed_packed(p->s, both, 2, p->s.max_pos, target_layer, target_dim, e, d)) return -1;
  *result = EmbeddingSimilarityResult{cosine(e.data(), e.data() + d, d), 0, static_cast<float>(now_ms() - t0), false};
  return 0;
}

int calculate_similarity_batch(const char* query, const char** candidates, int num_candidates, int top_k, int target_layer,
                               int target_dim, BatchSimilarityResult* result) {
  if (!query || !candidates || !result || num_candidates <= 0) return -1;
  *result = BatchSimilarityResult{nullptr, 0, -1, 0.0f, true};
  if (!valid_utf8(query)) return -1;
  std::vector<const char*> all{query};
  for (int i = 0; i < num_candidates; ++i) {
    if (!valid_utf8(candidates[i])) return -1;
    all.push_back(candidates[i]);
  }
  SlotPtr p = embed_slot();
  if (!p) return -1;
  const double t0 = now_ms();
  std::vector<float> e;
  int d = 0;
  if (!embed_packed(p->s, all.data(), static_cast<int>(all.size()), p->s.max_pos, target_layer, target_dim, e, d)) return -1;
  std::vector<std::pair<int, float>> sims(num_candidates);
  for (int i = 0; i < num_candidates; ++i) sims[i] = {i, cosine(e.data(), e.data() + static_cast<size_t>(i + 1) * d, d)};
  // sort_by(|a, b| b.1.partial_cmp(&a.1).unwrap_or(Equal)): stable, descending
  std::stable_sort(sims.begin(), sims.end(), [](const auto& a, const auto& b) { return a.second > b.second; });
  const int k = (top_k <= 0 || top_k > num_candidates) ? num_candidates : top_k;
  SimilarityMatch* m = static_cast<SimilarityMatch*>(malloc(sizeof(SimilarityMatch) * k));
  if (!m) return -1;
  for (int i = 0; i < k; ++i) m[i] = SimilarityMatch{sims[i].first, sims[i].second};
  *result = BatchSimilarityResult{m, k, 0, static_cast<float>(now_ms() - t0), false};
  return 0;
}

int get_embedding_models_info(EmbeddingModelsInfoResult* result) {
  if (!result) return -1;
  EmbeddingModelInfo* mi = static_cast<EmbeddingModelInfo*>(malloc(sizeof(EmbeddingModelInfo)));
  if (!mi) { *result = EmbeddingModelsInfoResult{nullptr, 0, true}; return -1; }
  SlotPtr p = embed_slot();
  if (p) {
    sr_model_info_t info;
    sr_model_info(p->s.model, &info);
    std::string layers;  // every depth is an exit here (no per-layer ONNX sessions needed)
    for (int l = 1; l <= info.layers; ++l) layers += (l > 1 ? "," : "") + std::to_string(l);
    const std::string desc = "MmBertEmbeddingModel(path=" + p->s.dir + ", hidden_size=" + std::to_string(info.hidden) +
                             ", layers=" + std::to_string(info.layers) + ", layer_exit=true, backend=b200)";
    *mi = EmbeddingModelInfo{dup_cstr("mmbert"), true, info.max_pos, info.hidden, dup_cstr(desc), true, dup_cstr(layers)};
  } else {
    *mi = EmbeddingModelInfo{dup_cstr("mmbert"), false, 0, 0, dup_cstr(""), false, dup_cstr("")};
  }
  *result = EmbeddingModelsInfoResult{mi, 1, false};
  return 0;
}

void free_embedding(float* data, int) { free(data); }
void free_batch_similarity_result(BatchSimilarityResult* result) {
  if (!result) return;
  free(result->matches);
  result->matches = nullptr;
  result->num_matches = 0;
}
void free_embedding_models_info(EmbeddingModelsInfoResult* result) {
  if (!result || !result->models) return;
  for (int i = 0; i < result->num_models; ++i) {
    free(result->models[i].model_name);
    free(result->models[i].model_path);
    free(result->models[i].available_layers);
  }
  free(result->models);
  result->models = nullptr;
  result->num_models = 0;
}

// ================================================================================================
// multi-modal embedding: outside the encoder-classifier path (SURVEY section 8 "out of scope"); the symbols exist
// so the Go package links, and fail the way the reference does when its model is not loaded
// ================================================================================================
static int mm_fail(MultiModalEmbeddingResult* r) {
  if (r) *r = MultiModalEmbeddingResult{nullptr, 0, true, -1, 0.0f};
  return -1;
}
bool init_multimodal_embedding_model(const char*, bool) {
  fprintf(stderr, "[srb200] init_multimodal_embedding_model: not on the B200 hot path\n");
  return false;
}
int multimodal_encode_text(const char*, int, MultiModalEmbeddingResult* r) { return mm_fail(r); }
int multimodal_encode_image(const float*, int, int, int, MultiModalEmbeddingResult* r) { return mm_fail(r); }
int multimodal_encode_audio(const float*, int, int, int, MultiModalEmbeddingResult* r) { return mm_fail(r); }
void free_multimodal_embedding(float* data, int) { free(data); }

// ================================================================================================
// unified / LoRA batch entries that pkg/classification/unified_classifier.go:66-81 links under -tags=onnx
// ================================================================================================
#include "abi_unified.h"

}  // extern "C"
