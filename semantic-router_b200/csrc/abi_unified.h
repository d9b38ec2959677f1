// The seven entries of pkg/classification/unified_classifier.go:66-81 (include/unified_classifier_abi.h), shared by the
// two drop-in libraries: abi.cu (candle twin) and onnx_abi.cu (ONNX twin; the reference's own ONNX build only stubs
// them, onnx-binding/src/ffi/unified.rs:107-200, so a `-tags=onnx` router loses its batch classifier -- here it does
// not).  Included INSIDE the including file's extern "C" block, after abi_core.h; SRB_ABI_HEAD_FLAVOR picks the head
// semantics of the slots loaded here (0 candle, 1 the HF graph an ONNX export carries).
#pragma once

namespace {
Slot g_lora_intent, g_lora_pii, g_lora_security;
// The three LoRA tasks as ONE grouped model when their checkpoints share one encoder shape (sr_b200.h:
// sr_model_load_lora_shared for unmerged adapters over one base, sr_model_load_grouped for merged or fine-tuned
// checkpoints): a batch then runs once through the encoder instead of three times, with the three-slot results.
// SR_B200_LORA_SHARED=0 keeps the three slots; so does anything the grouped loaders refuse.
Slot g_lora_shared;
std::map<int, std::string> g_lora_labels[3];
Slot g_unified;  // shared encoder + 3 heads (legacy unified classifier)
int g_unified_heads[3] = {-1, -1, -1};
std::vector<std::string> g_unified_labels[3];
// A grouped model tokenises a text once for all its tasks and runs one pooler mode (lora_config.json, slot_init): it
// answers like separate slots only where those would tokenise and pool alike -- the same tokenizer.json bytes, and
// lora_config.json in every directory or in none.
bool same_serving_files(const char* const* dirs, int n) {
  auto slurp = [](const std::string& path, std::string& out) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    char buf[65536];
    size_t k;
    out.clear();
    while ((k = fread(buf, 1, sizeof buf, f)) > 0) out.append(buf, k);
    fclose(f);
    return true;
  };
  std::string first, other;
  const bool lora0 = file_exists(std::string(dirs[0]) + "/lora_config.json");
  if (!slurp(std::string(dirs[0]) + "/tokenizer.json", first)) return false;
  for (int i = 1; i < n; ++i)
    if (file_exists(std::string(dirs[i]) + "/lora_config.json") != lora0 ||
        !slurp(std::string(dirs[i]) + "/tokenizer.json", other) || other != first)
      return false;
  return true;
}
bool unified_slot_init(Slot& s, const char* dir, int token_level) {
  if (!slot_init(s, dir, token_level, true)) return false;
  if (SRB_ABI_HEAD_FLAVOR != 0)
    for (auto& rep : s.reps) sr_model_set_head_flavor(rep->model, SRB_ABI_HEAD_FLAVOR);
  return true;
}
}  // namespace

void free_cstring(char* s) { free(s); }

// ================================================================================================
// batch entries
// ================================================================================================
bool init_lora_unified_classifier(const char* intent, const char* pii, const char* security, const char* architecture, bool use_cpu) {
  (void)architecture;
  note_use_cpu(use_cpu);
  if (!intent || !pii || !security) return false;
  if (g_lora_shared.ready()) return true;
  static const bool shared_on = [] { const char* e = getenv("SR_B200_LORA_SHARED"); return !(e && e[0] == '0'); }();
  const bool fresh = !g_lora_intent.ready() && !g_lora_pii.ready() && !g_lora_security.ready();
  if (shared_on && fresh) {
    const char* dirs[3] = {intent, pii, security};
    const int token_level[3] = {0, 1, 0};
    const bool adapters = sr_checkpoint_has_adapters(intent) == 1 && sr_checkpoint_has_adapters(pii) == 1 &&
                          sr_checkpoint_has_adapters(security) == 1;
    const bool same_files = same_serving_files(dirs, 3);
    const bool ok = slot_init(g_lora_shared, intent, -2, true, [&](int device, sr_model** out) {
      if (adapters && sr_model_load_lora_shared(dirs, token_level, 3, device, out) == 0) return 0;
      return same_files ? sr_model_load_grouped(dirs, token_level, 3, device, out) : -1;
    });
    if (ok) {
      if (SRB_ABI_HEAD_FLAVOR != 0)
        for (auto& rep : g_lora_shared.reps) sr_model_set_head_flavor(rep->model, SRB_ABI_HEAD_FLAVOR);
      for (int t = 0; t < 3; ++t) {
        g_lora_labels[t].clear();
        load_id2label(std::string(dirs[t]) + "/config.json", g_lora_labels[t]);
      }
      return true;
    }
    // different encoder shapes, architectures (or anything else the grouped loaders refuse): three independent slots
  }
  const bool a = unified_slot_init(g_lora_intent, intent, 0);
  const bool b = unified_slot_init(g_lora_pii, pii, 1);
  const bool c = unified_slot_init(g_lora_security, security, 0);
  if (a && b && c) {
    g_lora_labels[0] = g_lora_intent.id2label;
    g_lora_labels[1] = g_lora_pii.id2label;
    g_lora_labels[2] = g_lora_security.id2label;
  }
  return a && b && c;
}

static std::string lora_label(int task, int cls) {
  auto it = g_lora_labels[task].find(cls);
  return it == g_lora_labels[task].end() ? "LABEL_" + std::to_string(cls) : it->second;
}

// intent classes / confidences, per-token PII predictions, security classes / confidences of `n` texts from ONE encoder
// pass per piece over the grouped model (three copies of the rows, each with its task's weights)
static bool lora_shared_packed(const char* const* texts, int n, std::vector<int32_t>& icls, std::vector<float>& iconf,
                               std::vector<std::vector<TokenPred>>& toks_out, std::vector<int32_t>& scls, std::vector<float>& sconf) {
  Slot& s = g_lora_shared;
  const std::vector<Tokens> toks = tokenize_many(s, texts, n, s.max_len);
  for (const Tokens& t : toks)
    if (t.ids.empty()) return false;
  icls.assign(n, -1); iconf.assign(n, 0.f); scls.assign(n, -1); sconf.assign(n, 0.f);
  toks_out.assign(n, {});
  return for_pieces(s, toks, [&](sr_model* m, int first, int b, std::vector<int32_t>& ids, std::vector<int32_t>& cu) {
    std::vector<int32_t> pred(ids.size());
    std::vector<float> pconf(ids.size());
    int32_t* cp[3] = {icls.data() + first, pred.data(), scls.data() + first};
    float* fp[3] = {iconf.data() + first, pconf.data(), sconf.data() + first};
    if (sr_classify_lora_shared_ids(m, ids.data(), cu.data(), b, s.pooler_mode, nullptr, cp, fp) != 0) return false;
    for (int i = 0; i < b; ++i) {
      const Tokens& t = toks[first + i];
      std::vector<TokenPred>& o = toks_out[first + i];
      o.resize(t.ids.size());
      for (size_t k = 0; k < t.ids.size(); ++k)
        o[k] = {pred[cu[i] + k], pconf[cu[i] + k], t.offsets[k].first, t.offsets[k].second, t.tokens[k]};
    }
    return true;
  }, 3);
}

LoRABatchResult classify_batch_with_lora(const char** texts, int num_texts) {
  LoRABatchResult none{nullptr, nullptr, nullptr, 0, 0.0f};
  const bool shared = g_lora_shared.ready();
  if (!texts || num_texts <= 0 || (!shared && (!g_lora_intent.ready() || !g_lora_pii.ready() || !g_lora_security.ready()))) return none;
  LoRABatchResult r{static_cast<LoRAIntentResult*>(calloc(num_texts, sizeof(LoRAIntentResult))),
                    static_cast<LoRAPIIResult*>(calloc(num_texts, sizeof(LoRAPIIResult))),
                    static_cast<LoRASecurityResult*>(calloc(num_texts, sizeof(LoRASecurityResult))), num_texts, 0.0f};
  if (!r.intent_results || !r.pii_results || !r.security_results) { free(r.intent_results); free(r.pii_results); free(r.security_results); return none; }
  std::vector<float> ip, sp, iconf, sconf;
  std::vector<int32_t> icls, scls;
  std::vector<std::vector<TokenPred>> toks;
  int iC = 0, sC = 0;
  bool iok, pok, sok;
  if (shared) {
    // one packed varlen pass per piece, the three tasks as three copies of the rows in ONE grouped model (abi_unified.h top)
    iok = pok = sok = lora_shared_packed(texts, num_texts, icls, iconf, toks, scls, sconf);
  } else {
    // three packed varlen passes (intent, PII tokens, security) over the whole batch -- the reference's
    // parallel engine runs the three tasks over the batch as well (classifiers/lora/parallel_engine.rs)
    iok = classify_packed(g_lora_intent, texts, num_texts, ip, iC, &icls, &iconf);
    pok = tokens_packed(g_lora_pii, texts, num_texts, toks);
    sok = classify_packed(g_lora_security, texts, num_texts, sp, sC, &scls, &sconf);
  }
  float total = 0.f;
  for (int i = 0; i < num_texts; ++i) {
    const int ic = iok ? icls[i] : -1;
    r.intent_results[i] = LoRAIntentResult{dup_cstr(ic >= 0 ? lora_label(0, ic) : "unknown"), ic >= 0 ? iconf[i] : 0.f};
    total += r.intent_results[i].confidence;
    // PII (classifiers/lora/pii_lora.rs:103-160): per-token classes, class 0 = "O"
    std::vector<std::string> types;
    float pii_sum = 0.f, o_sum = 0.f;
    int pii_n = 0, o_n = 0;
    if (pok)
      for (const auto& t : toks[i]) {
        if (t.pred > 0) {
          pii_sum += t.conf; ++pii_n;
          const std::string ty = lora_label(1, t.pred);
          if (std::find(types.begin(), types.end(), ty) == types.end()) types.push_back(ty);
        } else { o_sum += t.conf; ++o_n; }
      }
    LoRAPIIResult& p = r.pii_results[i];
    p.has_pii = pii_n > 0;
    p.num_pii_types = static_cast<int>(types.size());
    p.pii_types = types.empty() ? nullptr : static_cast<char**>(malloc(sizeof(char*) * types.size()));
    for (size_t k = 0; k < types.size() && p.pii_types; ++k) p.pii_types[k] = dup_cstr(types[k]);
    p.confidence = pii_n > 0 ? pii_sum / pii_n : (o_n > 0 ? o_sum / o_n : 0.f);
    total += p.confidence;
    // security (classifiers/lora/security_lora.rs:168-205)
    const int sc = sok ? scls[i] : -1;
    std::string threat = sc >= 0 ? lora_label(2, sc) : "unknown";
    std::string low = threat;
    for (auto& ch : low) ch = static_cast<char>(tolower(static_cast<unsigned char>(ch)));
    const bool is_threat = sc >= 0 && low.find("safe") == std::string::npos && low.find("benign") == std::string::npos &&
                           low.find("no_threat") == std::string::npos;
    r.security_results[i] = LoRASecurityResult{is_threat, dup_cstr(threat), sc >= 0 ? sconf[i] : 0.f};
    total += r.security_results[i].confidence;
  }
  r.avg_confidence = total / (3.0f * num_texts);
  return r;
}
void free_lora_batch_result(LoRABatchResult result) {
  for (int i = 0; i < result.batch_size; ++i) {
    if (result.intent_results) free(result.intent_results[i].category);
    if (result.pii_results) {
      for (int k = 0; k < result.pii_results[i].num_pii_types; ++k) free(result.pii_results[i].pii_types[k]);
      free(result.pii_results[i].pii_types);
    }
    if (result.security_results) free(result.security_results[i].threat_type);
  }
  free(result.intent_results);
  free(result.pii_results);
  free(result.security_results);
}

// Legacy unified classifier: ONE shared encoder + three heads (done properly, unlike ffi/init.rs:1076-1194 which
// ignores the head paths and replicates one aggregate result -- documented divergence, SURVEY section 0 fact 4).
bool init_unified_classifier_c(const char* modernbert_path, const char* intent_head_path, const char* pii_head_path,
                               const char* security_head_path, const char** intent_labels, int intent_labels_count,
                               const char** pii_labels, int pii_labels_count, const char** security_labels,
                               int security_labels_count, bool use_cpu) {
  note_use_cpu(use_cpu);
  if (!unified_slot_init(g_unified, modernbert_path, -2)) return false;
  std::lock_guard<std::mutex> lk(g_unified.mu);
  if (g_unified_heads[0] >= 0) return true;
  const char* paths[3] = {intent_head_path, pii_head_path, security_head_path};
  const int tok_level[3] = {0, 1, 0};
  for (int i = 0; i < 3; ++i) {
    if (!paths[i]) return false;
    int h = -1;
    for (auto& rep : g_unified.reps) {   // the same head ids on every replica (heads are appended in this order)
      const int hr = sr_model_add_head(rep->model, paths[i], tok_level[i]);
      if (hr < 0 || (h >= 0 && hr != h)) return false;
      h = hr;
    }
    if (h < 0) return false;
    g_unified_heads[i] = h;
  }
  const char** labels[3] = {intent_labels, pii_labels, security_labels};
  const int counts[3] = {intent_labels_count, pii_labels_count, security_labels_count};
  for (int i = 0; i < 3; ++i) {
    g_unified_labels[i].clear();
    for (int k = 0; labels[i] && k < counts[i]; ++k) g_unified_labels[i].push_back(labels[i][k] ? labels[i][k] : "");
  }
  return true;
}

UnifiedBatchResult classify_unified_batch(const char** texts, int num_texts) {
  UnifiedBatchResult err{nullptr, nullptr, nullptr, 0, true, nullptr};
  if (!texts || num_texts <= 0 || !g_unified.ready() || g_unified_heads[2] < 0) { err.error_message = dup_cstr("unified classifier not initialized"); return err; }
  // tokenise all texts (worker threads for large batches), ONE encoder pass per piece of the batch, three heads
  const std::vector<Tokens> toks = tokenize_many(g_unified, texts, num_texts, g_unified.max_len);
  std::vector<int32_t> cu{0};
  for (const Tokens& t : toks) {
    if (t.ids.empty()) { err.error_message = dup_cstr("tokenization failed"); return err; }
    cu.push_back(cu.back() + static_cast<int32_t>(t.ids.size()));
  }
  const int T = cu.back();
  const int C0 = sr_head_num_classes(g_unified.model, g_unified_heads[0]);
  const int C1 = sr_head_num_classes(g_unified.model, g_unified_heads[1]);
  const int C2 = sr_head_num_classes(g_unified.model, g_unified_heads[2]);
  std::vector<float> p0(static_cast<size_t>(num_texts) * C0), p1(static_cast<size_t>(T) * C1), p2(static_cast<size_t>(num_texts) * C2);
  std::vector<int32_t> c0(num_texts), c1(T), c2(num_texts);
  // pieces bounded by the engine's batch limits, spread over the replicas (abi_core.h: for_pieces)
  const bool ok = for_pieces(g_unified, toks, [&](sr_model* m, int first, int b, std::vector<int32_t>& ids, std::vector<int32_t>& pcu) {
    float* pp[3] = {p0.data() + static_cast<size_t>(first) * C0, p1.data() + static_cast<size_t>(cu[first]) * C1,
                    p2.data() + static_cast<size_t>(first) * C2};
    int32_t* cp[3] = {c0.data() + first, c1.data() + cu[first], c2.data() + first};
    return sr_classify_multi_ids(m, g_unified_heads, 3, ids.data(), pcu.data(), b, pp, cp) == 0;
  });
  if (!ok) {
    err.error_message = dup_cstr("inference failed");
    return err;
  }
  UnifiedBatchResult r{static_cast<CIntentResult*>(calloc(num_texts, sizeof(CIntentResult))),
                       static_cast<CPIIResult*>(calloc(num_texts, sizeof(CPIIResult))),
                       static_cast<CSecurityResult*>(calloc(num_texts, sizeof(CSecurityResult))), num_texts, false, nullptr};
  auto lab = [&](int which, int cls) {
    return (cls >= 0 && cls < static_cast<int>(g_unified_labels[which].size())) ? g_unified_labels[which][cls] : "LABEL_" + std::to_string(cls);
  };
  for (int i = 0; i < num_texts; ++i) {
    r.intent_results[i].category = dup_cstr(lab(0, c0[i]));
    r.intent_results[i].confidence = p0[static_cast<size_t>(i) * C0 + c0[i]];
    r.intent_results[i].probabilities = static_cast<float*>(malloc(sizeof(float) * C0));
    if (r.intent_results[i].probabilities) memcpy(r.intent_results[i].probabilities, &p0[static_cast<size_t>(i) * C0], sizeof(float) * C0);
    r.intent_results[i].num_probabilities = C0;
    std::vector<std::string> types;
    float sum = 0.f;
    int n = 0;
    for (int t = cu[i]; t < cu[i + 1]; ++t)
      if (c1[t] > 0) {
        const std::string ty = lab(1, c1[t]);
        if (std::find(types.begin(), types.end(), ty) == types.end()) types.push_back(ty);
        sum += p1[static_cast<size_t>(t) * C1 + c1[t]];
        ++n;
      }
    r.pii_results[i].has_pii = n > 0;
    r.pii_results[i].num_pii_types = static_cast<int>(types.size());
    r.pii_results[i].pii_types = types.empty() ? nullptr : static_cast<char**>(malloc(sizeof(char*) * types.size()));
    for (size_t k = 0; k < types.size() && r.pii_results[i].pii_types; ++k) r.pii_results[i].pii_types[k] = dup_cstr(types[k]);
    r.pii_results[i].confidence = n > 0 ? sum / n : 0.f;
    r.security_results[i].is_jailbreak = c2[i] != 0;
    r.security_results[i].threat_type = dup_cstr(lab(2, c2[i]));
    r.security_results[i].confidence = p2[static_cast<size_t>(i) * C2 + c2[i]];
  }
  return r;
}
void free_unified_batch_result(UnifiedBatchResult result) {
  for (int i = 0; i < result.batch_size; ++i) {
    if (result.intent_results) { free(result.intent_results[i].category); free(result.intent_results[i].probabilities); }
    if (result.pii_results) {
      for (int k = 0; k < result.pii_results[i].num_pii_types; ++k) free(result.pii_results[i].pii_types[k]);
      free(result.pii_results[i].pii_types);
    }
    if (result.security_results) free(result.security_results[i].threat_type);
  }
  free(result.intent_results);
  free(result.pii_results);
  free(result.security_results);
  free(result.error_message);
}

