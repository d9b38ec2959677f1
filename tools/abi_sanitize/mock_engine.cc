// CPU stand-in for the engine side of include/sr_b200.h, used ONLY by tools/abi_sanitize.sh: the text ABI's host code
// (abi.cu, onnx_abi.cu, abi_core.h, tokenizer.cc -- slots, request coalescing, packing, span logic, result ownership) is
// compiled with g++ under AddressSanitizer / ThreadSanitizer and linked against this file instead of the CUDA engine.
// Results are deterministic functions of the token ids (no model arithmetic): what is under test is the host code.
#include "../../include/sr_b200.h"
#include "../../semantic-router_b200/csrc/json.hpp"

#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <mutex>
#include <sstream>
#include <string>
#include <vector>

namespace srb {
bool parse_json_file(const std::string& path, Json& out) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return false;
  std::stringstream ss;
  ss << f.rdbuf();
  const std::string s = ss.str();
  JsonParser p(s.data(), s.size());
  return p.parse(out);
}
}  // namespace srb

struct MockHead { int classes; bool token_level; };
struct sr_model {
  int arch = 0, hidden = 64, layers = 4, max_pos = 1024, device = 0;
  std::vector<MockHead> heads;
  std::mutex mu;
  int flavor = 0;
};

namespace {
int classes_of(const std::string& dir) {
  srb::Json j;
  if (!srb::parse_json_file(dir + "/config.json", j)) return -1;
  const srb::Json* m = j.get("id2label");
  const int named = (m && m->is_obj()) ? static_cast<int>(m->obj.size()) : 0;
  return static_cast<int>(j.num_or("num_labels", named));   // more classes than names: the library must say "LABEL_<id>"
}
uint32_t mix(uint32_t h, uint32_t v) { h ^= v + 0x9e3779b9u + (h << 6) + (h >> 2); return h; }
void fake_probs(uint32_t seed, int C, float* p) {
  float s = 0.f;
  for (int c = 0; c < C; ++c) { seed = mix(seed, static_cast<uint32_t>(c) * 2654435761u); p[c] = 0.05f + static_cast<float>(seed % 1000) / 1000.f; s += p[c]; }
  for (int c = 0; c < C; ++c) p[c] /= s;
}
int argmax(const float* p, int C) { int b = 0; for (int c = 1; c < C; ++c) if (p[c] > p[b]) b = c; return b; }
}  // namespace

extern "C" {
const char* sr_last_error(void) { return "mock"; }
// SR_MOCK_DEVICES=n pretends the box has n GPUs (the multi-device dispatch of abi_core.h is host code too)
int sr_device_count(void) {
  const char* e = getenv("SR_MOCK_DEVICES");
  const int n = e ? atoi(e) : 1;
  return n > 0 && n <= 64 ? n : 1;
}
static std::atomic<long long> g_dev_calls[64], g_dev_rows[64];
// calls / rows (sequences) the mock engine served on `device` since the process started
long long sr_mock_device_calls(int device) { return device >= 0 && device < 64 ? g_dev_calls[device].load() : -1; }
long long sr_mock_device_rows(int device) { return device >= 0 && device < 64 ? g_dev_rows[device].load() : -1; }
static void note(const sr_model* m, int rows) { g_dev_calls[m->device]++; g_dev_rows[m->device] += rows; }
int sr_model_load(const char* dir, int device, sr_model** out) {
  if (!dir || !out || device < 0 || device >= sr_device_count()) return -1;
  const int C = classes_of(dir);
  if (C < 0) return -1;
  sr_model* m = new sr_model();
  m->device = device;
  srb::Json j;
  srb::parse_json_file(std::string(dir) + "/config.json", j);
  m->arch = j.str_or("model_type", "modernbert") == "bert" ? 1 : 0;
  m->max_pos = static_cast<int>(j.num_or("max_position_embeddings", 1024));
  if (C > 0) m->heads.push_back({C, false});
  *out = m;
  return 0;
}
int sr_model_add_head(sr_model* m, const char* dir, int token_level) {
  if (!m || !dir) return -1;
  const int C = classes_of(dir);
  if (C <= 0) return -1;
  std::lock_guard<std::mutex> lk(m->mu);
  m->heads.push_back({C, token_level == 1});
  return static_cast<int>(m->heads.size()) - 1;
}
void sr_model_free(sr_model* m) { delete m; }
int sr_model_info(const sr_model* m, sr_model_info_t* o) {
  if (!m || !o) return -1;
  *o = sr_model_info_t{m->arch, m->hidden, m->layers, 4, 128, 1000, m->max_pos, static_cast<int>(m->heads.size()), m->device};
  return 0;
}
int sr_head_num_classes(const sr_model* m, int head) {
  if (!m || head < 0 || head >= static_cast<int>(m->heads.size())) return -1;
  return m->heads[head].classes;
}
int sr_model_set_head_flavor(sr_model* m, int f) { if (!m) return -1; m->flavor = f; return 0; }
int sr_classify_ids(sr_model* m, int head, const int32_t* ids, const int32_t* cu, int batch, int, float* probs, float* logits,
                    int32_t* cls, float* conf) {
  if (!m || head < 0 || head >= static_cast<int>(m->heads.size()) || batch <= 0) return -1;
  std::lock_guard<std::mutex> lk(m->mu);
  note(m, batch);
  const int C = m->heads[head].classes;
  std::vector<float> p(C);
  for (int b = 0; b < batch; ++b) {
    uint32_t h = 17;
    for (int t = cu[b]; t < cu[b + 1]; ++t) h = mix(h, static_cast<uint32_t>(ids[t]));
    fake_probs(h, C, p.data());
    if (probs) memcpy(probs + static_cast<size_t>(b) * C, p.data(), sizeof(float) * C);
    if (logits) for (int c = 0; c < C; ++c) logits[static_cast<size_t>(b) * C + c] = logf(p[c]);
    const int k = argmax(p.data(), C);
    if (cls) cls[b] = k;
    if (conf) conf[b] = p[k];
  }
  return 0;
}
int sr_classify_tokens_ids(sr_model* m, int head, const int32_t* ids, const int32_t* cu, int batch, float* probs, float* logits,
                           int32_t* pred, float* conf) {
  if (!m || head < 0 || head >= static_cast<int>(m->heads.size()) || batch <= 0) return -1;
  std::lock_guard<std::mutex> lk(m->mu);
  note(m, batch);
  const int C = m->heads[head].classes, T = cu[batch];
  std::vector<float> p(C);
  for (int t = 0; t < T; ++t) {
    fake_probs(mix(99, static_cast<uint32_t>(ids[t]) / 3u), C, p.data());   // neighbouring ids share labels: spans appear
    if (probs) memcpy(probs + static_cast<size_t>(t) * C, p.data(), sizeof(float) * C);
    if (logits) for (int c = 0; c < C; ++c) logits[static_cast<size_t>(t) * C + c] = logf(p[c]);
    const int k = argmax(p.data(), C);
    if (pred) pred[t] = k;
    if (conf) conf[t] = p[k];
  }
  return 0;
}
int sr_embed_ids(sr_model* m, const int32_t* ids, const int32_t* cu, int batch, int target_layer, int target_dim, float* emb) {
  if (!m || !emb || batch <= 0 || target_layer > m->layers || target_dim > m->hidden) return -1;
  std::lock_guard<std::mutex> lk(m->mu);
  note(m, batch);
  const int d = target_dim <= 0 ? m->hidden : target_dim;
  for (int b = 0; b < batch; ++b) {
    uint32_t h = 5;
    float n = 0.f;
    for (int t = cu[b]; t < cu[b + 1]; ++t) h = mix(h, static_cast<uint32_t>(ids[t]));
    for (int i = 0; i < d; ++i) { h = mix(h, static_cast<uint32_t>(i)); emb[static_cast<size_t>(b) * d + i] = static_cast<float>(h % 2001) / 1000.f - 1.f; n += emb[static_cast<size_t>(b) * d + i] * emb[static_cast<size_t>(b) * d + i]; }
    n = sqrtf(n) + 1e-12f;
    for (int i = 0; i < d; ++i) emb[static_cast<size_t>(b) * d + i] /= n;
  }
  return 0;
}
int sr_embed_ids_padded(sr_model* m, const int32_t* ids, const int32_t* cu, const int32_t* real_lens, int batch, float* emb) {
  if (!real_lens) return -1;
  std::vector<int32_t> rcu(batch + 1, 0), rids;   // the mock embeds the real tokens only
  for (int b = 0; b < batch; ++b) {
    rids.insert(rids.end(), ids + cu[b], ids + cu[b] + real_lens[b]);
    rcu[b + 1] = static_cast<int32_t>(rids.size());
  }
  return sr_embed_ids(m, rids.data(), rcu.data(), batch, 0, 0, emb);
}
int sr_classify_multi_ids(sr_model* m, const int* heads, int n_heads, const int32_t* ids, const int32_t* cu, int batch,
                          float** probs_out, int32_t** cls_out) {
  if (!m || !heads) return -1;
  for (int i = 0; i < n_heads; ++i) {
    if (heads[i] < 0 || heads[i] >= static_cast<int>(m->heads.size())) return -1;
    const bool tok = m->heads[heads[i]].token_level;
    if (tok ? sr_classify_tokens_ids(m, heads[i], ids, cu, batch, probs_out[i], nullptr, cls_out[i], nullptr)
            : sr_classify_ids(m, heads[i], ids, cu, batch, 0, probs_out[i], nullptr, cls_out[i], nullptr))
      return -1;
  }
  return 0;
}
// shared-LoRA model: SR_MOCK_LORA_SHARED=1 makes every directory look like an unmerged adapter checkpoint; the mock model
// carries one head per task and answers exactly what the per-task entries answer (so the host code of both paths can be
// compared result by result)
int sr_checkpoint_has_adapters(const char* dir) {
  if (!dir) return -1;
  const char* e = getenv("SR_MOCK_LORA_SHARED");
  return (e && e[0] == '1') ? 1 : 0;
}
struct MockShared { int tasks; };
static std::mutex g_shared_mu;
static std::vector<std::pair<const sr_model*, int>> g_shared;   // models loaded by sr_model_load_lora_shared -> tasks
int sr_model_load_lora_shared(const char* const* dirs, const int* token_level, int n, int device, sr_model** out) {
  if (!dirs || n <= 0 || !out || device < 0 || device >= sr_device_count()) return -1;
  sr_model* m = nullptr;
  if (sr_model_load(dirs[0], device, &m) != 0) return -1;
  m->heads.clear();
  for (int t = 0; t < n; ++t) {
    const int C = classes_of(dirs[t]);
    if (C <= 0) { delete m; return -1; }
    m->heads.push_back({C, token_level && token_level[t] == 1});
  }
  { std::lock_guard<std::mutex> lk(g_shared_mu); g_shared.emplace_back(m, n); }
  *out = m;
  return 0;
}
// grouped model of merged checkpoints: SR_MOCK_GROUPED=1 makes the loader accept the directories (the same mock model as
// the shared-LoRA one); otherwise it refuses them as the engine refuses checkpoints of different encoder shapes
int sr_model_load_grouped(const char* const* dirs, const int* token_level, int n, int device, sr_model** out) {
  const char* e = getenv("SR_MOCK_GROUPED");
  if (!(e && e[0] == '1')) return -1;
  return sr_model_load_lora_shared(dirs, token_level, n, device, out);
}
int sr_lora_shared_tasks(const sr_model* m) {
  std::lock_guard<std::mutex> lk(g_shared_mu);
  for (const auto& kv : g_shared)
    if (kv.first == m) return kv.second;
  return m ? 0 : -1;
}
int sr_classify_lora_shared_ids(sr_model* m, const int32_t* ids, const int32_t* cu, int batch, int pooler_mode, float** probs_out,
                                int32_t** cls_out, float** conf_out) {
  const int n = sr_lora_shared_tasks(m);
  if (n <= 0) return -1;
  for (int t = 0; t < n; ++t) {
    float* p = probs_out ? probs_out[t] : nullptr;
    int32_t* c = cls_out ? cls_out[t] : nullptr;
    float* f = conf_out ? conf_out[t] : nullptr;
    if (m->heads[t].token_level ? sr_classify_tokens_ids(m, t, ids, cu, batch, p, nullptr, c, f)
                                : sr_classify_ids(m, t, ids, cu, batch, pooler_mode, p, nullptr, c, f))
      return -1;
  }
  return 0;
}
}  // extern "C"
