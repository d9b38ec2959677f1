// Engine implementation: safetensors/config loading, weight layout for the kernels, forward orchestration.
// See engine.h.  Weight names follow the reference loaders (SURVEY.md section 3.2):
//   ModernBERT  candle_models/modernbert.rs:108-109,224-229,266-273,407-449; traditional/modernbert.rs:723-755
//               prefixes tried like embedding/mmbert_embedding.rs:445-486,583-588
//   BERT        traditional/bert.rs:98-116 (+ candle BertModel::load names), core/similarity.rs:135
#include "engine.h"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <fstream>
#include <sstream>

#include "common.cuh"
#include "gemm.h"
#include "json.hpp"

#include <atomic>

namespace srb {

static std::atomic<long long> g_launches{0};
void note_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launches_total() { return g_launches.load(std::memory_order_relaxed); }
bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("SRB_PDL");
    return e && e[0] == '1';
  }();
  return on;
}

namespace {
struct ProfScope {
  Model& m;
  cudaEvent_t a = nullptr, b = nullptr;
  int cat;
  ProfScope(Model& mm, int c) : m(mm), cat(c) {
    Profiler& p = m.prof;
    if (!p.on) return;
    while (p.pool.size() < p.used + 2) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      p.pool.push_back(e);
    }
    a = p.pool[p.used++];
    b = p.pool[p.used++];
    cudaEventRecord(a, m.stream);
  }
  ~ProfScope() {
    if (!a) return;
    cudaEventRecord(b, m.stream);
    m.prof.recs.push_back({cat, a, b});
  }
};
}  // namespace

void profile_enable(Model& m, bool on) {
  m.prof.on = on;
  m.prof.used = 0;
  m.prof.recs.clear();
  for (int i = 0; i < PC_COUNT; ++i) { m.prof.ms[i] = 0.f; m.prof.count[i] = 0; }
}
int profile_collect(Model& m) {
  if (cudaStreamSynchronize(m.stream) != cudaSuccess) return -1;
  for (const auto& r : m.prof.recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { m.prof.ms[r.cat] += ms; m.prof.count[r.cat]++; }
  }
  m.prof.recs.clear();
  m.prof.used = 0;
  return 0;
}

bool read_file(const std::string& path, std::string& out) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return false;
  std::stringstream ss;
  ss << f.rdbuf();
  out = ss.str();
  return true;
}
bool parse_json_file(const std::string& path, Json& out) {
  std::string s;
  if (!read_file(path, s)) return false;
  JsonParser p(s.data(), s.size());
  return p.parse(out);
}

namespace {

// ------------------------------------------------------------------------------------------------
// safetensors (mmap)
// ------------------------------------------------------------------------------------------------
struct StTensor {
  std::string dtype;
  std::vector<int64_t> shape;
  const uint8_t* data = nullptr;
  size_t bytes = 0;
  size_t numel() const {
    size_t n = 1;
    for (auto d : shape) n *= static_cast<size_t>(d);
    return n;
  }
};

struct SafeTensors {
  int fd = -1;
  void* map = nullptr;
  size_t size = 0;
  std::map<std::string, StTensor> tensors;
  ~SafeTensors() {
    if (map) munmap(map, size);
    if (fd >= 0) close(fd);
  }
  bool open(const std::string& path, std::string* err) {
    fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) { *err = "cannot open " + path; return false; }
    struct stat st;
    if (fstat(fd, &st) != 0 || st.st_size < 8) { *err = "bad safetensors file " + path; return false; }
    size = static_cast<size_t>(st.st_size);
    map = mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (map == MAP_FAILED) { map = nullptr; *err = "mmap failed for " + path; return false; }
    const uint8_t* base = static_cast<const uint8_t*>(map);
    uint64_t hlen;
    memcpy(&hlen, base, 8);
    if (hlen > size - 8) { *err = "safetensors header exceeds file"; return false; }
    Json hdr;
    JsonParser jp(reinterpret_cast<const char*>(base + 8), hlen);
    if (!jp.parse(hdr) || !hdr.is_obj()) { *err = "safetensors header is not JSON"; return false; }
    const uint8_t* data0 = base + 8 + hlen;
    for (const auto& kv : hdr.obj) {
      if (kv.first == "__metadata__") continue;
      const Json* dt = kv.second.get("dtype");
      const Json* sh = kv.second.get("shape");
      const Json* off = kv.second.get("data_offsets");
      if (!dt || !sh || !off || off->arr.size() != 2) continue;
      StTensor t;
      t.dtype = dt->str;
      for (const auto& d : sh->arr) t.shape.push_back(static_cast<int64_t>(d.num));
      const double bd = off->arr[0].num, ed = off->arr[1].num;
      const size_t room = size - 8 - static_cast<size_t>(hlen);
      if (!(bd >= 0.0) || !(ed >= bd) || ed > static_cast<double>(room)) { *err = "tensor " + kv.first + " out of bounds"; return false; }
      const size_t b = static_cast<size_t>(bd), e = static_cast<size_t>(ed);
      if (e > room || e < b) { *err = "tensor " + kv.first + " out of bounds"; return false; }
      t.data = data0 + b;
      t.bytes = e - b;
      tensors.emplace(kv.first, std::move(t));
    }
    return true;
  }
  const StTensor* find(const std::string& name) const {
    auto it = tensors.find(name);
    return it == tensors.end() ? nullptr : &it->second;
  }
};

bool to_f32(const StTensor& t, std::vector<float>& out) {
  const size_t n = t.numel();
  out.resize(n);
  if (t.dtype == "F32") {
    if (t.bytes != n * 4) return false;
    memcpy(out.data(), t.data, n * 4);
  } else if (t.dtype == "F16") {
    if (t.bytes != n * 2) return false;
    const __half* h = reinterpret_cast<const __half*>(t.data);
    for (size_t i = 0; i < n; ++i) out[i] = __half2float(h[i]);
  } else if (t.dtype == "BF16") {
    if (t.bytes != n * 2) return false;
    const uint16_t* h = reinterpret_cast<const uint16_t*>(t.data);
    for (size_t i = 0; i < n; ++i) {
      uint32_t u = static_cast<uint32_t>(h[i]) << 16;
      memcpy(&out[i], &u, 4);
    }
  } else {
    return false;
  }
  return true;
}

// Unmerged LoRA checkpoints (model_architectures/lora/lora_adapter.rs:76-170): next to `X.weight` [out, in] sit
// `X.lora_A.weight` [r, in] and `X.lora_B.weight` [out, r]; the adapted layer computes x W^T + (x A^T) B^T * (alpha / r)
// (:136-144), i.e. W' = W + (alpha / r) B A (merge_weights, :157-168).  The fold happens at load time, in double precision,
// BEFORE the fp16 rounding of the weight, so the device sees exactly the merged matrix the reference's merge would produce.
bool lora_fold(const SafeTensors& st, const std::string& name, const StTensor& base, double alpha, std::vector<float>& w,
               std::string* err) {
  const std::string suffix = ".weight";
  if (base.shape.size() != 2 || name.size() <= suffix.size() || name.compare(name.size() - suffix.size(), suffix.size(), suffix) != 0)
    return true;
  const std::string stem = name.substr(0, name.size() - suffix.size());
  const StTensor* ta = st.find(stem + ".lora_A.weight");
  const StTensor* tb = st.find(stem + ".lora_B.weight");
  if (!ta && !tb) return true;
  if (!ta || !tb) { *err = "LoRA adapter of " + name + " is incomplete (lora_A / lora_B)"; return false; }
  const int64_t out = base.shape[0], in = base.shape[1];
  if (ta->shape.size() != 2 || tb->shape.size() != 2 || ta->shape[1] != in || tb->shape[0] != out || ta->shape[0] != tb->shape[1]) {
    *err = "LoRA adapter of " + name + " does not fit the base weight";
    return false;
  }
  const int64_t r = ta->shape[0];
  std::vector<float> a, b;
  if (!to_f32(*ta, a) || !to_f32(*tb, b)) { *err = "LoRA adapter of " + name + " has an unsupported dtype"; return false; }
  const double scaling = alpha / static_cast<double>(r);
  std::vector<double> row(static_cast<size_t>(in));
  for (int64_t o = 0; o < out; ++o) {
    std::fill(row.begin(), row.end(), 0.0);
    for (int64_t k = 0; k < r; ++k) {
      const double bk = b[static_cast<size_t>(o * r + k)];
      const float* ak = a.data() + static_cast<size_t>(k * in);
      for (int64_t i = 0; i < in; ++i) row[i] += bk * ak[i];
    }
    float* wo = w.data() + static_cast<size_t>(o * in);
    for (int64_t i = 0; i < in; ++i) wo[i] = static_cast<float>(static_cast<double>(wo[i]) + scaling * row[i]);
  }
  return true;
}
double lora_alpha_of(const std::string& dir) {
  Json lj;
  if (parse_json_file(dir + "/lora_config.json", lj)) return lj.num_or("alpha", lj.num_or("lora_alpha", 32.0));
  return 32.0;
}

// ------------------------------------------------------------------------------------------------
// device upload helpers
// ------------------------------------------------------------------------------------------------
struct Loader {
  Model* m;
  const SafeTensors* st;
  std::string err;
  bool ok = true;

  void fail(const std::string& e) {
    if (ok) err = e;
    ok = false;
  }
  void* dalloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) {
      fail("cudaMalloc failed (" + std::to_string(bytes) + " bytes)");
      return nullptr;
    }
    m->allocs.push_back(p);
    return p;
  }
  bool host_f32(const std::string& name, std::vector<float>& out, const std::vector<int64_t>& shape,
                bool required = true) {
    const StTensor* t = st->find(name);
    if (!t) {
      if (required) fail("missing tensor " + name);
      return false;
    }
    if (!shape.empty() && t->shape != shape) {
      std::string s = "tensor " + name + " has shape [";
      for (auto d : t->shape) s += std::to_string(d) + ",";
      s += "] expected [";
      for (auto d : shape) s += std::to_string(d) + ",";
      fail(s + "]");
      return false;
    }
    if (!to_f32(*t, out)) { fail("tensor " + name + " has unsupported dtype " + t->dtype); return false; }
    if (!merge_lora(name, *t, out)) return false;
    return true;
  }
  double lora_alpha = 32.0;   // LoRAConfig::default (lora_adapter.rs:29-38); <dir>/lora_config.json {"alpha", "rank"} overrides
  bool keep_adapters = false; // shared-LoRA models: the base weights load unmerged
  bool merge_lora(const std::string& name, const StTensor& base, std::vector<float>& w) {
    if (keep_adapters) return true;
    std::string e;
    if (!lora_fold(*st, name, base, lora_alpha, w, &e)) { fail(e); return false; }
    return true;
  }
  float* up_f32(const std::vector<float>& v) {
    float* d = static_cast<float*>(dalloc(v.size() * 4));
    if (d && cudaMemcpy(d, v.data(), v.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) fail("H2D copy failed");
    return d;
  }
  __half* up_f16(const std::vector<float>& v) {
    std::vector<__half> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = __float2half_rn(v[i]);
    __half* d = static_cast<__half*>(dalloc(h.size() * 2));
    if (d && cudaMemcpy(d, h.data(), h.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess) fail("H2D copy failed");
    return d;
  }
  float* f32(const std::string& name, const std::vector<int64_t>& shape, bool required = true) {
    std::vector<float> v;
    if (!host_f32(name, v, shape, required)) return nullptr;
    return up_f32(v);
  }
  __half* f16(const std::string& name, const std::vector<int64_t>& shape) {
    std::vector<float> v;
    if (!host_f32(name, v, shape)) return nullptr;
    return up_f16(v);
  }
};

void parse_id2label(const Json& cfg, std::map<int, std::string>& out) {
  const Json* m = cfg.get("id2label");
  if (!m || !m->is_obj()) return;
  for (const auto& kv : m->obj)
    if (kv.second.is_str()) out[atoi(kv.first.c_str())] = kv.second.str;
}

// RotaryEmbedding::new (candle_models/modernbert.rs:61-80): inv_freq = 1f32 / (theta.powf(i/dim) as f32),
// freqs = t(f32) * inv_freq (f32), sin/cos in f32.
void rope_tables(int head_dim, double theta, int max_pos, std::vector<float>& cs, std::vector<float>& sn) {
  const int half = head_dim / 2;
  std::vector<float> inv(half);
  for (int i = 0; i < half; ++i) {
    const float denom = static_cast<float>(std::pow(theta, static_cast<double>(2 * i) / head_dim));
    inv[i] = 1.0f / denom;
  }
  cs.resize(static_cast<size_t>(max_pos) * half);
  sn.resize(cs.size());
  for (int t = 0; t < max_pos; ++t)
    for (int i = 0; i < half; ++i) {
      const float f = static_cast<float>(t) * inv[i];
      cs[static_cast<size_t>(t) * half + i] = cosf(f);
      sn[static_cast<size_t>(t) * half + i] = sinf(f);
    }
}

bool load_head(Loader& ld, const Json& cfgj, Arch arch, int H, const std::string& bert_prefix,
               int force_token_level, Head& hd) {
  const SafeTensors& st = *ld.st;
  const StTensor* cw = st.find("classifier.weight");
  if (!cw || cw->shape.size() != 2 || cw->shape[1] != H) return false;
  hd.num_classes = static_cast<int>(cw->shape[0]);
  bool token = false;
  if (const Json* a = cfgj.get("architectures"))
    for (const auto& s : a->arr)
      if (s.is_str() && s.str.find("TokenClassification") != std::string::npos) token = true;
  if (force_token_level >= 0) token = force_token_level != 0;
  hd.token_level = token;
  hd.cls_w = ld.f32("classifier.weight", {hd.num_classes, H});
  hd.cls_b = ld.f32("classifier.bias", {hd.num_classes});
  parse_id2label(cfgj, hd.id2label);
  if (arch == ARCH_MODERNBERT) {
    if (st.find("head.dense.weight")) {
      hd.has_dense = true;
      std::vector<float> w;
      if (ld.host_f32("head.dense.weight", w, {H, H})) {
        hd.dense_w32 = ld.up_f32(w);
        hd.dense_w16 = ld.up_f16(w);
      }
      hd.norm_w = ld.f32("head.norm.weight", {H});
    }
  } else {
    const std::string pn = bert_prefix + "pooler.dense.weight";
    if (st.find(pn)) {
      hd.has_dense = true;
      hd.dense_w32 = ld.f32(pn, {H, H});
      hd.dense_b = ld.f32(bert_prefix + "pooler.dense.bias", {H});
    }
  }
  return ld.ok;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// model load
// ------------------------------------------------------------------------------------------------
// SRB_LN_FOLD=0 keeps the separate LayerNorm kernels (exact LayerNorm input rounding; A/B measurements)
bool ln_fold_enabled() {
  static const bool on = [] {
    const char* e = getenv("SRB_LN_FOLD");
    return !(e && e[0] == '0');
  }();
  return on;
}

// W'' = W diag(gamma), every row re-centred to sum zero, rounded to fp16.  Two refinement passes push the sum of the
// ROUNDED row (what the tensor core multiplies) from ~1e-4 down to the last bit of its largest elements, so the
// residual mean * sum(W''[n,:]) is far below the fp16 rounding of the output.
static void fold_weights(Loader& ld, const std::vector<float>& w, const std::vector<float>& gamma, int n, int k, __half** w_f) {
  std::vector<float> wf(w.size());
  std::vector<double> row(k);
  for (int r = 0; r < n; ++r) {
    double s = 0.0;
    for (int c = 0; c < k; ++c) { row[c] = static_cast<double>(w[static_cast<size_t>(r) * k + c]) * gamma[c]; s += row[c]; }
    const double mu = s / k;
    for (int c = 0; c < k; ++c) row[c] -= mu;
    for (int pass = 0; pass < 3; ++pass) {
      double rs = 0.0;
      for (int c = 0; c < k; ++c) rs += __half2float(__float2half_rn(static_cast<float>(row[c])));
      if (rs == 0.0) break;
      for (int c = 0; c < k; ++c) row[c] -= rs / k;
    }
    for (int c = 0; c < k; ++c) wf[static_cast<size_t>(r) * k + c] = static_cast<float>(row[c]);
  }
  *w_f = ld.up_f16(wf);
}

Model* model_load(const std::string& dir, int device, std::string* err, int flags) {
  std::string e;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    *err = "no CUDA device available (this library has no CPU path)";
    return nullptr;
  }
  if (device < 0 || device >= ndev) { *err = "invalid device index " + std::to_string(device); return nullptr; }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9 || prop.minor != 0) {
    *err = std::string("device ") + prop.name + " is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) +
           "; this library is built for sm_90a only";
    return nullptr;
  }
  if (cudaSetDevice(device) != cudaSuccess) { *err = "cudaSetDevice failed"; return nullptr; }

  Json cfgj;
  if (!parse_json_file(dir + "/config.json", cfgj)) { *err = "cannot read " + dir + "/config.json"; return nullptr; }
  SafeTensors st;
  if (!st.open(dir + "/model.safetensors", &e)) { *err = e; return nullptr; }

  Model* m = new Model();
  m->device = device;
  m->dir = dir;
  Loader ld{m, &st};
  ld.lora_alpha = lora_alpha_of(dir);
  ld.keep_adapters = (flags & kLoadKeepAdapters) != 0;
  EncoderConfig& c = m->cfg;
  const std::string mt = cfgj.str_or("model_type", "");
  std::string P;  // tensor-name prefix
  if (mt == "modernbert" || st.find("model.embeddings.tok_embeddings.weight") ||
      st.find("embeddings.tok_embeddings.weight") || st.find("_orig_mod.model.embeddings.tok_embeddings.weight")) {
    c.arch = ARCH_MODERNBERT;
    const char* prefixes[] = {"model.", "_orig_mod.model.", "", "_orig_mod."};
    bool found = false;
    for (const char* p : prefixes)
      if (st.find(std::string(p) + "embeddings.tok_embeddings.weight")) { P = p; found = true; break; }
    if (!found) ld.fail("no tok_embeddings tensor under any known prefix");
  } else {
    c.arch = ARCH_BERT;
    if (st.find("bert.embeddings.word_embeddings.weight")) P = "bert.";
    else if (st.find("embeddings.word_embeddings.weight")) P = "";
    else ld.fail("no BERT word_embeddings tensor found");
  }
  c.vocab = static_cast<int>(cfgj.num_or("vocab_size", 0));
  c.H = static_cast<int>(cfgj.num_or("hidden_size", 0));
  c.L = static_cast<int>(cfgj.num_or("num_hidden_layers", 0));
  c.heads = static_cast<int>(cfgj.num_or("num_attention_heads", 0));
  c.I = static_cast<int>(cfgj.num_or("intermediate_size", 0));
  c.max_pos = static_cast<int>(cfgj.num_or("max_position_embeddings", 512));
  c.pad_id = static_cast<int>(cfgj.num_or("pad_token_id", 0));
  if (c.arch == ARCH_MODERNBERT) {
    c.ln_eps = static_cast<float>(cfgj.num_or("layer_norm_eps", cfgj.num_or("norm_eps", 1e-5)));
    c.global_every = static_cast<int>(cfgj.num_or("global_attn_every_n_layers", 3));
    c.theta_global = cfgj.num_or("global_rope_theta", 160000.0);
    c.theta_local = cfgj.num_or("local_rope_theta", 10000.0);
    c.local_attention = static_cast<int>(cfgj.num_or("local_attention", 128));
    if (const Json* cp = cfgj.get("classifier_pooling")) c.cls_pooling = (cp->is_str() && cp->str == "mean") ? 1 : 0;
  } else {
    c.ln_eps = static_cast<float>(cfgj.num_or("layer_norm_eps", 1e-12));
    c.type_vocab = static_cast<int>(cfgj.num_or("type_vocab_size", 2));
  }
  parse_id2label(cfgj, c.id2label);
  if (ld.ok && (c.H <= 0 || c.L <= 0 || c.heads <= 0 || c.vocab <= 0 || c.I <= 0)) ld.fail("config.json incomplete");
  const int head_dim = (c.heads > 0) ? c.H / c.heads : 0;
  if (ld.ok && (c.H % (c.heads > 0 ? c.heads : 1) != 0 || !(head_dim == 64 || (head_dim == 32 && c.arch == ARCH_BERT))))
    ld.fail("head_dim " + std::to_string(head_dim) + " unsupported (64; 32 for BERT/MiniLM encoders)");
  c.attn_w = c.heads * 64;
  if (ld.ok && !(c.H == 384 || c.H == 768 || c.H == 1024)) ld.fail("hidden_size unsupported");

  const int H = c.H, I = c.I;
  if (ld.ok && c.arch == ARCH_MODERNBERT) {
    if (I % 32 != 0) ld.fail("intermediate_size must be a multiple of 32");
    m->emb_word = ld.f32(P + "embeddings.tok_embeddings.weight", {c.vocab, H});
    m->emb_ln_w = ld.f32(P + "embeddings.norm.weight", {H});
    m->layers.resize(c.L);
    for (int li = 0; li < c.L && ld.ok; ++li) {
      const std::string Lp = P + "layers." + std::to_string(li) + ".";
      LayerWeights& lw = m->layers[li];
      if (st.find(Lp + "attn_norm.weight")) lw.attn_norm_w = ld.f32(Lp + "attn_norm.weight", {H});
      std::vector<float> wq, g_attn, g_mlp;
      if (ld.host_f32(Lp + "attn.Wqkv.weight", wq, {3 * H, H})) lw.wqkv = ld.up_f16(wq);
      lw.wo = ld.f16(Lp + "attn.Wo.weight", {H, H});
      lw.mid_norm_w = ld.f32(Lp + "mlp_norm.weight", {H});
      const bool fold = ln_fold_enabled() && H % 128 == 0;
      if (fold && lw.attn_norm_w && ld.host_f32(Lp + "attn_norm.weight", g_attn, {H}))
        fold_weights(ld, wq, g_attn, 3 * H, H, &lw.wqkv_f);
      if (fold) ld.host_f32(Lp + "mlp_norm.weight", g_mlp, {H});
      std::vector<float> wi, wi_perm;
      if (ld.host_f32(Lp + "mlp.Wi.weight", wi, {2 * I, H})) {
        // GeGLU interleave for the fused epilogue: 32-row groups [a(32j..) | b(32j..)] (gemm.h EPI_GEGLU)
        wi_perm.resize(wi.size());
        for (int j = 0; j < I / 32; ++j) {
          memcpy(&wi_perm[static_cast<size_t>(64 * j) * H], &wi[static_cast<size_t>(32 * j) * H], sizeof(float) * 32 * H);
          memcpy(&wi_perm[static_cast<size_t>(64 * j + 32) * H], &wi[static_cast<size_t>(I + 32 * j) * H],
                 sizeof(float) * 32 * H);
        }
        lw.wi = ld.up_f16(wi_perm);
        if (fold && !g_mlp.empty()) fold_weights(ld, wi_perm, g_mlp, 2 * I, H, &lw.wi_f);
      }
      lw.wo2 = ld.f16(Lp + "mlp.Wo.weight", {H, I});
    }
    m->final_norm_w = ld.f32(P + "final_norm.weight", {H});
    if (ld.ok) {
      m->rope_len = c.max_pos;
      std::vector<float> cs, sn;
      rope_tables(64, c.theta_global, c.max_pos, cs, sn);
      m->rope_cos_g = ld.up_f32(cs);
      m->rope_sin_g = ld.up_f32(sn);
      rope_tables(64, c.theta_local, c.max_pos, cs, sn);
      m->rope_cos_l = ld.up_f32(cs);
      m->rope_sin_l = ld.up_f32(sn);
    }
  } else if (ld.ok) {
    const std::string E = P + "embeddings.";
    m->emb_word = ld.f32(E + "word_embeddings.weight", {c.vocab, H});
    m->emb_pos = ld.f32(E + "position_embeddings.weight", {c.max_pos, H});
    std::vector<float> tt;
    if (ld.host_f32(E + "token_type_embeddings.weight", tt, {c.type_vocab, H})) {
      tt.resize(H);  // token_type_ids are always zero (traditional/bert.rs:227)
      m->emb_type0 = ld.up_f32(tt);
    }
    m->emb_ln_w = ld.f32(E + "LayerNorm.weight", {H});
    m->emb_ln_b = ld.f32(E + "LayerNorm.bias", {H});
    m->layers.resize(c.L);
    for (int li = 0; li < c.L && ld.ok; ++li) {
      const std::string Lp = P + "encoder.layer." + std::to_string(li) + ".";
      LayerWeights& lw = m->layers[li];
      std::vector<float> q, k, v, bq, bk, bv;
      if (ld.host_f32(Lp + "attention.self.query.weight", q, {H, H}) &&
          ld.host_f32(Lp + "attention.self.key.weight", k, {H, H}) &&
          ld.host_f32(Lp + "attention.self.value.weight", v, {H, H}) &&
          ld.host_f32(Lp + "attention.self.query.bias", bq, {H}) &&
          ld.host_f32(Lp + "attention.self.key.bias", bk, {H}) &&
          ld.host_f32(Lp + "attention.self.value.bias", bv, {H})) {
        if (head_dim == 32) {
          // rows (h*64 + d) <- rows (h*32 + d), zeros for d >= 32.  The kernels scale scores by 64^-0.5; the model
          // wants 32^-0.5, so the query projection carries the missing sqrt(2).
          auto pad_rows = [&](std::vector<float>& wgt, std::vector<float>& bias, float scale) {
            std::vector<float> pw(static_cast<size_t>(c.attn_w) * H, 0.f), pb(c.attn_w, 0.f);
            for (int h = 0; h < c.heads; ++h)
              for (int d = 0; d < 32; ++d) {
                const size_t src = static_cast<size_t>(h * 32 + d), dst = static_cast<size_t>(h * 64 + d);
                for (int kk = 0; kk < H; ++kk) pw[dst * H + kk] = wgt[src * H + kk] * scale;
                pb[dst] = bias[src] * scale;
              }
            wgt.swap(pw);
            bias.swap(pb);
          };
          pad_rows(q, bq, 1.41421356237309504880f);
          pad_rows(k, bk, 1.0f);
          pad_rows(v, bv, 1.0f);
        }
        q.insert(q.end(), k.begin(), k.end());
        q.insert(q.end(), v.begin(), v.end());
        bq.insert(bq.end(), bk.begin(), bk.end());
        bq.insert(bq.end(), bv.begin(), bv.end());
        lw.wqkv = ld.up_f16(q);
        lw.bqkv = ld.up_f32(bq);
      }
      if (head_dim == 32) {   // attention-output projection reads the padded context rows: zero columns for d >= 32
        std::vector<float> wo;
        if (ld.host_f32(Lp + "attention.output.dense.weight", wo, {H, H})) {
          std::vector<float> pw(static_cast<size_t>(H) * c.attn_w, 0.f);
          for (int o = 0; o < H; ++o)
            for (int h = 0; h < c.heads; ++h)
              for (int d = 0; d < 32; ++d)
                pw[static_cast<size_t>(o) * c.attn_w + h * 64 + d] = wo[static_cast<size_t>(o) * H + h * 32 + d];
          lw.wo = ld.up_f16(pw);
        }
      } else {
        lw.wo = ld.f16(Lp + "attention.output.dense.weight", {H, H});
      }
      lw.bo = ld.f32(Lp + "attention.output.dense.bias", {H});
      lw.mid_norm_w = ld.f32(Lp + "attention.output.LayerNorm.weight", {H});
      lw.mid_norm_b = ld.f32(Lp + "attention.output.LayerNorm.bias", {H});
      lw.wi = ld.f16(Lp + "intermediate.dense.weight", {I, H});
      lw.bi = ld.f32(Lp + "intermediate.dense.bias", {I});
      lw.wo2 = ld.f16(Lp + "output.dense.weight", {H, I});
      lw.bo2 = ld.f32(Lp + "output.dense.bias", {H});
      lw.out_norm_w = ld.f32(Lp + "output.LayerNorm.weight", {H});
      lw.out_norm_b = ld.f32(Lp + "output.LayerNorm.bias", {H});
    }
  }
  if (ld.ok && !(flags & kLoadNoHead) && st.find("classifier.weight")) {
    Head hd;
    if (load_head(ld, cfgj, c.arch, H, P, -1, hd)) m->heads.push_back(hd);
  }
  if (ld.ok && cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess) ld.fail("stream create failed");
  if (!ld.ok) {
    *err = ld.err;
    model_free(m);
    return nullptr;
  }
  cudaDeviceSynchronize();
  return m;
}

int model_add_head(Model* m, const std::string& dir, int force_token_level, std::string* err) {
  if (cudaSetDevice(m->device) != cudaSuccess) { *err = "cudaSetDevice failed"; return -1; }
  Json cfgj;
  if (!parse_json_file(dir + "/config.json", cfgj)) { *err = "cannot read " + dir + "/config.json"; return -1; }
  SafeTensors st;
  std::string e;
  if (!st.open(dir + "/model.safetensors", &e)) { *err = e; return -1; }
  Loader ld{m, &st};
  Head hd;
  const std::string bp = st.find("bert.pooler.dense.weight") ? "bert." : "";
  if (!load_head(ld, cfgj, m->cfg.arch, m->cfg.H, bp, force_token_level, hd) || !ld.ok) {
    *err = ld.ok ? "no classifier.weight in " + dir : ld.err;
    return -1;
  }
  m->heads.push_back(hd);
  return static_cast<int>(m->heads.size()) - 1;
}


// ------------------------------------------------------------------------------------------------
// shared-base multi-task model from unmerged LoRA checkpoints (engine.h: LoraShared)
// ------------------------------------------------------------------------------------------------
namespace {
bool is_head_tensor(const std::string& n) {
  return n.compare(0, 11, "classifier.") == 0 || n.compare(0, 5, "head.") == 0 || n.find("pooler.") != std::string::npos;
}
struct AdapterSeg { std::string stem; int row0, rows; };   // one adapted nn.Linear inside a (possibly fused) projection

// Stacks the adapters of every task for one projection [N, K] made of `segs` (engine.h: LoraProj).  gamma: LayerNorm
// weight for the fold form (empty: none).  perm: destination row of source row n in the device weight (GeGLU
// interleave), empty: identity.  Returns false on a malformed adapter; leaves lp empty when no task adapts the projection.
bool build_lora_proj(Loader& ld, const std::vector<std::unique_ptr<SafeTensors>>& sts, const std::vector<double>& alpha,
                     const std::vector<AdapterSeg>& segs, int N, int K, int rp, const std::vector<float>& gamma,
                     const std::vector<int>& perm, LoraProj& lp) {
  const int T = static_cast<int>(sts.size());
  const int nseg = static_cast<int>(segs.size());
  const int block = nseg * rp;
  const int R = (T * block + 63) / 64 * 64;
  std::vector<float> a(static_cast<size_t>(R) * K, 0.f), b(static_cast<size_t>(N) * R, 0.f);
  bool any = false;
  for (int t = 0; t < T; ++t)
    for (int sg = 0; sg < nseg; ++sg) {
      const StTensor* ta = sts[t]->find(segs[sg].stem + ".lora_A.weight");
      const StTensor* tb = sts[t]->find(segs[sg].stem + ".lora_B.weight");
      if (!ta && !tb) continue;
      if (!ta || !tb || ta->shape.size() != 2 || tb->shape.size() != 2 || ta->shape[1] != K || tb->shape[0] != segs[sg].rows ||
          ta->shape[0] != tb->shape[1] || ta->shape[0] > rp) {
        ld.fail("LoRA adapter of " + segs[sg].stem + " (task " + std::to_string(t) + ") does not fit the base weight");
        return false;
      }
      const int r = static_cast<int>(ta->shape[0]);
      std::vector<float> av, bv;
      if (!to_f32(*ta, av) || !to_f32(*tb, bv)) { ld.fail("LoRA adapter of " + segs[sg].stem + " has an unsupported dtype"); return false; }
      const double scaling = alpha[t] / static_cast<double>(r);   // lora_adapter.rs:117
      const int c0 = t * block + sg * rp;
      for (int j = 0; j < r; ++j) memcpy(&a[static_cast<size_t>(c0 + j) * K], &av[static_cast<size_t>(j) * K], sizeof(float) * K);
      for (int n = 0; n < segs[sg].rows; ++n) {
        const int src = segs[sg].row0 + n;
        const int dst = perm.empty() ? src : perm[src];
        for (int j = 0; j < r; ++j)
          b[static_cast<size_t>(dst) * R + c0 + j] = static_cast<float>(scaling * static_cast<double>(bv[static_cast<size_t>(n) * r + j]));
      }
      any = true;
    }
  if (!any) return true;
  lp.a = ld.up_f16(a);
  lp.b = ld.up_f16(b);
  if (!gamma.empty()) fold_weights(ld, a, gamma, R, K, &lp.a_f);
  lp.R = R;
  lp.block = block;
  return ld.ok;
}
}  // namespace

Model* model_load_lora_shared(const std::vector<std::string>& dirs, const std::vector<int>& token_level, int device,
                              bool grouped, std::string* err) {
  const int T = static_cast<int>(dirs.size());
  if (T < 1 || token_level.size() != dirs.size()) { *err = "bad arguments"; return nullptr; }
  std::vector<std::unique_ptr<SafeTensors>> sts;
  std::vector<double> alpha;
  for (const std::string& d : dirs) {
    sts.emplace_back(new SafeTensors());
    if (!sts.back()->open(d + "/model.safetensors", err)) return nullptr;
    alpha.push_back(lora_alpha_of(d));
  }
  // one base: every non-adapter, non-head tensor of task 0 must sit, bit for bit, in the other checkpoints
  int max_rank = 0;
  for (const auto& kv : sts[0]->tensors) {
    if (kv.first.find(".lora_") != std::string::npos || is_head_tensor(kv.first)) continue;
    for (int t = 1; t < T; ++t) {
      const StTensor* o = sts[t]->find(kv.first);
      if (!o || o->dtype != kv.second.dtype || o->shape != kv.second.shape || o->bytes != kv.second.bytes ||
          memcmp(o->data, kv.second.data, o->bytes) != 0) {
        *err = "the checkpoints do not share one base: " + kv.first + " differs in " + dirs[t];
        return nullptr;
      }
    }
  }
  for (int t = 0; t < T; ++t)
    for (const auto& kv : sts[t]->tensors)
      if (kv.first.size() > 14 && kv.first.compare(kv.first.size() - 14, 14, ".lora_A.weight") == 0 && kv.second.shape.size() == 2)
        max_rank = std::max(max_rank, static_cast<int>(kv.second.shape[0]));
  if (max_rank <= 0) { *err = "no lora_A / lora_B tensors in these checkpoints (merged models load as separate slots)"; return nullptr; }
  if (max_rank > 256) { *err = "LoRA rank above 256"; return nullptr; }
  Model* m = model_load(dirs[0], device, err, kLoadKeepAdapters | kLoadNoHead);
  if (!m) return nullptr;
  const EncoderConfig& c = m->cfg;
  if (c.attn_w != c.H) { *err = "shared-LoRA serving is not available for padded-head (MiniLM) encoders"; model_free(m); return nullptr; }
  Loader ld{m, sts[0].get()};
  const int rp = (max_rank + 7) / 8 * 8;
  const int H = c.H, I = c.I;
  m->lora.layers.resize(c.L);
  std::string P;
  if (c.arch == ARCH_MODERNBERT) {
    const char* prefixes[] = {"model.", "_orig_mod.model.", "", "_orig_mod."};
    for (const char* p : prefixes)
      if (sts[0]->find(std::string(p) + "embeddings.tok_embeddings.weight")) { P = p; break; }
  } else if (sts[0]->find("bert.embeddings.word_embeddings.weight")) {
    P = "bert.";
  }
  std::vector<int> geglu_perm;   // source row of Wi -> row of the interleaved device weight (model_load)
  if (c.arch == ARCH_MODERNBERT) {
    geglu_perm.resize(static_cast<size_t>(2) * I);
    for (int j = 0; j < I / 32; ++j)
      for (int i = 0; i < 32; ++i) {
        geglu_perm[32 * j + i] = 64 * j + i;
        geglu_perm[I + 32 * j + i] = 64 * j + 32 + i;
      }
  }
  const std::vector<float> none;
  const std::vector<int> ident;
  if (grouped) {
    // every task's merged weights, stacked along N.  Loader{.., sts[t]} merges task t's adapters exactly as a separately
    // loaded model would (lora_fold, double precision, before the fp16 rounding).
    m->lora.glayers = m->layers;   // norms / biases are the base's (adapters touch projection weights only)
    auto stack = [&](const std::vector<std::string>& names, int rows_each, int K, std::vector<float>& out) {
      // out = [task 0: names[0]; names[1]; ... | task 1: ... ], each name a [rows_each, K] Linear weight
      out.clear();
      out.reserve(static_cast<size_t>(T) * names.size() * rows_each * K);
      for (int t = 0; t < T && ld.ok; ++t) {
        Loader lt{m, sts[t].get()};
        lt.lora_alpha = alpha[t];
        for (const std::string& nm : names) {
          std::vector<float> v;
          if (!lt.host_f32(nm, v, {rows_each, K})) { ld.fail(lt.err.empty() ? "missing tensor " + nm : lt.err); return; }
          out.insert(out.end(), v.begin(), v.end());
        }
      }
    };
    for (int li = 0; li < c.L && ld.ok; ++li) {
      LayerWeights& gw = m->lora.glayers[li];
      const LayerWeights& lw = m->layers[li];
      std::vector<float> w;
      if (c.arch == ARCH_MODERNBERT) {
        const std::string Lp = P + "layers." + std::to_string(li) + ".";
        std::vector<float> g_attn, g_mlp;
        if (lw.wqkv_f) ld.host_f32(Lp + "attn_norm.weight", g_attn, {H});
        if (lw.wi_f) ld.host_f32(Lp + "mlp_norm.weight", g_mlp, {H});
        stack({Lp + "attn.Wqkv.weight"}, 3 * H, H, w);
        if (!ld.ok) break;
        gw.wqkv = ld.up_f16(w);
        if (lw.wqkv_f) fold_weights(ld, w, g_attn, T * 3 * H, H, &gw.wqkv_f);
        stack({Lp + "attn.Wo.weight"}, H, H, w);
        if (!ld.ok) break;
        gw.wo = ld.up_f16(w);
        stack({Lp + "mlp.Wi.weight"}, 2 * I, H, w);
        if (!ld.ok) break;
        {   // GeGLU interleave inside every task's block (model_load)
          std::vector<float> perm(w.size());
          for (int t = 0; t < T; ++t) {
            const float* src = w.data() + static_cast<size_t>(t) * 2 * I * H;
            float* dst = perm.data() + static_cast<size_t>(t) * 2 * I * H;
            for (int j = 0; j < I / 32; ++j) {
              memcpy(dst + static_cast<size_t>(64 * j) * H, src + static_cast<size_t>(32 * j) * H, sizeof(float) * 32 * H);
              memcpy(dst + static_cast<size_t>(64 * j + 32) * H, src + static_cast<size_t>(I + 32 * j) * H, sizeof(float) * 32 * H);
            }
          }
          gw.wi = ld.up_f16(perm);
          if (lw.wi_f) fold_weights(ld, perm, g_mlp, T * 2 * I, H, &gw.wi_f);
        }
        stack({Lp + "mlp.Wo.weight"}, H, I, w);
        if (!ld.ok) break;
        gw.wo2 = ld.up_f16(w);
      } else {
        const std::string Lp = P + "encoder.layer." + std::to_string(li) + ".";
        stack({Lp + "attention.self.query.weight", Lp + "attention.self.key.weight", Lp + "attention.self.value.weight"}, H, H, w);
        if (!ld.ok) break;
        gw.wqkv = ld.up_f16(w);
        stack({Lp + "attention.output.dense.weight"}, H, H, w);
        if (!ld.ok) break;
        gw.wo = ld.up_f16(w);
        stack({Lp + "intermediate.dense.weight"}, I, H, w);
        if (!ld.ok) break;
        gw.wi = ld.up_f16(w);
        stack({Lp + "output.dense.weight"}, H, I, w);
        if (!ld.ok) break;
        gw.wo2 = ld.up_f16(w);
      }
    }
    m->lora.grouped = true;
  }
  for (int li = 0; li < c.L && ld.ok && !grouped; ++li) {
    LoraLayer& ll = m->lora.layers[li];
    const LayerWeights& lw = m->layers[li];
    if (c.arch == ARCH_MODERNBERT) {
      const std::string Lp = P + "layers." + std::to_string(li) + ".";
      std::vector<float> g_attn, g_mlp;
      if (lw.wqkv_f) ld.host_f32(Lp + "attn_norm.weight", g_attn, {H});
      if (lw.wi_f) ld.host_f32(Lp + "mlp_norm.weight", g_mlp, {H});
      build_lora_proj(ld, sts, alpha, {{Lp + "attn.Wqkv", 0, 3 * H}}, 3 * H, H, rp, g_attn, ident, ll.qkv);
      build_lora_proj(ld, sts, alpha, {{Lp + "attn.Wo", 0, H}}, H, H, rp, none, ident, ll.wo);
      build_lora_proj(ld, sts, alpha, {{Lp + "mlp.Wi", 0, 2 * I}}, 2 * I, H, rp, g_mlp, geglu_perm, ll.wi);
      build_lora_proj(ld, sts, alpha, {{Lp + "mlp.Wo", 0, H}}, H, I, rp, none, ident, ll.wo2);
    } else {
      const std::string Lp = P + "encoder.layer." + std::to_string(li) + ".";
      build_lora_proj(ld, sts, alpha, {{Lp + "attention.self.query", 0, H}, {Lp + "attention.self.key", H, H}, {Lp + "attention.self.value", 2 * H, H}},
                      3 * H, H, rp, none, ident, ll.qkv);
      build_lora_proj(ld, sts, alpha, {{Lp + "attention.output.dense", 0, H}}, H, H, rp, none, ident, ll.wo);
      build_lora_proj(ld, sts, alpha, {{Lp + "intermediate.dense", 0, I}}, I, H, rp, none, ident, ll.wi);
      build_lora_proj(ld, sts, alpha, {{Lp + "output.dense", 0, H}}, H, I, rp, none, ident, ll.wo2);
    }
    for (const LoraProj* lp : {&ll.qkv, &ll.wo, &ll.wi, &ll.wo2}) m->lora.max_R = std::max(m->lora.max_R, lp->R);
  }
  if (!ld.ok) { *err = ld.err; model_free(m); return nullptr; }
  for (int t = 0; t < T; ++t) {
    const int h = model_add_head(m, dirs[t], token_level[t], err);
    if (h < 0) { model_free(m); return nullptr; }
    m->lora.head_of_task.push_back(h);
  }
  m->lora.tasks = T;
  cudaDeviceSynchronize();
  return m;
}

// 1: <dir>/model.safetensors carries lora_A / lora_B tensors; 0: it does not; -1: unreadable
int checkpoint_has_adapters(const std::string& dir) {
  SafeTensors st;
  std::string err;
  if (!st.open(dir + "/model.safetensors", &err)) return -1;
  for (const auto& kv : st.tensors)
    if (kv.first.find(".lora_A.weight") != std::string::npos) return 1;
  return 0;
}

// fp32 host copy of one tensor of <dir>/model.safetensors (precise.cu builds its split weights from the originals)
bool load_host_tensor(const std::string& dir, const std::string& name, const std::vector<int64_t>& shape, std::vector<float>& out,
                      std::string* err) {
  static thread_local std::string cached_dir;
  static thread_local std::unique_ptr<SafeTensors> cached;
  if (!cached || cached_dir != dir) {
    cached.reset(new SafeTensors());
    cached_dir = dir;
    if (!cached->open(dir + "/model.safetensors", err)) { cached.reset(); return false; }
  }
  const StTensor* t = cached->find(name);
  if (!t) { *err = "missing tensor " + name; return false; }
  if (t->shape != shape) { *err = "tensor " + name + " has an unexpected shape"; return false; }
  if (!to_f32(*t, out)) { *err = "tensor " + name + " has unsupported dtype " + t->dtype; return false; }
  return lora_fold(*cached, name, *t, lora_alpha_of(dir), out, err);   // same merged matrix the production weights hold
}
std::string modernbert_prefix(const std::string& dir) {
  std::string err;
  std::vector<float> tmp;
  const char* prefixes[] = {"model.", "_orig_mod.model.", "", "_orig_mod."};
  SafeTensors st;
  if (!st.open(dir + "/model.safetensors", &err)) return "model.";
  for (const char* p : prefixes)
    if (st.find(std::string(p) + "embeddings.tok_embeddings.weight")) return p;
  return "model.";
}

void model_free(Model* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  if (m->stream) { cudaStreamSynchronize(m->stream); cudaStreamDestroy(m->stream); }
  precise_free(*m);
  for (void* p : m->allocs) cudaFree(p);
  Workspace& w = m->ws;
  void* dev[] = {w.x, w.h, w.lo, w.qkv, w.ctx, w.mid, w.ids, w.pos, w.cu, w.pooled, w.pool_part, w.pool_arrived, w.logits, w.probs, w.cls, w.conf, w.emb, w.row_stats, w.kv_lens, w.lora_u};
  for (void* p : dev) if (p) cudaFree(p);
  void* host[] = {w.h_ids, w.h_cu, w.h_out, w.h_cls, w.h_conf};
  for (void* p : host) if (p) cudaFreeHost(p);
  delete m;
}

// ------------------------------------------------------------------------------------------------
// workspace
// ------------------------------------------------------------------------------------------------
namespace {
template <typename T>
int regrow(T*& p, size_t n) {
  if (p) cudaFree(p);
  p = nullptr;
  return cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T)) == cudaSuccess ? 0 : -1;
}
template <typename T>
int regrow_host(T*& p, size_t n) {
  if (p) cudaFreeHost(p);
  p = nullptr;
  return cudaMallocHost(reinterpret_cast<void**>(&p), n * sizeof(T)) == cudaSuccess ? 0 : -1;
}
}  // namespace

int workspace_reserve(Model& m, int tokens, int seqs, size_t out_elems) {
  Workspace& w = m.ws;
  const int H = m.cfg.H;
  const int Imid = m.cfg.I > H ? m.cfg.I : H;
  int rc = 0;
  if (tokens > w.cap_tokens) {
    cudaStreamSynchronize(m.stream);
    ++w.generation;
    // round up so that TMA boxes of 128 rows never leave the allocation
    const size_t T = (static_cast<size_t>(tokens) + 127) / 128 * 128;
    rc |= regrow(w.x, T * H);
    rc |= regrow(w.h, T * H);
    rc |= regrow(w.lo, T * H);
    const size_t Hq = static_cast<size_t>(m.cfg.attn_w > H ? m.cfg.attn_w : H);   // padded heads (MiniLM) widen q/k/v/ctx
    rc |= regrow(w.qkv, T * 3 * Hq);
    rc |= regrow(w.ctx, T * Hq);
    rc |= regrow(w.mid, T * Imid);
    rc |= regrow(w.ids, T);
    rc |= regrow(w.pos, T);
    rc |= regrow(w.row_stats, 2 * (T * (2 * static_cast<size_t>(H / 128 > 0 ? H / 128 : 1) + 1) + 4));
    if (m.lora.max_R > 0) rc |= regrow(w.lora_u, T * static_cast<size_t>(m.lora.max_R));
    w.cap_tokens = rc ? 0 : static_cast<int>(T);
  }
  if (seqs > w.cap_seqs) {
    cudaStreamSynchronize(m.stream);
    ++w.generation;
    const size_t B = (static_cast<size_t>(seqs) + 63) / 64 * 64;
    rc |= regrow(w.cu, B + 1);
    rc |= regrow(w.kv_lens, B);
    rc |= regrow(w.pooled, B * H);
    rc |= regrow(w.pool_part, B * kPoolParts * H);
    rc |= regrow(w.pool_arrived, B);
    if (!rc) rc |= cudaMemset(w.pool_arrived, 0, B * sizeof(int)) == cudaSuccess ? 0 : -1;
    rc |= regrow(w.emb, B * H);
    w.cap_seqs = rc ? 0 : static_cast<int>(B);
  }
  if (out_elems > w.out_elems) {
    cudaStreamSynchronize(m.stream);
    ++w.generation;
    rc |= regrow(w.logits, out_elems);
    rc |= regrow(w.probs, out_elems);
    w.out_elems = rc ? 0 : out_elems;
  }
  const int rows = tokens > seqs ? tokens : seqs;
  static_assert(sizeof(int) == 4, "int32");
  if (!w.cls || rows > w.h_cap_tokens) {  // cls/conf sized by rows (tokens for token heads)
    cudaStreamSynchronize(m.stream);
    ++w.generation;
    rc |= regrow(w.cls, static_cast<size_t>(rows));
    rc |= regrow(w.conf, static_cast<size_t>(rows));
    rc |= regrow_host(w.h_ids, static_cast<size_t>(rows));
    rc |= regrow_host(w.h_cls, static_cast<size_t>(rows));
    rc |= regrow_host(w.h_conf, static_cast<size_t>(rows));
    w.h_cap_tokens = rc ? 0 : rows;
  }
  if (seqs > w.h_cap_seqs) {
    cudaStreamSynchronize(m.stream);
    rc |= regrow_host(w.h_cu, static_cast<size_t>(seqs) + 1);
    w.h_cap_seqs = rc ? 0 : seqs;
  }
  const size_t want_out = out_elems > static_cast<size_t>(seqs) * H ? out_elems : static_cast<size_t>(seqs) * H;
  if (want_out > w.h_out_elems) {
    cudaStreamSynchronize(m.stream);
    rc |= regrow_host(w.h_out, 2 * want_out);
    w.h_out_elems = rc ? 0 : want_out;
  }
  if (rc) fprintf(stderr, "[srb200] workspace allocation failed (tokens=%d seqs=%d)\n", tokens, seqs);
  return rc;
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
// SRB_RESID_HL=0 keeps the fp32 residual stream + fp16 copy on the LayerNorm-fold path (A/B measurements)
static bool resid_hl_enabled() {
  static const bool on = [] {
    const char* e = getenv("SRB_RESID_HL");
    return !(e && e[0] == '0');
  }();
  return on;
}

int encoder_forward(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int num_layers) {
  if (m.precise.on) return encoder_forward_precise(m, d_ids, d_cu, B, T, max_len, num_layers);
  const EncoderConfig& c = m.cfg;
  Workspace& w = m.ws;
  cudaStream_t s = m.stream;
  const int H = c.H, I = c.I;
  if (T > w.cap_tokens || B > w.cap_seqs) return -1;
  if (c.arch == ARCH_MODERNBERT && max_len > m.rope_len) {
    fprintf(stderr, "[srb200] sequence length %d exceeds max_position_embeddings %d\n", max_len, m.rope_len);
    return -1;
  }
  if (c.arch == ARCH_BERT && max_len > c.max_pos) {
    fprintf(stderr, "[srb200] sequence length %d exceeds max_position_embeddings %d\n", max_len, c.max_pos);
    return -1;
  }
  const int L = (num_layers <= 0 || num_layers > c.L) ? c.L : num_layers;
  if (compute_positions(s, d_cu, B, w.pos)) return -1;
  GemmDesc g;
  g.M = T;
  g.a_rows = w.cap_tokens;
  // shared-LoRA pass (engine.h: LoraShared): U = A-operand x a^T with every row keeping its own task's block, then the
  // projection takes U b^T as a K extension of its accumulator
  const bool lora_on = m.lora.tasks > 0 && m.lora.rows_per_task > 0;
  if (lora_on && (T != m.lora.tasks * m.lora.rows_per_task || (!m.lora.grouped && !w.lora_u))) return -1;
  auto lora_ext = [&](GemmDesc& gd, const LoraProj& lp, bool folded_form, int cat) {
    if (!lora_on || !lp.b) return 0;
    GemmDesc u;
    u.M = T; u.a_rows = w.cap_tokens; u.N = lp.R; u.K = gd.K; u.A = gd.A; u.W = folded_form ? lp.a_f : lp.a;
    u.out = w.lora_u; u.ldo = lp.R; u.epi = EPI_F16;
    u.mask_block = lp.block; u.mask_rows = m.lora.rows_per_task;
    if (!u.W) return -1;
    { ProfScope ps(m, cat); if (gemm_f16(s, u)) return -1; }
    gd.A2 = w.lora_u; gd.W2 = lp.b; gd.K2 = lp.R;
    return 0;
  };
  const LoraLayer no_lora;
  // grouped form: every projection GEMM picks the task's matrix per row block (gemm.h: w_groups)
  const bool grouped = lora_on && m.lora.grouped;
  if (grouped && (m.lora.rows_per_task % 256 != 0 || static_cast<int>(m.lora.glayers.size()) != c.L)) return -1;
  auto run_proj = [&](GemmDesc& gd) {
    if (grouped) { gd.w_groups = m.lora.tasks; gd.w_group_rows = m.lora.rows_per_task; }
    return gemm_f16(s, gd);
  };
  if (c.arch == ARCH_MODERNBERT) {
    // Residual stream as an fp16 pair (gemm.h: EPI_RESID_HL) whenever every LayerNorm of the stack is folded: w.h / w.lo hold
    // x - pivot, the residual GEMMs update the pair in place, and the fp32 form is rebuilt once after the last layer.
    bool hl = resid_hl_enabled() && w.lo != nullptr;
    for (int li = 0; li < c.L && hl; ++li) hl = m.layers[li].wi_f != nullptr && (li == 0 || m.layers[li].wqkv_f != nullptr);
    { ProfScope ps(m, PC_EMBED);
      if (embed_ln_modernbert(s, d_ids, T, H, c.vocab, m.emb_word, m.emb_ln_w, c.ln_eps, hl ? nullptr : w.x, w.h, hl ? w.lo : nullptr)) return -1; }
    // LayerNorm fold (gemm.h): the residual GEMM that finishes x also leaves fp16(x) in w.h and the per-row
    // (sum, sum of squares) in w.row_stats; the projection that consumes LN(x) multiplies the raw rows with
    // W diag(gamma) and corrects per row in its epilogue -- no LayerNorm pass over the fp32 stream.
    // `folded` says which of the two forms w.h currently holds.
    bool folded = false;
    // one statistics record, padded so that the second record keeps the float2 alignment of the partials
    const size_t rec = (static_cast<size_t>(T) * (2 * static_cast<size_t>(H / 128) + 1) + 3) & ~static_cast<size_t>(3);
    int n_rec = 0;                 // records written so far in this forward (ping-pong between the two)
    const float* cur_stats = nullptr;
    auto emit_for = [&](GemmDesc& gd, bool want) {   // make this residual GEMM produce the fold operands
      if (!want) return 0;
      float* dst = w.row_stats + (n_rec & 1) * rec;
      gd.row_stats = dst;                                   // [H/128][T][2] partials, every one overwritten
      gd.pivot_out = dst + static_cast<size_t>(T) * 2 * (H / 128);
      if (n_rec > 0) {                                      // pivot = the row mean after the previous residual GEMM
        const float* prev = w.row_stats + ((n_rec - 1) & 1) * rec;
        gd.pivot_in_stats = prev;
        gd.pivot_in = prev + static_cast<size_t>(T) * 2 * (H / 128);
      }
      if (hl) { gd.epi = EPI_RESID_HL; gd.out = w.h; gd.lo16 = w.lo; gd.resid = nullptr; gd.ldr = 0; }
      else gd.raw16 = w.h;
      cur_stats = dst;
      ++n_rec;
      return 0;
    };
    for (int li = 0; li < L; ++li) {
      const LayerWeights& lw = grouped ? m.lora.glayers[li] : m.layers[li];
      const LoraLayer& ll = lora_on ? m.lora.layers[li] : no_lora;
      const bool local = (li % c.global_every) != 0;
      if (folded) {
        // w.h = fp16(x) and w.row_stats were written by the previous layer's MLP-out GEMM
      } else if (lw.attn_norm_w) {
        ProfScope ps(m, PC_NORM);
        if (layernorm_rows(s, w.x, T, H, lw.attn_norm_w, nullptr, c.ln_eps, nullptr, w.h)) return -1;
      } else if (li != 0) {
        ProfScope ps(m, PC_NORM);
        if (cast_rows_f16(s, w.x, static_cast<size_t>(T) * H, w.h)) return -1;
      }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = 3 * H; g.K = H; g.A = w.h; g.W = lw.wqkv; g.out = w.qkv; g.ldo = 3 * H;
      if (folded) { g.W = lw.wqkv_f; g.fold_stats = cur_stats; g.fold_eps = c.ln_eps; g.fold_h = H; }
      g.epi = EPI_ROPE; g.pos = w.pos; g.rope_cols = 2 * H;
      g.rope_cos = local ? m.rope_cos_l : m.rope_cos_g;
      g.rope_sin = local ? m.rope_sin_l : m.rope_sin_g;
      if (lora_ext(g, ll.qkv, folded, PC_GEMM_QKV)) return -1;
      { ProfScope ps(m, PC_GEMM_QKV); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_ATTN);   // sliding-window layers visit only the key blocks inside the window
        if (attention_wgmma_fwd(s, w.qkv, w.ctx, d_cu, B, max_len, c.heads, 64, local ? c.local_attention / 2 : 0)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = H; g.A = w.ctx; g.W = lw.wo; g.out = w.x; g.ldo = H;
      g.epi = EPI_RESID; g.resid = w.x; g.ldr = H;
      const bool fold_mlp = lw.wi_f != nullptr;
      if (emit_for(g, fold_mlp || hl)) return -1;
      if (lora_ext(g, ll.wo, false, PC_GEMM_WO)) return -1;
      { ProfScope ps(m, PC_GEMM_WO); if (run_proj(g)) return -1; }
      if (!fold_mlp) { ProfScope ps(m, PC_NORM); if (layernorm_rows(s, w.x, T, H, lw.mid_norm_w, nullptr, c.ln_eps, nullptr, w.h)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = 2 * I; g.K = H; g.A = w.h; g.W = lw.wi; g.out = w.mid; g.ldo = I;
      if (fold_mlp) { g.W = lw.wi_f; g.fold_stats = cur_stats; g.fold_eps = c.ln_eps; g.fold_h = H; }
      g.epi = EPI_GEGLU;
      if (lora_ext(g, ll.wi, fold_mlp, PC_GEMM_WI)) return -1;
      { ProfScope ps(m, PC_GEMM_WI); if (run_proj(g)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = I; g.A = w.mid; g.W = lw.wo2; g.out = w.x; g.ldo = H;
      g.epi = EPI_RESID; g.resid = w.x; g.ldr = H;
      // the next layer's attn_norm rides on this GEMM (the last executed layer feeds final_norm, which the heads fuse)
      folded = li + 1 < L && m.layers[li + 1].wqkv_f != nullptr;
      if (emit_for(g, folded || hl)) return -1;
      if (lora_ext(g, ll.wo2, false, PC_GEMM_WO2)) return -1;
      { ProfScope ps(m, PC_GEMM_WO2); if (run_proj(g)) return -1; }
    }
    if (hl) {   // x = pivot + hi + lo for the heads (final_norm, pooling, token heads read the fp32 stream)
      ProfScope ps(m, PC_NORM);
      const float* piv = n_rec > 0 ? w.row_stats + ((n_rec - 1) & 1) * rec + static_cast<size_t>(T) * 2 * (H / 128) : nullptr;
      if (hl_to_f32(s, w.h, w.lo, piv, T, H, w.x)) return -1;
    }
  } else {
    ProfScope ps_embed(m, PC_EMBED);
    if (embed_ln_bert(s, d_ids, w.pos, T, H, c.vocab, c.max_pos, m.emb_word, m.emb_pos, m.emb_type0, m.emb_ln_w,
                      m.emb_ln_b, c.ln_eps, w.x, w.h))
      return -1;
    for (int li = 0; li < L; ++li) {
      const LayerWeights& lw = grouped ? m.lora.glayers[li] : m.layers[li];
      const LoraLayer& ll = lora_on ? m.lora.layers[li] : no_lora;
      g = GemmDesc();
      const int Hq = c.attn_w;   // == H unless the heads were padded (MiniLM)
      g.M = T; g.a_rows = w.cap_tokens; g.N = 3 * Hq; g.K = H; g.A = w.h; g.W = lw.wqkv; g.out = w.qkv; g.ldo = 3 * Hq;
      g.epi = EPI_F16; g.bias = lw.bqkv;
      if (lora_ext(g, ll.qkv, false, PC_GEMM_QKV)) return -1;
      { ProfScope ps(m, PC_GEMM_QKV); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_ATTN); if (attention_wgmma_fwd(s, w.qkv, w.ctx, d_cu, B, max_len, c.heads, 64, 0, m.cur_kv_lens)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = Hq; g.A = w.ctx; g.W = lw.wo; g.out = w.x; g.ldo = H;
      g.epi = EPI_RESID; g.resid = w.x; g.ldr = H; g.bias = lw.bo;
      if (lora_ext(g, ll.wo, false, PC_GEMM_WO)) return -1;
      { ProfScope ps(m, PC_GEMM_WO); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_NORM); if (layernorm_rows(s, w.x, T, H, lw.mid_norm_w, lw.mid_norm_b, c.ln_eps, w.x, w.h)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = I; g.K = H; g.A = w.h; g.W = lw.wi; g.out = w.mid; g.ldo = I;
      g.epi = EPI_GELU; g.bias = lw.bi;
      if (lora_ext(g, ll.wi, false, PC_GEMM_WI)) return -1;
      { ProfScope ps(m, PC_GEMM_WI); if (run_proj(g)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = I; g.A = w.mid; g.W = lw.wo2; g.out = w.x; g.ldo = H;
      g.epi = EPI_RESID; g.resid = w.x; g.ldr = H; g.bias = lw.bo2;
      if (lora_ext(g, ll.wo2, false, PC_GEMM_WO2)) return -1;
      { ProfScope ps(m, PC_GEMM_WO2); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_NORM); if (layernorm_rows(s, w.x, T, H, lw.out_norm_w, lw.out_norm_b, c.ln_eps, w.x, w.h)) return -1; }
    }
  }
  return 0;
}

int head_sequence(Model& m, int head, const int* d_cu, int B, int pooler_mode) {
  if (head < 0 || head >= static_cast<int>(m.heads.size())) return -1;
  const Head& hd = m.heads[head];
  const EncoderConfig& c = m.cfg;
  Workspace& w = m.ws;
  if (static_cast<size_t>(B) * hd.num_classes > w.out_elems) return -1;
  SeqHeadWeights sw;
  sw.cls_w = hd.cls_w; sw.cls_b = hd.cls_b; sw.num_classes = hd.num_classes;
  if (c.arch == ARCH_MODERNBERT) {
    // always MEAN pooling over final_norm(hidden) (traditional/modernbert.rs:818,1146-1169)
    const bool hf = m.head_flavor == 1;
    if (pool_rows(m.stream, w.x, d_cu, B, c.H, (hf && c.cls_pooling == 0) ? POOL_CLS : POOL_MEAN, m.final_norm_w, nullptr,
                  c.ln_eps, w.pooled, w.pool_part, w.pool_arrived))
      return -1;
    sw.dense_mode = hd.has_dense ? 1 : 0;
    sw.dense_w = hd.dense_w32; sw.norm_w = hd.norm_w;
    sw.argmax_last = hf ? 1 : 0;
    sw.gelu_erf = hf ? 1 : 0;
    sw.head_eps = hf ? c.ln_eps : 1e-12f;
  } else {
    if (pool_rows(m.stream, w.x, d_cu, B, c.H, POOL_CLS, nullptr, nullptr, 0.f, w.pooled, w.pool_part, w.pool_arrived)) return -1;
    sw.dense_mode = hd.has_dense ? (pooler_mode == 1 ? 2 : 3) : 0;
    sw.dense_w = hd.dense_w32; sw.dense_b = hd.dense_b;
    sw.argmax_last = 1;
  }
  return seq_head(m.stream, w.pooled, B, c.H, sw, w.logits, w.probs, w.cls, w.conf);
}

int head_tokens(Model& m, int head, int B, int T, int row0) {
  (void)B;
  if (head < 0 || head >= static_cast<int>(m.heads.size())) return -1;
  const Head& hd = m.heads[head];
  const EncoderConfig& c = m.cfg;
  Workspace& w = m.ws;
  if (static_cast<size_t>(T) * hd.num_classes > w.out_elems || row0 < 0 || row0 + T > w.cap_tokens) return -1;
  const size_t off = static_cast<size_t>(row0) * c.H;   // the head reads rows [row0, row0 + T) of the hidden states
  const float* x = w.x + off;
  if (c.arch == ARCH_MODERNBERT) {
    if (hd.has_dense) {
      // final_norm -> fp16, head.dense on the wgmma GEMM, then gelu/LN/classifier per token
      if (layernorm_rows(m.stream, x, T, c.H, m.final_norm_w, nullptr, c.ln_eps, nullptr, w.h + off)) return -1;
      GemmDesc g;
      g.M = T; g.a_rows = w.cap_tokens - row0; g.N = c.H; g.K = c.H; g.A = w.h + off; g.W = hd.dense_w16; g.out = w.ctx + off; g.ldo = c.H;
      g.epi = EPI_F16;
      if (gemm_f16(m.stream, g)) return -1;
      const bool hf = m.head_flavor == 1;
      return token_head(m.stream, nullptr, w.ctx + off, T, c.H, hd.norm_w, nullptr, 0.f, hd.cls_w, hd.cls_b, hd.num_classes,
                        hf ? 1 : 0, w.logits, w.probs, w.cls, w.conf, hf ? 1 : 0, hf ? c.ln_eps : 1e-12f);
    }
    return token_head(m.stream, x, nullptr, T, c.H, nullptr, m.final_norm_w, c.ln_eps, hd.cls_w, hd.cls_b,
                      hd.num_classes, 0, w.logits, w.probs, w.cls, w.conf);
  }
  return token_head(m.stream, x, nullptr, T, c.H, nullptr, nullptr, 0.f, hd.cls_w, hd.cls_b, hd.num_classes, 1,
                    w.logits, w.probs, w.cls, w.conf);
}

int head_embedding(Model& m, const int* d_cu, int B, int dim, float norm_eps) {
  const EncoderConfig& c = m.cfg;
  Workspace& w = m.ws;
  if (dim <= 0 || dim > c.H) dim = c.H;
  if (c.arch == ARCH_MODERNBERT) {
    if (pool_rows(m.stream, w.x, d_cu, B, c.H, POOL_MEAN, m.final_norm_w, nullptr, c.ln_eps, w.pooled, w.pool_part, w.pool_arrived)) return -1;
  } else {
    if (pool_rows(m.stream, w.x, d_cu, B, c.H, POOL_MEAN, nullptr, nullptr, 0.f, w.pooled, w.pool_part, w.pool_arrived, m.cur_kv_lens)) return -1;
  }
  return l2_normalize_rows(m.stream, w.pooled, B, c.H, dim, norm_eps, w.emb);
}

}  // namespace srb
