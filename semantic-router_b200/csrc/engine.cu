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
#include <array>
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
  SafeTensors() = default;
  SafeTensors(const SafeTensors&) = delete;   // owns the mapping
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
    if (hlen > size - 8) { *err = path + ": safetensors header exceeds file"; return false; }
    Json hdr;
    JsonParser jp(reinterpret_cast<const char*>(base + 8), hlen);
    if (!jp.parse(hdr) || !hdr.is_obj()) { *err = path + ": safetensors header is not JSON"; return false; }
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
      if (!(bd >= 0.0) || !(ed >= bd) || ed > static_cast<double>(room)) { *err = path + ": tensor " + kv.first + " out of bounds"; return false; }
      const size_t b = static_cast<size_t>(bd), e = static_cast<size_t>(ed);
      if (e > room || e < b) { *err = path + ": tensor " + kv.first + " out of bounds"; return false; }
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
    m->weight_bytes += bytes;
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
  bool merge_lora(const std::string& name, const StTensor& base, std::vector<float>& w) {
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

// Tensor-name prefix of the encoder in a checkpoint.  ModernBERT: the first prefix the reference loaders try whose
// tok_embeddings exist.  BERT: "bert." or "" by its word_embeddings or, in a head-only checkpoint, by its pooler.
// false: no encoder embeddings under any known prefix.
bool tensor_prefix(const SafeTensors& st, Arch arch, std::string& P) {
  if (arch == ARCH_MODERNBERT) {
    for (const char* p : {"model.", "_orig_mod.model.", "", "_orig_mod."})
      if (st.find(std::string(p) + "embeddings.tok_embeddings.weight")) { P = p; return true; }
    P.clear();
    return false;
  }
  if (st.find("bert.embeddings.word_embeddings.weight")) { P = "bert."; return true; }
  if (st.find("embeddings.word_embeddings.weight")) { P.clear(); return true; }
  P = st.find("bert.pooler.dense.weight") ? "bert." : "";
  return false;
}

std::string layer_prefix(const EncoderConfig& c, const std::string& P, int li) {
  return P + (c.arch == ARCH_MODERNBERT ? "layers." : "encoder.layer.") + std::to_string(li) + ".";
}

// config.json and the checkpoint's tensor names -> the encoder's shape and its tensor-name prefix P.  false: *err says why
// the checkpoint cannot be served.  Host only.
bool read_encoder_config(const Json& cfgj, const SafeTensors& st, EncoderConfig& c, std::string& P, std::string* err) {
  std::string e;
  const std::string mt = cfgj.str_or("model_type", "");
  c.arch = (mt == "modernbert" || tensor_prefix(st, ARCH_MODERNBERT, P)) ? ARCH_MODERNBERT : ARCH_BERT;
  if (!tensor_prefix(st, c.arch, P))
    e = c.arch == ARCH_MODERNBERT ? "no tok_embeddings tensor under any known prefix" : "no BERT word_embeddings tensor found";
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
  if (e.empty() && (c.H <= 0 || c.L <= 0 || c.heads <= 0 || c.vocab <= 0 || c.I <= 0)) e = "config.json incomplete";
  const int head_dim = (c.heads > 0) ? c.H / c.heads : 0;
  if (e.empty() && (c.H % (c.heads > 0 ? c.heads : 1) != 0 || !(head_dim == 64 || (head_dim == 32 && c.arch == ARCH_BERT))))
    e = "head_dim " + std::to_string(head_dim) + " unsupported (64; 32 for BERT/MiniLM encoders)";
  c.attn_w = c.heads * 64;
  if (e.empty() && !(c.H == 384 || c.H == 768 || c.H == 1024)) e = "hidden_size unsupported";
  // gemm_f16 refuses EPI_GEGLU unless N = 2 I is a multiple of 128 (its host check, not the tile walk: the kernel stores
  // 64-column (a | b) groups one by one).  Whether that check can be relaxed is unmeasured; until then such a model is
  // refused here instead of failing in every forward.
  if (e.empty() && c.arch == ARCH_MODERNBERT && c.I % 64 != 0) e = "intermediate_size must be a multiple of 64";
  if (!e.empty()) { *err = e; return false; }
  return true;
}

// The load's device step: an sm_90 device at index `device`, made current
bool use_device(int device, std::string* err) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    *err = "no CUDA device available (this library has no CPU path)";
    return false;
  }
  if (device < 0 || device >= ndev) { *err = "invalid device index " + std::to_string(device); return false; }
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  if (prop.major != 9 || prop.minor != 0) {
    *err = std::string("device ") + prop.name + " is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) +
           "; this library is built for sm_90a only";
    return false;
  }
  if (cudaSetDevice(device) != cudaSuccess) { *err = "cudaSetDevice failed"; return false; }
  return true;
}

// One encoder projection: how the checkpoint stores it and how the kernels read it.
struct Segment {        // `stem`.weight [rows, K] fills source rows [row0, row0 + rows); its device rows carry `scale`
  std::string stem;
  int row0, rows;
  float scale;
};
struct Projection {
  std::vector<Segment> segs;
  int N = 0, K = 0;                  // source shape
  bool bias = false;                 // BERT: `stem`.bias [rows] beside every segment's weight
  int dN = 0, dK = 0;                // device shape
  std::vector<int> row_of, col_of;   // source row / column -> device row / column; empty: identity
  std::string gamma;                 // LayerNorm weight the device weight is folded with (fold_weights); empty: none
};
Projection projection(std::vector<Segment> segs, int N, int K) {
  Projection p;
  p.segs = std::move(segs);
  p.N = p.dN = N;
  p.K = p.dK = K;
  return p;
}

// The four projections of layer li in the order qkv, attention output, intermediate, output (PreciseLayer).
std::array<Projection, 4> layer_projections(const EncoderConfig& c, const std::string& P, int li, bool has_attn_norm) {
  const int H = c.H, I = c.I;
  const std::string Lp = layer_prefix(c, P, li);
  std::array<Projection, 4> pr;
  if (c.arch == ARCH_MODERNBERT) {
    pr[0] = projection({{Lp + "attn.Wqkv", 0, 3 * H, 1.f}}, 3 * H, H);
    pr[1] = projection({{Lp + "attn.Wo", 0, H, 1.f}}, H, H);
    pr[2] = projection({{Lp + "mlp.Wi", 0, 2 * I, 1.f}}, 2 * I, H);
    pr[3] = projection({{Lp + "mlp.Wo", 0, H, 1.f}}, H, I);
    // Wqkv runs LayerNorm-folded where its attn_norm follows a residual GEMM; layer 0 and layers without attn_norm
    // multiply the plain weight (encoder_forward).  Wi always runs folded with mlp_norm.
    if (li > 0 && has_attn_norm) pr[0].gamma = Lp + "attn_norm.weight";
    pr[2].gamma = Lp + "mlp_norm.weight";
    // GeGLU interleave for the fused epilogue: 32-row groups [a(32j..) | b(32j..)] (gemm.h EPI_GEGLU)
    pr[2].row_of.resize(static_cast<size_t>(2) * I);
    for (int j = 0; j < I / 32; ++j)
      for (int i = 0; i < 32; ++i) {
        pr[2].row_of[32 * j + i] = 64 * j + i;
        pr[2].row_of[I + 32 * j + i] = 64 * j + 32 + i;
      }
    return pr;
  }
  // MiniLM: heads of 32 are zero-padded to 64 (EncoderConfig::attn_w).  The kernels scale scores by 64^-0.5; the model
  // wants 32^-0.5, so the query rows carry the missing sqrt(2).
  const bool padded = c.attn_w != H;
  const float qs = padded ? 1.41421356237309504880f : 1.f;
  pr[0] = projection({{Lp + "attention.self.query", 0, H, qs}, {Lp + "attention.self.key", H, H, 1.f},
                      {Lp + "attention.self.value", 2 * H, H, 1.f}}, 3 * H, H);
  pr[1] = projection({{Lp + "attention.output.dense", 0, H, 1.f}}, H, H);
  pr[2] = projection({{Lp + "intermediate.dense", 0, I, 1.f}}, I, H);
  pr[3] = projection({{Lp + "output.dense", 0, H, 1.f}}, H, I);
  for (Projection& p : pr) p.bias = true;
  if (padded) {   // q / k / v rows (h*64 + d) <- (h*32 + d); the attention output reads the padded context columns
    const int hd = H / c.heads;
    pr[0].dN = 3 * c.attn_w;
    pr[1].dK = c.attn_w;
    pr[1].col_of.resize(H);
    pr[0].row_of.resize(static_cast<size_t>(3) * H);
    for (int i = 0; i < H; ++i) {
      pr[1].col_of[i] = i / hd * 64 + i % hd;
      for (int s = 0; s < 3; ++s) pr[0].row_of[s * H + i] = s * c.attn_w + pr[1].col_of[i];
    }
  }
  return pr;
}

// Source-order host weight of a projection (its segments stacked, adapters merged unless the loader keeps them) and,
// when `bias` is given, its bias
bool read_projection(Loader& ld, const Projection& pr, std::vector<float>& w, std::vector<float>* bias) {
  std::vector<float> v;
  w.clear();
  for (const Segment& s : pr.segs) {
    if (!ld.host_f32(s.stem + ".weight", v, {s.rows, pr.K})) return false;
    w.insert(w.end(), v.begin(), v.end());
  }
  if (bias) {
    bias->clear();
    for (const Segment& s : pr.segs) {
      if (!ld.host_f32(s.stem + ".bias", v, {s.rows})) return false;
      bias->insert(bias->end(), v.begin(), v.end());
    }
  }
  return true;
}

// read_projection, then into the device layout: rows through row_of, columns through col_of, times the segment's scale,
// zeros where no source element lands
bool device_projection(Loader& ld, const Projection& pr, std::vector<float>& w, std::vector<float>* bias) {
  if (!read_projection(ld, pr, w, bias)) return false;
  std::vector<float> dw(static_cast<size_t>(pr.dN) * pr.dK, 0.f), db(bias ? pr.dN : 0, 0.f);
  for (const Segment& s : pr.segs)
    for (int n = s.row0; n < s.row0 + s.rows; ++n) {
      const size_t r = pr.row_of.empty() ? n : pr.row_of[n];
      for (int k = 0; k < pr.K; ++k)
        dw[r * pr.dK + (pr.col_of.empty() ? k : pr.col_of[k])] = w[static_cast<size_t>(n) * pr.K + k] * s.scale;
      if (bias) db[r] = (*bias)[n] * s.scale;
    }
  w.swap(dw);
  if (bias) bias->swap(db);
  return true;
}

// W'' = W diag(gamma), every row re-centred to sum zero, rounded to fp16.  Two refinement passes push the sum of the
// ROUNDED row (what the tensor core multiplies) from ~1e-4 down to the last bit of its largest elements, so the
// residual mean * sum(W''[n,:]) is far below the fp16 rounding of the output.
std::vector<float> fold_weights(const std::vector<float>& w, const std::vector<float>& gamma, int n, int k) {
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
  return wf;
}

// device_projection, then folded with the projection's LayerNorm gamma when it names one: the fp32 host form of what the
// device multiplies
bool device_weight(Loader& ld, const Projection& pr, std::vector<float>& w, std::vector<float>* bias) {
  if (!device_projection(ld, pr, w, bias)) return false;
  if (pr.gamma.empty()) return true;
  std::vector<float> g;
  if (!ld.host_f32(pr.gamma, g, {pr.dK})) return false;
  w = fold_weights(w, g, pr.dN, pr.dK);
  return true;
}

// fp16 upload of projection p of a layer (the device weights of one task, or of several stacked along N) into its plain
// or its folded slot, and of its bias
void store_projection(Loader& ld, const Projection& pr, int p, const std::vector<float>& w, const std::vector<float>& b,
                      LayerWeights& lw) {
  __half** plain[] = {&lw.wqkv, &lw.wo, &lw.wi, &lw.wo2};
  float** biases[] = {&lw.bqkv, &lw.bo, &lw.bi, &lw.bo2};
  *(pr.gamma.empty() ? plain[p] : (p == 0 ? &lw.wqkv_f : &lw.wi_f)) = ld.up_f16(w);
  if (pr.bias) *biases[p] = ld.up_f32(b);
}

// ModernBERT's rotary tables for both thetas, max_position_embeddings rows
void load_rope(Loader& ld, Model& m) {
  const EncoderConfig& c = m.cfg;
  std::vector<float> cs, sn;
  rope_tables(64, c.theta_global, c.max_pos, cs, sn);
  m.rope_cos_g = ld.up_f32(cs);
  m.rope_sin_g = ld.up_f32(sn);
  rope_tables(64, c.theta_local, c.max_pos, cs, sn);
  m.rope_cos_l = ld.up_f32(cs);
  m.rope_sin_l = ld.up_f32(sn);
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

bool is_head_tensor(const std::string& n) {
  return n.compare(0, 11, "classifier.") == 0 || n.compare(0, 5, "head.") == 0 || n.find("pooler.") != std::string::npos;
}

std::string num_text(double v) {
  char b[32];
  snprintf(b, sizeof b, "%.9g", v);
  return b;
}
// the EncoderConfig fields every task of a grouped model must share, by their config.json names
std::vector<std::pair<const char*, std::string>> shape_fields(const EncoderConfig& c) {
  return {{"architecture", c.arch == ARCH_MODERNBERT ? "modernbert" : "bert"},
          {"hidden_size", num_text(c.H)},
          {"num_hidden_layers", num_text(c.L)},
          {"num_attention_heads", num_text(c.heads)},
          {"intermediate_size", num_text(c.I)},
          {"vocab_size", num_text(c.vocab)},
          {"max_position_embeddings", num_text(c.max_pos)},
          {"global_attn_every_n_layers", num_text(c.global_every)},
          {"local_attention", num_text(c.local_attention)},
          {"global_rope_theta", num_text(c.theta_global)},
          {"local_rope_theta", num_text(c.theta_local)},
          {"layer_norm_eps", num_text(c.ln_eps)},
          {"classifier_pooling", c.cls_pooling ? "mean" : "cls"}};
}

bool has_adapter(const SafeTensors& st, const std::string& name) {
  const std::string suffix = ".weight";
  if (name.size() <= suffix.size() || name.compare(name.size() - suffix.size(), suffix.size(), suffix) != 0) return false;
  const std::string stem = name.substr(0, name.size() - suffix.size());
  return st.find(stem + ".lora_A.weight") || st.find(stem + ".lora_B.weight");
}

// One tensor of every task: names[t] in task t's checkpoint (the prefixes may differ).  A task whose tensor is bitwise
// that of an earlier task (neither with adapters) shares that task's device copy; `rows` > 0 keeps the first rows only.
// Missing and not required: null for that task.
std::vector<float*> load_each(std::vector<Loader>& lt, const std::vector<std::string>& names,
                              const std::vector<int64_t>& shape, bool required = true, int64_t rows = 0) {
  const size_t T = lt.size();
  std::vector<float*> out(T, nullptr);
  std::vector<float> v;
  for (size_t t = 0; t < T && lt[t].ok; ++t) {
    const SafeTensors& st = *lt[t].st;
    const StTensor* a = st.find(names[t]);
    if (!a && !required) continue;
    bool shared = false;
    for (size_t u = 0; u < t && a && !shared; ++u) {
      const StTensor* b = lt[u].st->find(names[u]);
      if (b && out[u] && a->dtype == b->dtype && a->shape == b->shape && a->bytes == b->bytes &&
          memcmp(a->data, b->data, a->bytes) == 0 && !has_adapter(st, names[t]) && !has_adapter(*lt[u].st, names[u])) {
        out[t] = out[u];
        shared = true;
      }
    }
    if (shared || !lt[t].host_f32(names[t], v, shape)) continue;
    if (rows > 0 && !shape.empty()) v.resize(static_cast<size_t>(rows) * (v.size() / shape[0]));
    out[t] = lt[t].up_f32(v);
  }
  return out;
}

// One checkpoint directory as the host reads it: config.json, the mapped safetensors file, the encoder shape and the
// tensor-name prefix
struct Checkpoint {
  std::string dir;
  Json cfgj;
  SafeTensors st;
  EncoderConfig cfg;
  std::string P;
};

// The load's host step.  false: *err names the directory and says why it cannot be served.
bool read_checkpoint(const std::string& dir, Checkpoint& ck, std::string* err) {
  ck.dir = dir;
  if (!parse_json_file(dir + "/config.json", ck.cfgj)) { *err = "cannot read " + dir + "/config.json"; return false; }
  if (!ck.st.open(dir + "/model.safetensors", err)) return false;
  if (read_encoder_config(ck.cfgj, ck.st, ck.cfg, ck.P, err)) return true;
  *err = dir + ": " + *err;
  return false;
}

// false: *err is the error of the first task whose upload failed, after its directory
bool tasks_ok(const std::vector<Checkpoint>& ck, const std::vector<Loader>& lt, std::string* err) {
  for (size_t t = 0; t < lt.size(); ++t)
    if (!lt[t].ok) { *err = ck[t].dir + ": " + lt[t].err; return false; }
  return true;
}

// The load's upload step, on the current device: a model of the tasks `ck` (host-read, one encoder shape) holding every
// task's embeddings and norms (Model::task; a tensor bitwise equal in every task once), the rotary tables, and every
// layer's projections -- each task's device weights (its own gamma folded in) and biases, stacked along N.  lt: one
// loader per task, left to the caller's heads.  null: *err says why.
Model* upload_tasks(const std::vector<Checkpoint>& ck, int device, std::vector<Loader>& lt, std::string* err) {
  const int T = static_cast<int>(ck.size());
  Model* m = new Model();
  m->device = device;
  m->dir = ck[0].dir;
  m->cfg = ck[0].cfg;
  const EncoderConfig& c = m->cfg;
  const int H = c.H;
  for (const Checkpoint& k : ck) {
    lt.push_back(Loader{m, &k.st});
    lt.back().lora_alpha = lora_alpha_of(k.dir);
  }
  auto ok = [&]() { return tasks_ok(ck, lt, err); };
  auto names = [&](const std::string& rest, int li = -1) {   // `rest` under every task's prefix (and layer li)
    std::vector<std::string> n(T);
    for (int t = 0; t < T; ++t) n[t] = (li < 0 ? ck[t].P : layer_prefix(c, ck[t].P, li)) + rest;
    return n;
  };
  std::vector<TaskTensors>& task = m->task;
  task.resize(T);
  for (TaskTensors& tt : task) tt.layers.resize(c.L);
  auto each = [&](std::vector<float*> v, float* TaskTensors::*f) { for (int t = 0; t < T; ++t) task[t].*f = v[t]; };
  auto each_layer = [&](std::vector<float*> v, int li, float* TaskNorms::*f) { for (int t = 0; t < T; ++t) task[t].layers[li].*f = v[t]; };
  if (c.arch == ARCH_MODERNBERT) {
    each(load_each(lt, names("embeddings.tok_embeddings.weight"), {c.vocab, H}), &TaskTensors::emb_word);
    each(load_each(lt, names("embeddings.norm.weight"), {H}), &TaskTensors::emb_ln_w);
    for (int li = 0; li < c.L && ok(); ++li) {
      each_layer(load_each(lt, names("attn_norm.weight", li), {H}, false), li, &TaskNorms::attn_w);
      each_layer(load_each(lt, names("mlp_norm.weight", li), {H}), li, &TaskNorms::mid_w);
      for (int t = 1; t < T && ok(); ++t)
        if ((task[t].layers[li].attn_w != nullptr) != (task[0].layers[li].attn_w != nullptr)) {
          *err = "layer " + std::to_string(li) + " has an attn_norm in " + ck[task[0].layers[li].attn_w ? 0 : t].dir +
                 " but not in " + ck[task[0].layers[li].attn_w ? t : 0].dir;
          model_free(m);
          return nullptr;
        }
    }
    each(load_each(lt, names("final_norm.weight"), {H}), &TaskTensors::final_norm_w);
    if (ok()) load_rope(lt[0], *m);
  } else {
    each(load_each(lt, names("embeddings.word_embeddings.weight"), {c.vocab, H}), &TaskTensors::emb_word);
    each(load_each(lt, names("embeddings.position_embeddings.weight"), {c.max_pos, H}), &TaskTensors::emb_pos);
    // token_type_ids are always zero (traditional/bert.rs:227): row 0 only
    each(load_each(lt, names("embeddings.token_type_embeddings.weight"), {c.type_vocab, H}, true, 1), &TaskTensors::emb_type0);
    each(load_each(lt, names("embeddings.LayerNorm.weight"), {H}), &TaskTensors::emb_ln_w);
    each(load_each(lt, names("embeddings.LayerNorm.bias"), {H}), &TaskTensors::emb_ln_b);
    for (int li = 0; li < c.L && ok(); ++li) {
      each_layer(load_each(lt, names("attention.output.LayerNorm.weight", li), {H}), li, &TaskNorms::mid_w);
      each_layer(load_each(lt, names("attention.output.LayerNorm.bias", li), {H}), li, &TaskNorms::mid_b);
      each_layer(load_each(lt, names("output.LayerNorm.weight", li), {H}), li, &TaskNorms::out_w);
      each_layer(load_each(lt, names("output.LayerNorm.bias", li), {H}), li, &TaskNorms::out_b);
    }
  }
  m->layers.resize(c.L);
  for (int li = 0; li < c.L && ok(); ++li) {
    std::vector<std::array<Projection, 4>> pr;
    for (int t = 0; t < T; ++t) pr.push_back(layer_projections(c, ck[t].P, li, task[t].layers[li].attn_w != nullptr));
    for (int p = 0; p < 4 && ok(); ++p) {
      std::vector<float> stack, bstack, w, b;
      for (int t = 0; t < T && ok(); ++t) {
        if (!device_weight(lt[t], pr[t][p], w, pr[t][p].bias ? &b : nullptr)) break;
        stack.insert(stack.end(), w.begin(), w.end());
        bstack.insert(bstack.end(), b.begin(), b.end());
      }
      if (ok()) store_projection(lt[0], pr[0][p], p, stack, bstack, m->layers[li]);
    }
  }
  if (!ok()) { model_free(m); return nullptr; }
  return m;
}

// The load's last step, after the caller's heads: the model with its stream, or null and *err (the model freed)
Model* finish_load(Model* m, const std::vector<Checkpoint>& ck, const std::vector<Loader>& lt, std::string* err) {
  if (!tasks_ok(ck, lt, err)) { model_free(m); return nullptr; }
  if (cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking) != cudaSuccess) {
    *err = "stream create failed";
    model_free(m);
    return nullptr;
  }
  cudaDeviceSynchronize();
  return m;
}
}  // namespace

// ------------------------------------------------------------------------------------------------
// model load: one checkpoint is a grouped model of one task (engine.h: Grouped).  Both entries read every directory on
// the host (read_checkpoint), then take the device (use_device), upload (upload_tasks) and add their heads.
// ------------------------------------------------------------------------------------------------
Model* model_load(const std::string& dir, int device, std::string* err) {
  std::vector<Checkpoint> ck(1);
  if (!read_checkpoint(dir, ck[0], err) || !use_device(device, err)) return nullptr;
  std::vector<Loader> lt;
  Model* m = upload_tasks(ck, device, lt, err);
  if (!m) return nullptr;
  Head hd;   // none when the checkpoint has no classifier.weight or one that does not fit hidden_size
  if (load_head(lt[0], ck[0].cfgj, m->cfg.arch, m->cfg.H, ck[0].P, -1, hd)) {
    hd.final_norm_w = m->task[0].final_norm_w;
    m->heads.push_back(hd);
  }
  return finish_load(m, ck, lt, err);
}

Model* model_load_grouped(const std::vector<std::string>& dirs, const std::vector<int>& token_level, int device,
                          std::string* err) {
  const int T = static_cast<int>(dirs.size());
  if (T < 1 || T > kMaxRowGroups) { *err = "a grouped model takes 1 to " + std::to_string(kMaxRowGroups) + " task checkpoints"; return nullptr; }
  if (token_level.size() != dirs.size()) { *err = "one token_level per task checkpoint"; return nullptr; }
  // every refusal of the directories first, on the host
  std::vector<Checkpoint> ck(T);
  for (int t = 0; t < T; ++t) {
    const std::string& d = dirs[t];
    if (!read_checkpoint(d, ck[t], err)) return nullptr;
    if (ck[t].cfg.attn_w != ck[t].cfg.H) { *err = d + ": grouped serving is not available for padded-head (MiniLM) encoders"; return nullptr; }
    const auto f0 = shape_fields(ck[0].cfg), ft = shape_fields(ck[t].cfg);
    for (size_t i = 0; i < f0.size(); ++i)
      if (f0[i].second != ft[i].second) {
        *err = std::string("the checkpoints do not share one encoder shape: ") + f0[i].first + " is " + ft[i].second + " in " + d +
               " and " + f0[i].second + " in " + dirs[0];
        return nullptr;
      }
    if (!ck[t].st.find("classifier.weight")) { *err = "no classifier.weight in " + d; return nullptr; }
    // BERT's Wi has N = intermediate_size, and gemm_f16 picks a task's matrix per row block only when N is whole
    // 128-column tiles (ModernBERT's Wi, N = 2 I with I % 64 == 0, always is)
    if (T > 1 && ck[t].cfg.arch == ARCH_BERT && ck[t].cfg.I % 128 != 0) {
      *err = d + ": intermediate_size " + std::to_string(ck[t].cfg.I) + " must be a multiple of 128 to serve several BERT tasks in one pass";
      return nullptr;
    }
  }
  if (!use_device(device, err)) return nullptr;
  std::vector<Loader> lt;
  Model* m = upload_tasks(ck, device, lt, err);
  if (!m) return nullptr;
  for (int t = 0; t < T; ++t) {
    Head hd;
    if (!load_head(lt[t], ck[t].cfgj, m->cfg.arch, m->cfg.H, ck[t].P, token_level[t], hd)) {
      if (lt[t].ok) lt[t].fail("classifier.weight does not fit hidden_size");
      break;
    }
    hd.final_norm_w = m->task[t].final_norm_w;
    m->heads.push_back(hd);
    m->group.head_of_task.push_back(t);
  }
  m->group.tasks = T;
  return finish_load(m, ck, lt, err);
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
  std::string bp;
  tensor_prefix(st, m->cfg.arch, bp);   // a head-only checkpoint has no embeddings: its pooler names the prefix
  if (!load_head(ld, cfgj, m->cfg.arch, m->cfg.H, bp, force_token_level, hd) || !ld.ok) {
    *err = ld.ok ? "no classifier.weight in " + dir : ld.err;
    return -1;
  }
  hd.final_norm_w = m->task[0].final_norm_w;
  m->heads.push_back(hd);
  return static_cast<int>(m->heads.size()) - 1;
}

Model* model_load_lora_shared(const std::vector<std::string>& dirs, const std::vector<int>& token_level, int device,
                              std::string* err) {
  const int T = static_cast<int>(dirs.size());
  if (T < 1 || token_level.size() != dirs.size()) { *err = "bad arguments"; return nullptr; }
  std::vector<std::unique_ptr<SafeTensors>> sts;
  for (const std::string& d : dirs) {
    sts.emplace_back(new SafeTensors());
    if (!sts.back()->open(d + "/model.safetensors", err)) return nullptr;
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
  // every task's adapters merged into its own copy of the projections (lora_fold, double precision, before the fp16
  // rounding), the base's other tensors once
  return model_load_grouped(dirs, token_level, device, err);
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

int precise_prepare(Model& m, std::string* err) {
  if (!m.precise.layers.empty()) return 0;
  if (cudaSetDevice(m.device) != cudaSuccess) { *err = "cudaSetDevice failed"; return -1; }
  SafeTensors st;
  if (!st.open(m.dir + "/model.safetensors", err)) return -1;
  Loader ld{&m, &st};
  ld.lora_alpha = lora_alpha_of(m.dir);
  std::string P;
  tensor_prefix(st, m.cfg.arch, P);
  const size_t loaded = m.weight_bytes;
  std::vector<PreciseLayer> layers(m.cfg.L);
  std::vector<float> w, b, split;
  for (int li = 0; li < m.cfg.L && ld.ok; ++li) {
    const auto pr = layer_projections(m.cfg, P, li, m.task[0].layers[li].attn_w != nullptr);
    PreciseLayer& pl = layers[li];
    __half** slot[] = {&pl.wqkv, &pl.wo, &pl.wi, &pl.wo2};
    float** bias[] = {&pl.bqkv, &pl.bo, &pl.bi, &pl.bo2};
    for (int p = 0; p < 4 && ld.ok; ++p) {
      if (!read_projection(ld, pr[p], w, pr[p].bias ? &b : nullptr)) break;
      // W [N, K] -> [W_hi | W_hi | W_lo] [N, 3K], hi = fp16(w), lo = fp16(w - hi): both are fp16 values, which up_f16
      // stores unchanged
      const int n = pr[p].N, k = pr[p].K;
      split.resize(static_cast<size_t>(n) * 3 * k);
      for (int r = 0; r < n; ++r)
        for (int c = 0; c < k; ++c) {
          const float v = w[static_cast<size_t>(r) * k + c];
          const float hi = __half2float(__float2half_rn(v));
          float* o = split.data() + static_cast<size_t>(r) * 3 * k + c;
          o[0] = o[k] = hi;
          o[2 * k] = __half2float(__float2half_rn(v - hi));
        }
      *slot[p] = ld.up_f16(split);
      if (pr[p].bias) *bias[p] = ld.up_f32(b);
    }
  }
  m.weight_bytes = loaded;   // derived from the loaded weights, not loaded: sr_model_device_bytes leaves them out
  if (!ld.ok) { *err = ld.err; return -1; }
  m.precise.layers.swap(layers);
  return 0;
}

void model_free(Model* m) {
  if (!m) return;
  cudaSetDevice(m->device);
  if (m->stream) { cudaStreamSynchronize(m->stream); cudaStreamDestroy(m->stream); }
  for (void* p : m->allocs) cudaFree(p);
  Workspace& w = m->ws;
  void* dev[] = {w.x, w.h, w.lo, w.qkv, w.ctx, w.mid, w.ids, w.pos, w.cu, w.pooled, w.pool_part, w.pool_arrived, w.logits,
                 w.probs, w.cls, w.conf, w.emb, w.row_stats, w.kv_lens, w.split, w.qkv32, w.ctx32, w.mid32, w.act32};
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
  if (m.precise.on) rc |= precise_reserve(m);
  if (rc) fprintf(stderr, "[srb200] workspace allocation failed (tokens=%d seqs=%d)\n", tokens, seqs);
  return rc;
}

int precise_reserve(Model& m) {
  Workspace& w = m.ws;
  if (w.cap_tokens <= w.cap_precise) return 0;
  cudaStreamSynchronize(m.stream);
  ++w.generation;
  const size_t T = static_cast<size_t>(w.cap_tokens), H = m.cfg.H, I = m.cfg.I;
  const bool bert = m.cfg.arch == ARCH_BERT;
  int rc = regrow(w.split, T * 3 * std::max(H, I));
  rc |= regrow(w.qkv32, T * 3 * H);
  rc |= regrow(w.ctx32, T * H);
  rc |= regrow(w.mid32, T * (bert ? 1 : 2) * I);
  if (!bert) rc |= regrow(w.act32, T * I);
  w.cap_precise = rc ? 0 : w.cap_tokens;
  if (rc) w.cap_tokens = 0;
  return rc;
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
int encoder_forward(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int num_layers) {
  const EncoderConfig& c = m.cfg;
  Workspace& w = m.ws;
  cudaStream_t s = m.stream;
  const int H = c.H, I = c.I;
  if (T > w.cap_tokens || B > w.cap_seqs) return -1;
  if (max_len > c.max_pos) {   // BERT's position embeddings and ModernBERT's rotary tables have max_pos rows
    fprintf(stderr, "[srb200] sequence length %d exceeds max_position_embeddings %d\n", max_len, c.max_pos);
    return -1;
  }
  const int L = (num_layers <= 0 || num_layers > c.L) ? c.L : num_layers;
  if (compute_positions(s, d_cu, B, w.pos)) return -1;
  if (m.precise.on) return encoder_forward_precise(m, d_ids, d_cu, B, T, max_len, L);
  GemmDesc g;
  g.M = T;
  g.a_rows = w.cap_tokens;
  // grouped pass (engine.h: Grouped): every projection GEMM picks the task's matrix and bias per row block (gemm.h:
  // w_groups), every row kernel the task's embeddings and norms (kernels.h: RowGroups)
  const Grouped& gp = m.group;
  const bool grouped = gp.tasks > 0 && gp.rows_per_task > 0;
  if (grouped && (T != gp.tasks * gp.rows_per_task || gp.rows_per_task % 256 != 0)) return -1;
  const int group_rows = grouped ? gp.rows_per_task : 0;
  auto run_proj = [&](GemmDesc& gd) {
    if (grouped) { gd.w_groups = gp.tasks; gd.w_group_rows = gp.rows_per_task; gd.bias_per_group = true; }
    return gemm_f16(s, gd);
  };
  // a task tensor per row group; outside a grouped pass task 0's
  const int row_groups = grouped ? gp.tasks : 1;
  auto per_task = [&](float* TaskTensors::*f) {
    RowGroups r;
    for (int t = 0; t < row_groups; ++t) r.p[t] = m.task[t].*f;
    return r;
  };
  auto per_task_norm = [&](int li, float* TaskNorms::*f) {
    RowGroups r;
    for (int t = 0; t < row_groups; ++t) r.p[t] = m.task[t].layers[li].*f;
    return r;
  };
  if (c.arch == ARCH_MODERNBERT) {
    // Residual stream as an fp16 pair (gemm.h: EPI_RESID_HL): w.h / w.lo hold x - pivot, the residual GEMMs update the
    // pair in place, and the fp32 form is rebuilt once after the last layer.  LayerNorm fold (gemm.h): each residual
    // GEMM also leaves the per-row (sum, sum of squares) of x - pivot in w.row_stats; the projection that consumes
    // LN(x) multiplies the raw rows w.h with W diag(gamma) and corrects per row in its epilogue -- no LayerNorm pass.
    // Layer 0's attn_norm (when the checkpoint has one) is the exception: it runs on the fp32 embedding output.
    const bool ln0 = m.task[0].layers[0].attn_w != nullptr;
    { ProfScope ps(m, PC_EMBED);
      if (embed_ln_modernbert(s, d_ids, T, H, c.vocab, per_task(&TaskTensors::emb_word),
                              per_task(&TaskTensors::emb_ln_w), group_rows, c.ln_eps, ln0 ? w.x : nullptr, w.h, w.lo))
        return -1; }
    // one statistics record [H/128][T][2] partials + [T] pivots, padded so that the second record keeps the float2
    // alignment of the partials; the residual GEMMs ping-pong between the two
    const size_t rec = (static_cast<size_t>(T) * (2 * static_cast<size_t>(H / 128) + 1) + 3) & ~static_cast<size_t>(3);
    const size_t piv_off = static_cast<size_t>(T) * 2 * (H / 128);
    int n_rec = 0;                 // records written so far in this forward
    const float* cur_stats = nullptr;
    auto emit_for = [&](GemmDesc& gd) {   // this residual GEMM updates the pair and writes the next record
      float* dst = w.row_stats + (n_rec & 1) * rec;
      gd.epi = EPI_RESID_HL; gd.out = w.h; gd.ldo = H; gd.lo16 = w.lo;
      gd.row_stats = dst;                                   // every partial overwritten
      gd.pivot_out = dst + piv_off;
      if (n_rec > 0) {                                      // pivot = the row mean after the previous residual GEMM
        gd.pivot_in_stats = cur_stats;
        gd.pivot_in = cur_stats + piv_off;
      }
      cur_stats = dst;
      ++n_rec;
    };
    for (int li = 0; li < L; ++li) {
      const LayerWeights& lw = m.layers[li];
      const bool local = (li % c.global_every) != 0;
      const bool folded = lw.wqkv_f != nullptr;   // layer_projections: li > 0 with attn_norm
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = 3 * H; g.K = H; g.A = w.h; g.W = lw.wqkv; g.out = w.qkv; g.ldo = 3 * H;
      if (folded) {
        g.W = lw.wqkv_f; g.fold_stats = cur_stats; g.fold_eps = c.ln_eps; g.fold_h = H;
      } else if (li > 0 || ln0) {
        // A = fp16(attn_norm(x)) or, without attn_norm, fp16(x) in w.ctx: free here (the previous Wo has consumed it,
        // this layer's attention has not written it yet)
        ProfScope ps(m, PC_NORM);
        if (li == 0) {
          if (layernorm_rows(s, w.x, T, H, per_task_norm(0, &TaskNorms::attn_w), RowGroups::one(nullptr),
                             group_rows, c.ln_eps, nullptr, w.ctx))
            return -1;
        } else {
          if (hl_to_f32(s, w.h, w.lo, cur_stats + piv_off, T, H, w.x)) return -1;
          if (cast_rows_f16(s, w.x, static_cast<size_t>(T) * H, w.ctx)) return -1;
        }
        g.A = w.ctx;
      }
      g.epi = EPI_ROPE; g.pos = w.pos; g.rope_cols = 2 * H;
      g.rope_cos = local ? m.rope_cos_l : m.rope_cos_g;
      g.rope_sin = local ? m.rope_sin_l : m.rope_sin_g;
      { ProfScope ps(m, PC_GEMM_QKV); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_ATTN);   // sliding-window layers visit only the key blocks inside the window
        if (attention_wgmma_fwd(s, w.qkv, w.ctx, d_cu, B, max_len, c.heads, 64, local ? c.local_attention / 2 : 0)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = H; g.A = w.ctx; g.W = lw.wo;
      emit_for(g);
      { ProfScope ps(m, PC_GEMM_WO); if (run_proj(g)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = 2 * I; g.K = H; g.A = w.h; g.W = lw.wi_f; g.out = w.mid; g.ldo = I;
      g.fold_stats = cur_stats; g.fold_eps = c.ln_eps; g.fold_h = H;
      g.epi = EPI_GEGLU;
      { ProfScope ps(m, PC_GEMM_WI); if (run_proj(g)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = I; g.A = w.mid; g.W = lw.wo2;
      emit_for(g);
      { ProfScope ps(m, PC_GEMM_WO2); if (run_proj(g)) return -1; }
    }
    {   // x = pivot + hi + lo for the heads (final_norm, pooling, token heads read the fp32 stream)
      ProfScope ps(m, PC_NORM);
      if (hl_to_f32(s, w.h, w.lo, cur_stats + piv_off, T, H, w.x)) return -1;
    }
  } else {
    ProfScope ps_embed(m, PC_EMBED);
    if (embed_ln_bert(s, d_ids, w.pos, T, H, c.vocab, c.max_pos, per_task(&TaskTensors::emb_word),
                      per_task(&TaskTensors::emb_pos), per_task(&TaskTensors::emb_type0),
                      per_task(&TaskTensors::emb_ln_w), per_task(&TaskTensors::emb_ln_b), group_rows,
                      c.ln_eps, w.x, w.h))
      return -1;
    for (int li = 0; li < L; ++li) {
      const LayerWeights& lw = m.layers[li];
      g = GemmDesc();
      const int Hq = c.attn_w;   // == H unless the heads were padded (MiniLM)
      g.M = T; g.a_rows = w.cap_tokens; g.N = 3 * Hq; g.K = H; g.A = w.h; g.W = lw.wqkv; g.out = w.qkv; g.ldo = 3 * Hq;
      g.epi = EPI_F16; g.bias = lw.bqkv;
      { ProfScope ps(m, PC_GEMM_QKV); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_ATTN); if (attention_wgmma_fwd(s, w.qkv, w.ctx, d_cu, B, max_len, c.heads, 64, 0, m.cur_kv_lens)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = Hq; g.A = w.ctx; g.W = lw.wo; g.out = w.x; g.ldo = H;
      g.epi = EPI_RESID; g.resid = w.x; g.ldr = H; g.bias = lw.bo;
      { ProfScope ps(m, PC_GEMM_WO); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_NORM);
        if (layernorm_rows(s, w.x, T, H, per_task_norm(li, &TaskNorms::mid_w),
                           per_task_norm(li, &TaskNorms::mid_b), group_rows, c.ln_eps, w.x, w.h))
          return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = I; g.K = H; g.A = w.h; g.W = lw.wi; g.out = w.mid; g.ldo = I;
      g.epi = EPI_GELU; g.bias = lw.bi;
      { ProfScope ps(m, PC_GEMM_WI); if (run_proj(g)) return -1; }
      g = GemmDesc();
      g.M = T; g.a_rows = w.cap_tokens; g.N = H; g.K = I; g.A = w.mid; g.W = lw.wo2; g.out = w.x; g.ldo = H;
      g.epi = EPI_RESID; g.resid = w.x; g.ldr = H; g.bias = lw.bo2;
      { ProfScope ps(m, PC_GEMM_WO2); if (run_proj(g)) return -1; }
      { ProfScope ps(m, PC_NORM);
        if (layernorm_rows(s, w.x, T, H, per_task_norm(li, &TaskNorms::out_w),
                           per_task_norm(li, &TaskNorms::out_b), group_rows, c.ln_eps, w.x, w.h))
          return -1; }
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
    if (pool_rows(m.stream, w.x, d_cu, B, c.H, (hf && c.cls_pooling == 0) ? POOL_CLS : POOL_MEAN, hd.final_norm_w, nullptr,
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
      if (layernorm_rows(m.stream, x, T, c.H, hd.final_norm_w, nullptr, c.ln_eps, nullptr, w.h + off)) return -1;
      GemmDesc g;
      g.M = T; g.a_rows = w.cap_tokens - row0; g.N = c.H; g.K = c.H; g.A = w.h + off; g.W = hd.dense_w16; g.out = w.ctx + off; g.ldo = c.H;
      g.epi = EPI_F16;
      if (gemm_f16(m.stream, g)) return -1;
      const bool hf = m.head_flavor == 1;
      return token_head(m.stream, nullptr, w.ctx + off, T, c.H, hd.norm_w, nullptr, 0.f, hd.cls_w, hd.cls_b, hd.num_classes,
                        hf ? 1 : 0, w.logits, w.probs, w.cls, w.conf, hf ? 1 : 0, hf ? c.ln_eps : 1e-12f);
    }
    return token_head(m.stream, x, nullptr, T, c.H, nullptr, hd.final_norm_w, c.ln_eps, hd.cls_w, hd.cls_b,
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
    if (pool_rows(m.stream, w.x, d_cu, B, c.H, POOL_MEAN, m.task[0].final_norm_w, nullptr, c.ln_eps, w.pooled, w.pool_part, w.pool_arrived)) return -1;
  } else {
    if (pool_rows(m.stream, w.x, d_cu, B, c.H, POOL_MEAN, nullptr, nullptr, 0.f, w.pooled, w.pool_part, w.pool_arrived, m.cur_kv_lens)) return -1;
  }
  return l2_normalize_rows(m.stream, w.pooled, B, c.H, dim, norm_eps, w.emb);
}

}  // namespace srb
