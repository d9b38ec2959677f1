// Host-side core shared by the two drop-in ABIs (abi.cu: candle-binding symbol table; onnx_abi.cu: onnx-binding
// symbol table): model slots, tokenise -> packed-varlen batch -> engine, request coalescing, BIO decode, result
// packing.  Everything lives in an anonymous namespace: each library gets its own copy and exports none of it.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <functional>
#include <future>
#include <climits>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/sr_b200.h"
#include "json.hpp"
#include "tokenizer.h"

using srb::Json;

namespace {

// ------------------------------------------------------------------------------------------------
// slots
// ------------------------------------------------------------------------------------------------
struct SeqRequest;
// One copy of a slot's model on one GPU.  `Incoming request batches shard naturally across the 8 GPUs of one box`
// (BASELINE north star) while the Go router stays ONE process calling this library from many goroutines
// (classifier_signal_dispatch.go:114-129): every slot therefore loads its weights on each device of the device set
// (below) and every call is handed to the least-loaded replica.  Each replica owns its coalescing queue.
struct Replica {
  sr_model* model = nullptr;
  int device = 0;
  std::atomic<int> inflight{0};   // requests assigned and not yet answered (text calls count 1, batch pieces their size)
  std::mutex bmu;
  std::condition_variable bcv;
  std::deque<SeqRequest*> bq;
  bool brunning = false;
};

struct Slot {
  std::mutex mu;
  std::atomic<sr_model*> model{nullptr};           // replica 0 (model facts: classes, shapes); set last by slot_init
  // filled once by slot_init, never resized afterwards.  Heap-held and deliberately not destroyed with the slot: the
  // global slots outlive every call (static destruction must not tear replicas down under a late caller, and at exit
  // the CUDA runtime may already be gone); release() is the explicit way out.
  std::vector<std::unique_ptr<Replica>>& reps = *new std::vector<std::unique_ptr<Replica>>();
  std::atomic<unsigned> rr{0};                     // tie-break cursor of pick()
  srb::Tokenizer* tok = nullptr;
  int head = 0;
  bool token_level = false;
  bool modernbert = true;
  int pooler_mode = 0;   // BERT: 0 = traditional/bert.rs:107 (x @ P), 1 = lora/bert_lora.rs:534 (x @ P^T)
  int max_len = 512;     // MAX_CLASSIFICATION_SEQ_LEN (traditional/modernbert.rs:20)
  int max_pos = 512;
  std::string dir;
  std::map<int, std::string> id2label;
  bool ready() const { return model.load() != nullptr; }
  // Global slots live for the process (no destructor work: at exit the CUDA runtime may already be gone); named ONNX
  // slots are replaced at run time and give their HBM back through release().
  void release() {
    model = nullptr;
    for (auto& r : reps)
      if (r && r->model) { sr_model_free(r->model); r->model = nullptr; }
    reps.clear();
    delete tok;
    tok = nullptr;
  }
  void destroy() { release(); delete &reps; }   // for slots that are themselves heap objects (named ONNX slots)
  // least-loaded replica; ties go round so that sequential callers still spread their first requests
  Replica& pick(int weight) {
    const size_t n = reps.size();
    size_t best = 0;
    if (n > 1) {
      const size_t start = rr.fetch_add(1, std::memory_order_relaxed) % n;
      int best_load = INT32_MAX;
      for (size_t i = 0; i < n; ++i) {
        const size_t k = (start + i) % n;
        const int load = reps[k]->inflight.load(std::memory_order_relaxed);
        if (load < best_load) { best_load = load; best = k; }
      }
    }
    reps[best]->inflight.fetch_add(weight, std::memory_order_relaxed);
    return *reps[best];
  }
};
std::atomic<long long> g_dev_requests[64];   // requests handed to each CUDA device by the text ABI (sr_abi_device_requests)
struct Assigned {   // RAII: a replica picked for `weight` requests until this goes out of scope
  Replica& r;
  int weight;
  Assigned(Slot& s, int w) : r(s.pick(w)), weight(w) {
    if (r.device >= 0 && r.device < 64) g_dev_requests[r.device].fetch_add(w, std::memory_order_relaxed);
  }
  ~Assigned() { r.inflight.fetch_sub(weight, std::memory_order_relaxed); }
  Assigned(const Assigned&) = delete;
  Assigned& operator=(const Assigned&) = delete;
};

// One-text-per-call ABI vs batch kernels (SURVEY section 7 "hard parts"): concurrent callers of one slot are
// coalesced without timers.  The first caller to find its replica idle becomes the leader and runs ONE packed
// varlen batch over everything queued there at that moment (itself included); requests arriving meanwhile queue up and
// form the next batch.  Idle latency is unchanged (batch of one), under load batches grow by themselves.
struct SeqRequest {
  const std::vector<int32_t>* ids = nullptr;
  int cls = -1;
  float conf = 0.f;
  std::vector<float> probs;
  bool done = false;
};
std::atomic<long long> g_batches{0}, g_batched_requests{0};
constexpr int kMaxBatchRequests = 256;
constexpr int kMaxBatchTokens = 131072;


// Device set of the text ABI.  SR_B200_DEVICES = "all" | "0,2,5": replicate every slot on these GPUs.  Unset: the single
// device SR_B200_DEVICE names if that is set (one process per GPU under torchrun sets it per rank), else every visible
// GPU -- an unchanged single-process router then uses the whole box (CUDA_VISIBLE_DEVICES narrows it as usual).
std::vector<int> env_devices() {
  const int n = sr_device_count();
  std::vector<int> out;
  const char* list = getenv("SR_B200_DEVICES");
  const char* one = getenv("SR_B200_DEVICE");
  if (list && *list && strcmp(list, "all") != 0) {
    for (const char* p = list; *p;) {
      char* e = nullptr;
      const long v = strtol(p, &e, 10);
      if (e == p) break;
      if (v >= 0 && v < n && std::find(out.begin(), out.end(), static_cast<int>(v)) == out.end()) out.push_back(static_cast<int>(v));
      p = (*e == ',') ? e + 1 : e;
      if (*e && *e != ',') break;
    }
  } else if (!(list && *list) && one && *one) {
    out.push_back(atoi(one));
  } else {
    for (int i = 0; i < n; ++i) out.push_back(i);
  }
  if (out.empty()) out.push_back(one ? atoi(one) : 0);   // no usable entry: let sr_model_load report the device error
  return out;
}
void note_use_cpu(bool use_cpu) {
  static std::once_flag once;
  if (use_cpu) std::call_once(once, [] {
    fprintf(stderr, "[srb200] use_cpu=true ignored: this library has no CPU path (runs on sm_90a only)\n");
  });
}
bool file_exists(const std::string& p) {
  FILE* f = fopen(p.c_str(), "rb");
  if (!f) return false;
  fclose(f);
  return true;
}
char* dup_cstr(const std::string& s) {
  char* p = static_cast<char*>(malloc(s.size() + 1));
  if (p) memcpy(p, s.c_str(), s.size() + 1);
  return p;
}
double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

void load_id2label(const std::string& config_path, std::map<int, std::string>& out) {
  Json cfg;
  if (!srb::parse_json_file(config_path, cfg)) return;
  if (const Json* m = cfg.get("id2label"))
    for (const auto& kv : m->obj)
      if (kv.second.is_str()) out[atoi(kv.first.c_str())] = kv.second.str;
}

// loads <dir>/{config.json, model.safetensors, tokenizer.json} on every device of the device set (in parallel);
// token_level: 1/0/-1 (auto from config), -2: encoder without a classifier is fine
// `loader` (optional): how one replica is loaded on a device (default: sr_model_load(dir)); `dir` always names the
// directory the tokenizer, labels and model facts come from
using ReplicaLoader = std::function<int(int device, sr_model** out)>;
bool slot_init(Slot& s, const char* dir, int token_level, bool reinit_returns, const ReplicaLoader& loader = nullptr) {
  if (!dir) return false;
  std::lock_guard<std::mutex> lk(s.mu);
  if (s.ready()) return reinit_returns;   // OnceLock semantics (SURVEY 8b "Error conventions")
  const std::vector<int> devs = env_devices();
  std::vector<sr_model*> models(devs.size(), nullptr);
  {
    std::vector<std::thread> th;
    auto load = [&](size_t i) {
      const int rc = loader ? loader(devs[i], &models[i]) : sr_model_load(dir, devs[i], &models[i]);
      if (rc != 0) models[i] = nullptr;
    };
    try {
      for (size_t i = 1; i < devs.size(); ++i) th.emplace_back(load, i);
    } catch (...) {}
    load(0);
    for (size_t i = th.size() + 1; i < devs.size(); ++i) load(i);   // threads that could not start: load here
    for (auto& t : th) t.join();
  }
  auto drop = [&] { for (sr_model* m : models) if (m) sr_model_free(m); };
  for (sr_model* m : models)
    if (!m) { drop(); return false; }
  std::string err;
  srb::Tokenizer* t = srb::Tokenizer::from_file(std::string(dir) + "/tokenizer.json", &err);
  if (!t) {
    fprintf(stderr, "[srb200] init: %s\n", err.c_str());
    drop();
    return false;
  }
  sr_model_info_t info;
  sr_model_info(models[0], &info);
  if (info.num_heads_loaded < 1 && token_level != -2) {
    fprintf(stderr, "[srb200] init: %s has no classifier.weight\n", dir);
    drop();
    delete t;
    return false;
  }
  s.reps.clear();
  for (size_t i = 0; i < devs.size(); ++i) {
    std::unique_ptr<Replica> r(new Replica());
    r->model = models[i];
    r->device = devs[i];
    s.reps.push_back(std::move(r));
  }
  s.tok = t;
  s.dir = dir;
  s.modernbert = info.arch == 0;
  s.max_pos = info.max_pos;
  s.token_level = token_level == 1;
  s.pooler_mode = file_exists(std::string(dir) + "/lora_config.json") ? 1 : 0;
  load_id2label(std::string(dir) + "/config.json", s.id2label);
  s.model = models[0];   // last: ready() turns true only when everything above is in place
  return true;
}

struct Tokens {
  std::vector<int32_t> ids;
  std::vector<std::pair<int, int>> offsets;
  std::vector<std::string> tokens;
};
Tokens tokenize(const Slot& s, const char* text, int max_len) {
  srb::Encoding e = s.tok->encode(text, true, max_len);
  return Tokens{std::move(e.ids), std::move(e.offsets), std::move(e.tokens)};
}

// Executes one coalesced batch on its replica (leader only).  Never throws: a failure marks the batch failed.
void run_seq_batch(Slot& s, Replica& rep, std::vector<SeqRequest*>& batch) noexcept {
  const int B = static_cast<int>(batch.size());
  bool ok = false;
  int C = 0;
  std::vector<float> probs, conf;
  std::vector<int32_t> cls;
  try {
    C = sr_head_num_classes(rep.model, s.head);
    std::vector<int32_t> ids, cu{0};
    for (SeqRequest* r : batch) {
      ids.insert(ids.end(), r->ids->begin(), r->ids->end());
      cu.push_back(static_cast<int32_t>(ids.size()));
    }
    probs.resize(static_cast<size_t>(B) * (C > 0 ? C : 1));
    conf.resize(B);
    cls.assign(B, -1);
    ok = C > 0 && sr_classify_ids(rep.model, s.head, ids.data(), cu.data(), B, s.pooler_mode, probs.data(), nullptr,
                                  cls.data(), conf.data()) == 0;
    if (ok)
      for (int i = 0; i < B; ++i)
        batch[i]->probs.assign(probs.begin() + static_cast<size_t>(i) * C, probs.begin() + static_cast<size_t>(i + 1) * C);
  } catch (...) {   // bad_alloc while packing: the callers get the documented failure value
    ok = false;
  }
  for (int i = 0; i < B; ++i) {
    SeqRequest* r = batch[i];
    if (ok) { r->cls = cls[i]; r->conf = conf[i]; }
    else r->cls = -1;
  }
  g_batches.fetch_add(1, std::memory_order_relaxed);
  g_batched_requests.fetch_add(B, std::memory_order_relaxed);
}

// sequence classification of one text; returns class (-1 on failure)
int run_seq(Slot& s, const char* text, float* conf, std::vector<float>* probs) {
  if (!text || !s.ready()) return -1;
  const Tokens t = tokenize(s, text, s.max_len);
  if (t.ids.empty()) return -1;
  SeqRequest req;
  req.ids = &t.ids;
  Assigned as(s, 1);
  Replica& rep = as.r;
  std::unique_lock<std::mutex> lk(rep.bmu);
  rep.bq.push_back(&req);
  while (!req.done) {
    if (!rep.brunning) {
      rep.brunning = true;   // become the leader
      while (!req.done) {
        std::vector<SeqRequest*> batch;
        int tokens = 0;
        // always at least one request per batch (a single request is never larger than the engine's limits: the
        // tokenizer truncates to max_len), then as many as fit
        while (!rep.bq.empty() && static_cast<int>(batch.size()) < kMaxBatchRequests &&
               (batch.empty() || tokens + static_cast<int>(rep.bq.front()->ids->size()) <= kMaxBatchTokens)) {
          tokens += static_cast<int>(rep.bq.front()->ids->size());
          batch.push_back(rep.bq.front());
          rep.bq.pop_front();
        }
        lk.unlock();
        run_seq_batch(s, rep, batch);
        lk.lock();
        for (SeqRequest* r : batch) r->done = true;
        rep.bcv.notify_all();
      }
      rep.brunning = false;   // hand over: a waiting caller (if any) becomes the next leader
      rep.bcv.notify_all();
    } else {
      rep.bcv.wait(lk);
    }
  }
  lk.unlock();
  if (req.cls < 0) return -1;
  if (conf) *conf = req.conf;
  if (probs) probs->swap(req.probs);
  return req.cls;
}

struct Entity {
  std::string type;
  int cls, start, end;
  float conf;
};
struct TokenPred {
  int pred;
  float conf;
  int start, end;
  std::string token;
};

bool run_tokens(Slot& s, const char* text, std::vector<TokenPred>& out) {
  if (!text || !s.ready()) return false;
  const Tokens t = tokenize(s, text, s.max_len);
  if (t.ids.empty()) return false;
  const int n = static_cast<int>(t.ids.size());
  std::vector<int32_t> pred(n);
  std::vector<float> conf(n);
  int32_t cu[2] = {0, n};
  Assigned as(s, 1);
  if (sr_classify_tokens_ids(as.r.model, s.head, t.ids.data(), cu, 1, nullptr, nullptr, pred.data(), conf.data()) != 0) return false;
  out.resize(n);
  for (int i = 0; i < n; ++i) out[i] = {pred[i], conf[i], t.offsets[i].first, t.offsets[i].second, t.tokens[i]};
  return true;
}

// Tokenises `n` texts.  The tokenizer is re-entrant (its word cache is locked), so a batch large enough to pay for
// the threads is split across workers -- the reference clones the Tokenizer and encodes serially per call
// (core/tokenization.rs:343-395), which caps its batch entries on the host side (SURVEY §8f-1).
std::vector<Tokens> tokenize_many(const Slot& s, const char* const* texts, int n, int max_len) {
  std::vector<Tokens> out(static_cast<size_t>(n > 0 ? n : 0));
  auto one = [&](int i) {
    try { if (texts[i]) out[i] = tokenize(s, texts[i], max_len); } catch (...) { out[i] = Tokens{}; }
  };
  const int hw = static_cast<int>(std::thread::hardware_concurrency());
  const int workers = n >= 16 ? std::min(std::min(hw > 0 ? hw : 1, 32), n / 4) : 1;
  if (workers <= 1) {
    for (int i = 0; i < n; ++i) one(i);
    return out;
  }
  std::atomic<int> next{0};
  auto work = [&] { for (int i; (i = next.fetch_add(1, std::memory_order_relaxed)) < n;) one(i); };
  std::vector<std::thread> th;
  try {
    for (int w = 1; w < workers; ++w) th.emplace_back(work);
  } catch (...) {}   // out of threads: the ones that started (and this one) still drain the queue
  work();
  for (auto& t : th) t.join();
  return out;
}

// Packs tokenised texts [done, done+b) into ids/cu under the engine's batch limits (and `limit` texts); returns b.
inline int pack_piece(const std::vector<Tokens>& toks, int done, std::vector<int32_t>& ids, std::vector<int32_t>& cu,
                      int limit = kMaxBatchRequests, int max_tokens = kMaxBatchTokens) {
  ids.clear();
  cu.assign(1, 0);
  const int n = static_cast<int>(toks.size());
  int b = 0;
  while (done + b < n && b < kMaxBatchRequests && b < limit) {
    const std::vector<int32_t>& t = toks[done + b].ids;
    if (b > 0 && ids.size() + t.size() > static_cast<size_t>(max_tokens)) break;
    ids.insert(ids.end(), t.begin(), t.end());
    cu.push_back(static_cast<int32_t>(ids.size()));
    ++b;
  }
  return b;
}

// Runs fn(model, first, b, ids, cu) over consecutive pieces [first, first + b) of `toks`.  With one replica the pieces
// run in order on the calling thread.  With several, the batch is cut into about one piece per replica (never below
// kMinPiece texts: a tiny piece would not pay for its launches) and worker threads hand each piece to the least-loaded
// replica, so ONE batch call of the unchanged Go API keeps every GPU of the box busy.  fn writes disjoint output ranges.
constexpr int kMinPiece = 16;
// `copies`: how many times the engine call replicates the rows of a piece (shared-LoRA passes run one copy per task), so
// that the replicated piece stays inside the engine's batch limits.
template <typename Fn>
bool for_pieces(Slot& s, const std::vector<Tokens>& toks, Fn&& fn, int copies = 1) {
  const int n = static_cast<int>(toks.size());
  const int R = static_cast<int>(s.reps.size());
  if (n <= 0 || R <= 0 || copies <= 0) return false;
  const int cap = std::max(1, kMaxBatchRequests / copies), max_tokens = kMaxBatchTokens / copies;
  const int limit = R > 1 ? std::min(cap, std::max(kMinPiece, (n + R - 1) / R)) : cap;
  std::mutex mu;
  int next = 0;
  bool ok = true;
  auto worker = [&] {
    std::vector<int32_t> ids, cu;
    for (;;) {
      int first, b;
      {
        std::lock_guard<std::mutex> lk(mu);
        if (!ok || next >= n) return;
        first = next;
        b = pack_piece(toks, first, ids, cu, limit, max_tokens);
        next += b;
      }
      bool good = false;
      try {
        Assigned as(s, b);
        good = fn(as.r.model, first, b, ids, cu);
      } catch (...) {}
      if (!good) { std::lock_guard<std::mutex> lk(mu); ok = false; return; }
    }
  };
  const int workers = std::min(R, (n + limit - 1) / limit);
  std::vector<std::thread> th;
  try {
    for (int w = 1; w < workers; ++w) th.emplace_back(worker);
  } catch (...) {}   // out of threads: the ones that started (and this one) still drain the pieces
  worker();
  for (auto& t : th) t.join();
  return ok;
}

// `n` texts through a sequence head as packed varlen batches: probs [n, C], cls/conf [n].  False on any failure.
bool classify_packed(Slot& s, const char* const* texts, int n, std::vector<float>& probs, int& C,
                     std::vector<int32_t>* cls_out = nullptr, std::vector<float>* conf_out = nullptr) {
  C = s.ready() ? sr_head_num_classes(s.model, s.head) : 0;
  if (C <= 0 || n <= 0) return false;
  probs.assign(static_cast<size_t>(n) * C, 0.f);
  std::vector<int32_t> cls(n, -1);
  std::vector<float> conf(n, 0.f);
  auto run = [&](const std::vector<Tokens>& toks, int base) {
    for (const Tokens& t : toks)
      if (t.ids.empty()) return false;
    return for_pieces(s, toks, [&](sr_model* m, int first, int b, std::vector<int32_t>& ids, std::vector<int32_t>& cu) {
      return sr_classify_ids(m, s.head, ids.data(), cu.data(), b, s.pooler_mode,
                             probs.data() + static_cast<size_t>(base + first) * C, nullptr, cls.data() + base + first,
                             conf.data() + base + first) == 0;
    });
  };
  // large batches: the first 64 texts go to the GPU while the rest are still being tokenised
  const int head_n = n >= 128 ? 64 : n;
  const std::vector<Tokens> first = tokenize_many(s, texts, head_n, s.max_len);
  std::future<std::vector<Tokens>> rest;
  if (head_n < n) {
    try {
      rest = std::async(std::launch::async, [&] { return tokenize_many(s, texts + head_n, n - head_n, s.max_len); });
    } catch (...) {}   // no thread to spare: tokenise the tail after the first piece instead
  }
  const bool ok_first = run(first, 0);
  if (head_n < n) {
    const std::vector<Tokens> tail = rest.valid() ? rest.get()   // always joined, also on failure
                                                  : tokenize_many(s, texts + head_n, n - head_n, s.max_len);
    if (!ok_first || !run(tail, head_n)) return false;
  } else if (!ok_first) {
    return false;
  }
  if (cls_out) cls_out->swap(cls);
  if (conf_out) conf_out->swap(conf);
  return true;
}

// `n` texts through a token head as packed varlen batches: out[i] = per-token predictions of text i.
bool tokens_packed(Slot& s, const char* const* texts, int n, std::vector<std::vector<TokenPred>>& out) {
  if (!s.ready() || n <= 0) return false;
  const std::vector<Tokens> toks = tokenize_many(s, texts, n, s.max_len);
  for (const Tokens& t : toks)
    if (t.ids.empty()) return false;
  out.assign(n, {});
  return for_pieces(s, toks, [&](sr_model* m, int first, int b, std::vector<int32_t>& ids, std::vector<int32_t>& cu) {
    std::vector<int32_t> pred(ids.size());
    std::vector<float> conf(ids.size());
    if (sr_classify_tokens_ids(m, s.head, ids.data(), cu.data(), b, nullptr, nullptr, pred.data(), conf.data()) != 0) return false;
    for (int i = 0; i < b; ++i) {
      const Tokens& t = toks[first + i];
      std::vector<TokenPred>& o = out[first + i];
      o.resize(t.ids.size());
      for (size_t k = 0; k < t.ids.size(); ++k)
        o[k] = {pred[cu[i] + k], conf[cu[i] + k], t.offsets[k].first, t.offsets[k].second, t.tokens[k]};
    }
    return true;
  });
}

// detect_hallucinations after the token classifier (ffi/classify.rs:1536-1660): tokens that start inside the answer,
// class 1 with confidence >= thr extend a span (span confidence = max token confidence), anything else closes it; only
// spans that slice the answer cleanly survive.
struct HallucSpan { int start, end; float conf; };
struct HallucSummary {
  std::vector<HallucSpan> spans;
  int n_hall = 0, n_answer = 0;
  float max_conf = 0.f;
};
HallucSummary hallucination_spans(const std::vector<TokenPred>& toks, int answer_start, int answer_len, float threshold) {
  const float thr = (threshold > 0.0f && threshold <= 1.0f) ? threshold : 0.5f;   // classify.rs:1553-1557
  HallucSummary r;
  bool open = false;
  HallucSpan cur{0, 0, 0.f};
  auto close = [&] {   // classify.rs:1580-1605
    if (open && cur.start >= 0 && cur.end > cur.start && cur.end <= answer_len) r.spans.push_back(cur);
    open = false;
  };
  for (const TokenPred& t : toks) {
    if (t.start < answer_start) continue;   // context / question / special tokens (offset 0)
    ++r.n_answer;
    if (t.pred == 1 && t.conf >= thr) {
      ++r.n_hall;
      if (t.conf > r.max_conf) r.max_conf = t.conf;
      if (!open) { cur = HallucSpan{t.start - answer_start, t.end - answer_start, t.conf}; open = true; }
      else cur.end = t.end - answer_start;
      if (t.conf > cur.conf) cur.conf = t.conf;
    } else {
      close();
    }
  }
  close();
  return r;
}

// embeddings of `n` texts as packed varlen batches -> [n, d]; d = dim clamped to the hidden size
// (truncate_dimension, pooling.rs:74-82), an unknown exit layer runs the full model
bool embed_packed(Slot& s, const char* const* texts, int n, int max_len, int layer, int dim, std::vector<float>& out, int& d) {
  if (!s.ready() || n <= 0) return false;
  sr_model_info_t info;
  sr_model_info(s.model, &info);
  d = (dim <= 0 || dim > info.hidden) ? info.hidden : dim;
  const int lay = (layer <= 0 || layer > info.layers) ? 0 : layer;
  const std::vector<Tokens> toks = tokenize_many(s, texts, n, max_len);
  for (const Tokens& t : toks)
    if (t.ids.empty()) return false;
  out.assign(static_cast<size_t>(n) * d, 0.f);
  const int dd = d;
  return for_pieces(s, toks, [&](sr_model* m, int first, int b, std::vector<int32_t>& ids, std::vector<int32_t>& cu) {
    return sr_embed_ids(m, ids.data(), cu.data(), b, lay, dd, out.data() + static_cast<size_t>(first) * dd) == 0;
  });
}

// BIO decode (traditional/modernbert.rs:1478-1567): B- opens, matching I- extends with a running pairwise mean,
// anything else closes; special tokens (offset (0,0)) are skipped.
std::vector<Entity> bio_decode(const std::vector<TokenPred>& toks, const std::map<int, std::string>& id2label) {
  std::vector<Entity> out;
  bool open = false;
  Entity cur{};
  auto class_of = [&](const std::string& type) {
    for (const auto& kv : id2label)
      if (kv.second.rfind("B-" + type, 0) == 0 || kv.second.rfind("I-" + type, 0) == 0) return kv.first;
    return 0;
  };
  for (const auto& t : toks) {
    if (t.start == 0 && t.end == 0) continue;
    auto it = id2label.find(t.pred);
    const std::string label = it == id2label.end() ? "O" : it->second;
    if (label.rfind("B-", 0) == 0) {
      if (open) out.push_back(cur);
      cur = Entity{label.substr(2), 0, t.start, t.end, t.conf};
      open = true;
    } else if (label.rfind("I-", 0) == 0) {
      if (open) {
        if (cur.type == label.substr(2)) { cur.end = t.end; cur.conf = (cur.conf + t.conf) / 2.0f; }
        else { out.push_back(cur); open = false; }
      }
    } else if (open) {
      out.push_back(cur);
      open = false;
    }
  }
  if (open) out.push_back(cur);
  for (auto& e : out) e.cls = class_of(e.type);
  return out;
}

template <typename EntT, typename ResT>
ResT pack_entities(const char* text, const std::vector<Entity>& ents, const std::vector<std::string>& types) {
  ResT r{nullptr, 0};
  if (ents.empty()) return r;
  r.entities = static_cast<EntT*>(malloc(sizeof(EntT) * ents.size()));
  if (!r.entities) return r;
  const int tl = static_cast<int>(strlen(text));
  for (size_t i = 0; i < ents.size(); ++i) {
    const Entity& e = ents[i];
    std::string span = (e.start >= 0 && e.end <= tl && e.start < e.end) ? std::string(text + e.start, text + e.end) : "";
    r.entities[i].entity_type = dup_cstr(types[i]);
    r.entities[i].start = e.start;
    r.entities[i].end = e.end;
    r.entities[i].text = dup_cstr(span);
    r.entities[i].confidence = e.conf;
  }
  r.num_entities = static_cast<int>(ents.size());
  return r;
}

// BertSimilarity::get_embedding keeps whatever padding the tokenizer.json carries (core/similarity.rs:189-205): with
// "strategy": {"Fixed": n} (the sentence-transformers MiniLM files) every text shorter than n is right-padded to n positions;
// the pads run through the encoder as queries, are masked as keys, and the pooling sums them (:220-222).  Reproduced on the
// device by sr_embed_ids_padded.  Left padding would shift the position ids: not reproduced (falls back to no padding).
bool embed_text_similarity(Slot& s, const char* text, int max_len, std::vector<float>& out) {
  if (!text || !s.ready()) return false;
  Tokens t = tokenize(s, text, max_len);
  if (t.ids.empty()) return false;
  sr_model_info_t info;
  sr_model_info(s.model, &info);
  const int real = static_cast<int>(t.ids.size());
  const int fixed = s.tok->pad_fixed();
  out.resize(info.hidden);
  Assigned as(s, 1);
  if (fixed > real && !s.tok->pad_left() && !s.modernbert && fixed <= info.max_pos) {
    t.ids.resize(fixed, s.tok->pad_id());
    int32_t cu[2] = {0, fixed};
    const int32_t rl[1] = {real};
    return sr_embed_ids_padded(as.r.model, t.ids.data(), cu, rl, 1, out.data()) == 0;
  }
  int32_t cu[2] = {0, real};
  return sr_embed_ids(as.r.model, t.ids.data(), cu, 1, 0, info.hidden, out.data()) == 0;
}

bool embed_text(Slot& s, const char* text, int max_len, int layer, int dim, std::vector<float>& out) {
  if (!text || !s.ready()) return false;
  const Tokens t = tokenize(s, text, max_len);
  if (t.ids.empty()) return false;
  sr_model_info_t info;
  sr_model_info(s.model, &info);
  const int d = (dim <= 0 || dim > info.hidden) ? info.hidden : dim;
  if (layer > info.layers) return false;
  out.resize(d);
  int32_t cu[2] = {0, static_cast<int32_t>(t.ids.size())};
  Assigned as(s, 1);
  return sr_embed_ids(as.r.model, t.ids.data(), cu, 1, layer, d, out.data()) == 0;
}
int word_count(const char* text) {  // `text.split_whitespace().count()` (ffi/embedding.rs:1186)
  int n = 0;
  bool in = false;
  for (const unsigned char* p = reinterpret_cast<const unsigned char*>(text); *p; ++p) {
    const bool ws = *p == ' ' || (*p >= 9 && *p <= 13);
    if (!ws && !in) ++n;
    in = !ws;
  }
  return n;
}
float* dup_floats(const std::vector<float>& v) {
  float* p = static_cast<float*>(malloc(sizeof(float) * (v.empty() ? 1 : v.size())));
  if (p && !v.empty()) memcpy(p, v.data(), sizeof(float) * v.size());
  return p;
}
float dot(const std::vector<float>& a, const std::vector<float>& b) {
  float s = 0.f;
  for (size_t i = 0; i < a.size() && i < b.size(); ++i) s += a[i] * b[i];
  return s;
}

}  // namespace
