// "Precise" encoder path (ModernBERT / mmBERT): fp32-equivalent arithmetic on the same tcgen05 GEMM, for the strict
// parity bound BASELINE's north star states ("logits and embeddings within 1e-3 fp32").
//
// The production path multiplies fp16 operands (2^-11 relative rounding of every activation and weight, fp16 q / k / v /
// P): measured |dlogit| 3e-3 .. 9e-3 on the x8-scaled synthetic heads, i.e. 3e-4 relative -- inside 1e-3 for the bounded
// outputs (probabilities, embeddings) but not for raw logits of that scale.  This path removes the operand rounding:
//
//   x = hi + lo        hi = fp16(x), lo = fp16(x - hi)      (|x - hi - lo| <= 2^-22 |x|; lo may be subnormal: still exact enough)
//   A W^T ~= A_hi W_hi^T + A_lo W_hi^T + A_hi W_lo^T         the dropped A_lo W_lo^T term is 2^-22 relative
//
// and runs it as ONE wgmma GEMM of three times the depth: A' = [A_hi | A_lo | A_hi] (K' = 3K), W' = [W_hi | W_hi | W_lo].
// fp16 x fp16 products are exact in fp32 and the accumulator is the fp32 TMEM one, so the result carries fp32-accumulation
// error only.  Everything between the GEMMs is plain fp32 (LayerNorm, RoPE, GeGLU with erff, softmax attention on the CUDA
// cores with expf): nothing is rounded to fp16 except through the split.  ~5x the time of the production path; selected
// per model with sr_model_set_precise() -- it exists for parity, not for serving.
//
// Replaces the same reference code as engine.cu's encoder_forward (candle_models/modernbert.rs:61-86,121-213,234-240,283-305).
#include <cuda_fp16.h>

#include <cmath>
#include <vector>

#include "common.cuh"
#include "engine.h"
#include "gemm.h"

namespace srb {
namespace {

// ---- fp32 rows -> [hi | lo | hi] fp16 rows (optionally through a no-bias LayerNorm first)
template <bool kNorm>
__global__ void __launch_bounds__(256)
split_rows_kernel(const float* __restrict__ x, int T, int H, const float* __restrict__ gamma, float eps, __half* __restrict__ out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= T) return;
  const float* row = x + static_cast<size_t>(warp) * H;
  float mean = 0.f, rstd = 1.f;
  if (kNorm) {
    float s = 0.f;
    for (int i = lane; i < H; i += 32) s += row[i];
    mean = warp_sum(s) / H;
    float v = 0.f;
    for (int i = lane; i < H; i += 32) { const float d = row[i] - mean; v += d * d; }
    rstd = rsqrtf(warp_sum(v) / H + eps);
  }
  __half* o = out + static_cast<size_t>(warp) * 3 * H;
  for (int i = lane; i < H; i += 32) {
    float v = row[i];
    if (kNorm) v = (v - mean) * rstd * gamma[i];
    const __half hi = __float2half_rn(v);
    const __half lo = __float2half_rn(v - __half2float(hi));
    o[i] = hi;
    o[H + i] = lo;
    o[2 * H + i] = hi;
  }
}

// ---- rotate-half RoPE on the q and k thirds of fp32 qkv rows (candle rope, modernbert.rs:82-83)
__global__ void rope_f32_kernel(float* __restrict__ qkv, const int* __restrict__ pos, int T, int heads, const float* __restrict__ cs,
                                const float* __restrict__ sn) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;   // (t, which in {q,k}, head, d < 32)
  const size_t n = static_cast<size_t>(T) * 2 * heads * 32;
  if (i >= n) return;
  const int d = i & 31;
  const int h = (i >> 5) % heads;
  const int which = (i / (32 * heads)) & 1;
  const int t = static_cast<int>(i / (static_cast<size_t>(64) * heads));
  const int H = heads * 64;
  float* p = qkv + static_cast<size_t>(t) * 3 * H + which * H + h * 64;
  const float c = cs[static_cast<size_t>(pos[t]) * 32 + d], s = sn[static_cast<size_t>(pos[t]) * 32 + d];
  const float a = p[d], b = p[d + 32];
  p[d] = a * c - b * s;
  p[d + 32] = b * c + a * s;
}

// ---- gelu_erf(a) * b over fp32 [T, 2I] (a = first I columns, b = last I; modernbert.rs:238)
__global__ void geglu_f32_kernel(const float* __restrict__ ab, int T, int I, float* __restrict__ out) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<size_t>(T) * I) return;
  const size_t t = i / I, c = i % I;
  const float a = ab[t * 2 * I + c], b = ab[t * 2 * I + I + c];
  out[i] = 0.5f * a * (1.0f + erff(a * 0.70710678118654752440f)) * b;
}

// ---- fp32 softmax attention on the CUDA cores: one thread per query row, K / V tiles of 32 keys through shared memory,
// online softmax per tile (expf).  window = 0: global; else |i - j| <= window.  Padding never exists (packed rows).
constexpr int kARows = 64, kAKeys = 32;
__global__ void __launch_bounds__(kARows)
attention_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, const int* __restrict__ cu, int heads, int window,
                     float scale) {
  __shared__ float ks[kAKeys][64], vs[kAKeys][64];
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kARows;
  const int seq0 = cu[b], len = cu[b + 1] - seq0;
  if (q0 >= len) return;
  const int H = heads * 64;
  const int qi = q0 + threadIdx.x;
  const bool live = qi < len;
  float q[64], o[64];
  const float* qp = qkv + static_cast<size_t>(seq0 + (live ? qi : q0)) * 3 * H + h * 64;
#pragma unroll
  for (int d = 0; d < 64; ++d) { q[d] = qp[d] * scale; o[d] = 0.f; }
  float m = -INFINITY, l = 0.f;
  int k_lo = 0, k_hi = len;
  if (window > 0) {
    k_lo = q0 - window > 0 ? q0 - window : 0;
    k_hi = q0 + kARows - 1 + window + 1 < len ? q0 + kARows + window : len;
  }
  for (int k0 = k_lo; k0 < k_hi; k0 += kAKeys) {
    __syncthreads();
    for (int e = threadIdx.x; e < kAKeys * 64; e += kARows) {
      const int j = e >> 6, d = e & 63;
      const bool ok = k0 + j < len;
      const float* base = qkv + static_cast<size_t>(seq0 + (ok ? k0 + j : 0)) * 3 * H + h * 64 + d;
      ks[j][d] = ok ? base[H] : 0.f;
      vs[j][d] = ok ? base[2 * H] : 0.f;
    }
    __syncthreads();
    float s[kAKeys];
    float tm = -INFINITY;
#pragma unroll
    for (int j = 0; j < kAKeys; ++j) {
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) acc = fmaf(q[d], ks[j][d], acc);
      const int kj = k0 + j;
      const bool vis = live && kj < len && (window == 0 || (kj - qi <= window && qi - kj <= window));
      s[j] = vis ? acc : -INFINITY;
      tm = fmaxf(tm, s[j]);
    }
    if (tm == -INFINITY) continue;          // (uniform control flow is not required: no barrier inside)
    const float mn = fmaxf(m, tm);
    const float alpha = (m == -INFINITY) ? 0.f : expf(m - mn);
    l *= alpha;
#pragma unroll
    for (int d = 0; d < 64; ++d) o[d] *= alpha;
#pragma unroll
    for (int j = 0; j < kAKeys; ++j) {
      const float p = (s[j] == -INFINITY) ? 0.f : expf(s[j] - mn);
      l += p;
#pragma unroll
      for (int d = 0; d < 64; ++d) o[d] = fmaf(p, vs[j][d], o[d]);
    }
    m = mn;
  }
  if (live) {
    float* op = out + static_cast<size_t>(seq0 + qi) * H + h * 64;
    const float inv = 1.0f / l;
#pragma unroll
    for (int d = 0; d < 64; ++d) op[d] = o[d] * inv;
  }
}

// W [N, K] fp32 -> [W_hi | W_hi | W_lo] fp16 [N, 3K]
__half* split_weight(Model& m, const std::vector<float>& w, int n, int k) {
  std::vector<__half> h(static_cast<size_t>(n) * 3 * k);
  for (int r = 0; r < n; ++r)
    for (int c = 0; c < k; ++c) {
      const float v = w[static_cast<size_t>(r) * k + c];
      const __half hi = __float2half_rn(v);
      const __half lo = __float2half_rn(v - __half2float(hi));
      h[static_cast<size_t>(r) * 3 * k + c] = hi;
      h[static_cast<size_t>(r) * 3 * k + k + c] = hi;
      h[static_cast<size_t>(r) * 3 * k + 2 * k + c] = lo;
    }
  __half* d = nullptr;
  if (cudaMalloc(reinterpret_cast<void**>(&d), h.size() * 2) != cudaSuccess) return nullptr;
  m.allocs.push_back(d);
  if (cudaMemcpy(d, h.data(), h.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
  return d;
}

template <typename T>
int grow(T*& p, size_t& cap, size_t n) {
  if (n <= cap) return 0;
  if (p) cudaFree(p);
  p = nullptr;
  cap = 0;
  if (cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T)) != cudaSuccess) return -1;
  cap = n;
  return 0;
}

}  // namespace

// engine.cu: fp32 host copy of one tensor of <dir>/model.safetensors (shape-checked)
bool load_host_tensor(const std::string& dir, const std::string& name, const std::vector<int64_t>& shape, std::vector<float>& out,
                      std::string* err);
std::string modernbert_prefix(const std::string& dir);

int precise_prepare(Model& m, std::string* err) {
  if (m.cfg.arch != ARCH_MODERNBERT) { *err = "the precise path covers ModernBERT / mmBERT encoders"; return -1; }
  if (!m.precise.layers.empty()) return 0;
  if (cudaSetDevice(m.device) != cudaSuccess) { *err = "cudaSetDevice failed"; return -1; }
  const int H = m.cfg.H, I = m.cfg.I;
  const std::string P = modernbert_prefix(m.dir);
  std::vector<PreciseLayer> layers(m.cfg.L);
  for (int li = 0; li < m.cfg.L; ++li) {
    const std::string Lp = P + "layers." + std::to_string(li) + ".";
    std::vector<float> w;
    PreciseLayer& pl = layers[li];
    if (!load_host_tensor(m.dir, Lp + "attn.Wqkv.weight", {3 * H, H}, w, err)) return -1;
    pl.wqkv = split_weight(m, w, 3 * H, H);
    if (!load_host_tensor(m.dir, Lp + "attn.Wo.weight", {H, H}, w, err)) return -1;
    pl.wo = split_weight(m, w, H, H);
    if (!load_host_tensor(m.dir, Lp + "mlp.Wi.weight", {2 * I, H}, w, err)) return -1;
    pl.wi = split_weight(m, w, 2 * I, H);
    if (!load_host_tensor(m.dir, Lp + "mlp.Wo.weight", {H, I}, w, err)) return -1;
    pl.wo2 = split_weight(m, w, H, I);
    if (!pl.wqkv || !pl.wo || !pl.wi || !pl.wo2) { *err = "allocation of the split weights failed"; return -1; }
  }
  m.precise.layers.swap(layers);
  return 0;
}

void precise_free(Model& m) {
  PreciseState& p = m.precise;
  if (p.split) cudaFree(p.split);
  if (p.qkv32) cudaFree(p.qkv32);
  if (p.ctx32) cudaFree(p.ctx32);
  if (p.mid32) cudaFree(p.mid32);
  if (p.act32) cudaFree(p.act32);
  p = PreciseState();
}

int encoder_forward_precise(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int num_layers) {
  const EncoderConfig& c = m.cfg;
  Workspace& w = m.ws;
  PreciseState& p = m.precise;
  cudaStream_t s = m.stream;
  const int H = c.H, I = c.I;
  if (p.layers.empty() || T > w.cap_tokens || B > w.cap_seqs) return -1;
  if (max_len > m.rope_len) {
    fprintf(stderr, "[srb200] sequence length %d exceeds max_position_embeddings %d\n", max_len, m.rope_len);
    return -1;
  }
  const size_t Tp = (static_cast<size_t>(T) + 127) / 128 * 128;   // TMA boxes of 128 rows stay inside the allocations
  const int wide = I > H ? I : H;
  cudaStreamSynchronize(s);   // the buffers below may be regrown: nothing queued may still use the old ones
  if (grow(p.split, p.split_cap, Tp * 3 * wide) || grow(p.qkv32, p.qkv_cap, Tp * 3 * H) || grow(p.ctx32, p.ctx_cap, Tp * H) ||
      grow(p.mid32, p.mid_cap, Tp * 2 * I) || grow(p.act32, p.act_cap, Tp * I))
    return -1;
  const int L = (num_layers <= 0 || num_layers > c.L) ? c.L : num_layers;
  if (compute_positions(s, d_cu, B, w.pos)) return -1;
  if (embed_ln_modernbert(s, d_ids, T, H, c.vocab, m.emb_word, m.emb_ln_w, c.ln_eps, w.x, w.h)) return -1;
  const int rows_grid = (T * 32 + 255) / 256;
  auto gemm = [&](const __half* a, const __half* wt, int n, int k, float* out, bool resid) {
    GemmDesc g;
    g.M = T; g.a_rows = static_cast<int>(Tp); g.N = n; g.K = 3 * k; g.A = a; g.W = wt; g.out = out; g.ldo = n;
    g.epi = EPI_RESID;
    g.resid = resid ? out : nullptr;
    g.ldr = n;
    return gemm_f16(s, g);
  };
  for (int li = 0; li < L; ++li) {
    const LayerWeights& lw = m.layers[li];
    const PreciseLayer& pl = p.layers[li];
    const bool local = (li % c.global_every) != 0;
    // attention input: LayerNorm (none on layer 0, modernbert.rs:266-271), split
    if (lw.attn_norm_w) split_rows_kernel<true><<<rows_grid, 256, 0, s>>>(w.x, T, H, lw.attn_norm_w, c.ln_eps, p.split);
    else split_rows_kernel<false><<<rows_grid, 256, 0, s>>>(w.x, T, H, nullptr, 0.f, p.split);
    if (gemm(p.split, pl.wqkv, 3 * H, H, p.qkv32, false)) return -1;
    {
      const size_t n = static_cast<size_t>(T) * 2 * c.heads * 32;
      rope_f32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(p.qkv32, w.pos, T, c.heads,
                                                                            local ? m.rope_cos_l : m.rope_cos_g,
                                                                            local ? m.rope_sin_l : m.rope_sin_g);
    }
    {
      const dim3 grid((max_len + kARows - 1) / kARows, c.heads, B);
      attention_f32_kernel<<<grid, kARows, 0, s>>>(p.qkv32, p.ctx32, d_cu, c.heads, local ? c.local_attention / 2 : 0, 0.125f);
    }
    split_rows_kernel<false><<<rows_grid, 256, 0, s>>>(p.ctx32, T, H, nullptr, 0.f, p.split);
    if (gemm(p.split, pl.wo, H, H, w.x, true)) return -1;
    split_rows_kernel<true><<<rows_grid, 256, 0, s>>>(w.x, T, H, lw.mid_norm_w, c.ln_eps, p.split);
    if (gemm(p.split, pl.wi, 2 * I, H, p.mid32, false)) return -1;
    {
      const size_t n = static_cast<size_t>(T) * I;
      geglu_f32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(p.mid32, T, I, p.act32);
    }
    split_rows_kernel<false><<<rows_grid, 256, 0, s>>>(p.act32, T, I, nullptr, 0.f, p.split);
    if (gemm(p.split, pl.wo2, H, I, w.x, true)) return -1;
    note_launch(7);
  }
  SRB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace srb
