// "Precise" encoder path (ModernBERT / mmBERT, BERT / MiniLM): fp32-equivalent arithmetic on the same wgmma GEMM, for the strict
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
// fp16 x fp16 products are exact in fp32 and the accumulator is fp32 in registers, so the result carries fp32-accumulation
// error only.  Everything between the GEMMs is plain fp32 (LayerNorm, RoPE, GeGLU / GELU with erff, softmax attention on the
// CUDA cores with expf, heads of 64 or MiniLM's 32): nothing is rounded to fp16 except through the split.  ~5x the time of the production path; selected
// per model with sr_model_set_precise() -- it exists for parity, not for serving.
//
// Replaces the same reference code as engine.cu's encoder_forward (candle_models/modernbert.rs:61-86,121-213,234-240,283-305;
// candle-transformers bert.rs for BERT, whose biases the GEMM epilogue adds in fp32).
#include <cuda_fp16.h>

#include <cmath>

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

// ---- gelu_erf in place over fp32 [T, I] (BERT's HiddenAct::Gelu; the GEMM has added the bias)
__global__ void gelu_f32_kernel(float* __restrict__ x, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float a = x[i];
  x[i] = 0.5f * a * (1.0f + erff(a * 0.70710678118654752440f));
}

// ---- fp32 softmax attention on the CUDA cores: one thread per query row, K / V tiles of 32 keys through shared memory,
// online softmax per tile (expf).  Heads of D = 32 or 64: qkv rows [T, 3 heads D], out rows [T, heads D], scores scaled
// by D^-1/2 on q.  window = 0: global, keys j < kv_lens[b] (kv_lens null: the whole sequence; every row stays a query);
// else |i - j| <= window.
// Each tile's weighted values are summed on their own and only then added to the running sums, o = o alpha + sum_j p_j v_j
// (one fmaf per tile): every term passes through at most 32 + tiles roundings.  One chain over every key would pass the
// first terms through n + n / 32 roundings, an error that increases linearly in n where the terms are correlated (constant
// V columns, near-uniform scores): oracle/precise_oracle.py.
constexpr int kARows = 64, kAKeys = 32;
template <int D>
__global__ void __launch_bounds__(kARows)
attention_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, const int* __restrict__ cu, int heads, int window,
                     float scale, const int* __restrict__ kv_lens) {
  __shared__ float ks[kAKeys][D], vs[kAKeys][D];
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kARows;
  const int seq0 = cu[b], len = cu[b + 1] - seq0;
  if (q0 >= len) return;
  const int klen = kv_lens ? min(len, kv_lens[b]) : len;   // keys >= klen are invisible to every query row
  const int H = heads * D;
  const int qi = q0 + threadIdx.x;
  const bool live = qi < len;
  float q[D], o[D];
  const float* qp = qkv + static_cast<size_t>(seq0 + (live ? qi : q0)) * 3 * H + h * D;
#pragma unroll
  for (int d = 0; d < D; ++d) { q[d] = qp[d] * scale; o[d] = 0.f; }
  float m = -INFINITY, l = 0.f;
  int k_lo = 0, k_hi = klen;
  if (window > 0) {
    k_lo = q0 - window > 0 ? q0 - window : 0;
    k_hi = q0 + kARows - 1 + window + 1 < len ? q0 + kARows + window : len;
  }
  for (int k0 = k_lo; k0 < k_hi; k0 += kAKeys) {
    __syncthreads();
    for (int e = threadIdx.x; e < kAKeys * D; e += kARows) {
      const int j = e / D, d = e % D;
      const bool ok = k0 + j < klen;
      const float* base = qkv + static_cast<size_t>(seq0 + (ok ? k0 + j : 0)) * 3 * H + h * D + d;
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
      for (int d = 0; d < D; ++d) acc = fmaf(q[d], ks[j][d], acc);
      const int kj = k0 + j;
      const bool vis = live && kj < klen && (window == 0 || (kj - qi <= window && qi - kj <= window));
      s[j] = vis ? acc : -INFINITY;
      tm = fmaxf(tm, s[j]);
    }
    if (tm == -INFINITY) continue;          // (uniform control flow is not required: no barrier inside)
    const float mn = fmaxf(m, tm);
    const float alpha = (m == -INFINITY) ? 0.f : expf(m - mn);
    float lt = 0.f;
#pragma unroll
    for (int j = 0; j < kAKeys; ++j) {      // s[j] becomes the weight p_j
      s[j] = (s[j] == -INFINITY) ? 0.f : expf(s[j] - mn);
      lt += s[j];
    }
    l = fmaf(l, alpha, lt);
#pragma unroll
    for (int d = 0; d < D; ++d) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < kAKeys; ++j) acc = fmaf(s[j], vs[j][d], acc);
      o[d] = fmaf(o[d], alpha, acc);
    }
    m = mn;
  }
  if (live) {
    float* op = out + static_cast<size_t>(seq0 + qi) * H + h * D;
    const float inv = 1.0f / l;
#pragma unroll
    for (int d = 0; d < D; ++d) op[d] = o[d] * inv;
  }
}

}  // namespace

int precise_split_rows(cudaStream_t s, const float* x, int T, int H, const float* gamma, float eps, __half* out) {
  if (T <= 0) return 0;
  const unsigned grid = static_cast<unsigned>((static_cast<size_t>(T) * 32 + 255) / 256);
  if (gamma) split_rows_kernel<true><<<grid, 256, 0, s>>>(x, T, H, gamma, eps, out);
  else split_rows_kernel<false><<<grid, 256, 0, s>>>(x, T, H, nullptr, 0.f, out);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int precise_rope(cudaStream_t s, float* qkv, const int* pos, int T, int heads, const float* cos_t, const float* sin_t) {
  const size_t n = static_cast<size_t>(T) * 2 * heads * 32;
  if (n == 0) return 0;
  rope_f32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(qkv, pos, T, heads, cos_t, sin_t);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int precise_geglu(cudaStream_t s, const float* ab, int T, int I, float* out) {
  const size_t n = static_cast<size_t>(T) * I;
  if (n == 0) return 0;
  geglu_f32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(ab, T, I, out);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int precise_gelu(cudaStream_t s, float* x, int T, int I) {
  const size_t n = static_cast<size_t>(T) * I;
  if (n == 0) return 0;
  gelu_f32_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, s>>>(x, n);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int precise_attention(cudaStream_t s, const float* qkv, float* out, const int* cu_seqlens, int batch, int max_len, int heads,
                      int head_dim, int window, const int* kv_lens) {
  if (head_dim != 32 && head_dim != 64) {
    fprintf(stderr, "[srb200] precise_attention: head_dim %d (32 or 64)\n", head_dim);
    return -1;
  }
  if (kv_lens && window > 0) {
    fprintf(stderr, "[srb200] precise_attention: kv_lens applies to global attention only\n");
    return -1;
  }
  if (batch <= 0 || max_len <= 0) return 0;
  // D^-1/2: 0.125 exactly for D = 64, fp32(32^-1/2) for D = 32
  const float scale = head_dim == 64 ? 0.125f : 0.17677669529663688110f;
  // gridDim.z holds at most 65 535 sequences: larger packs run as slices (the kernel reads absolute offsets from cu)
  for (int b0 = 0; b0 < batch; b0 += kMaxGridZ) {
    const int nb = batch - b0 < kMaxGridZ ? batch - b0 : kMaxGridZ;
    const dim3 grid((max_len + kARows - 1) / kARows, heads, nb);
    const int* kl = kv_lens ? kv_lens + b0 : nullptr;
    if (head_dim == 64) attention_f32_kernel<64><<<grid, kARows, 0, s>>>(qkv, out, cu_seqlens + b0, heads, window, scale, kl);
    else attention_f32_kernel<32><<<grid, kARows, 0, s>>>(qkv, out, cu_seqlens + b0, heads, window, scale, kl);
    SRB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  }
  return 0;
}

int encoder_forward_precise(Model& m, const int* d_ids, const int* d_cu, int B, int T, int max_len, int L) {
  const EncoderConfig& c = m.cfg;
  Workspace& w = m.ws;
  PreciseState& p = m.precise;
  cudaStream_t s = m.stream;
  const int H = c.H, I = c.I;
  const bool bert = c.arch == ARCH_BERT;
  const TaskTensors& task = m.task[0];
  // out = [out +] split(A) W'^T [+ bias] in fp32 (EPI_RESID; resid null: a plain store)
  auto gemm = [&](const __half* a, const __half* wt, int n, int k, float* out, bool resid, const float* bias) {
    GemmDesc g;
    g.M = T; g.a_rows = w.cap_tokens; g.N = n; g.K = 3 * k; g.A = a; g.W = wt; g.out = out; g.ldo = n;
    g.epi = EPI_RESID;
    g.resid = resid ? out : nullptr;
    g.ldr = n;
    g.bias = bias;
    return gemm_f16(s, g);
  };
  if (bert) {
    // candle's post-LN BertLayer: x = LN(x + attn(x) Wo + bo), then x = LN(x + gelu(x Wi + bi) Wo2 + bo2)
    if (embed_ln_bert(s, d_ids, w.pos, T, H, c.vocab, c.max_pos, task.emb_word, task.emb_pos, task.emb_type0, task.emb_ln_w,
                      task.emb_ln_b, c.ln_eps, w.x, w.h))
      return -1;
    for (int li = 0; li < L; ++li) {
      const TaskNorms& norms = task.layers[li];
      const PreciseLayer& pl = p.layers[li];
      if (precise_split_rows(s, w.x, T, H, nullptr, 0.f, w.split)) return -1;
      if (gemm(w.split, pl.wqkv, 3 * H, H, w.qkv32, false, pl.bqkv)) return -1;
      if (precise_attention(s, w.qkv32, w.ctx32, d_cu, B, max_len, c.heads, H / c.heads, 0, m.cur_kv_lens)) return -1;
      if (precise_split_rows(s, w.ctx32, T, H, nullptr, 0.f, w.split)) return -1;
      if (gemm(w.split, pl.wo, H, H, w.x, true, pl.bo)) return -1;
      if (layernorm_rows(s, w.x, T, H, norms.mid_w, norms.mid_b, c.ln_eps, w.x, nullptr)) return -1;
      if (precise_split_rows(s, w.x, T, H, nullptr, 0.f, w.split)) return -1;
      if (gemm(w.split, pl.wi, I, H, w.mid32, false, pl.bi)) return -1;
      if (precise_gelu(s, w.mid32, T, I)) return -1;
      if (precise_split_rows(s, w.mid32, T, I, nullptr, 0.f, w.split)) return -1;
      if (gemm(w.split, pl.wo2, H, I, w.x, true, pl.bo2)) return -1;
      if (layernorm_rows(s, w.x, T, H, norms.out_w, norms.out_b, c.ln_eps, w.x, nullptr)) return -1;
    }
    SRB_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  if (embed_ln_modernbert(s, d_ids, T, H, c.vocab, task.emb_word, task.emb_ln_w, c.ln_eps, w.x, w.h)) return -1;
  for (int li = 0; li < L; ++li) {
    const TaskNorms& norms = task.layers[li];
    const PreciseLayer& pl = p.layers[li];
    const bool local = (li % c.global_every) != 0;
    // attention input: LayerNorm (none on layer 0, modernbert.rs:266-271), split
    if (precise_split_rows(s, w.x, T, H, norms.attn_w, c.ln_eps, w.split)) return -1;
    if (gemm(w.split, pl.wqkv, 3 * H, H, w.qkv32, false, nullptr)) return -1;
    if (precise_rope(s, w.qkv32, w.pos, T, c.heads, local ? m.rope_cos_l : m.rope_cos_g, local ? m.rope_sin_l : m.rope_sin_g))
      return -1;
    if (precise_attention(s, w.qkv32, w.ctx32, d_cu, B, max_len, c.heads, 64, local ? c.local_attention / 2 : 0, nullptr))
      return -1;
    if (precise_split_rows(s, w.ctx32, T, H, nullptr, 0.f, w.split)) return -1;
    if (gemm(w.split, pl.wo, H, H, w.x, true, nullptr)) return -1;
    if (precise_split_rows(s, w.x, T, H, norms.mid_w, c.ln_eps, w.split)) return -1;
    if (gemm(w.split, pl.wi, 2 * I, H, w.mid32, false, nullptr)) return -1;
    if (precise_geglu(s, w.mid32, T, I, w.act32)) return -1;
    if (precise_split_rows(s, w.act32, T, I, nullptr, 0.f, w.split)) return -1;
    if (gemm(w.split, pl.wo2, H, I, w.x, true, nullptr)) return -1;
  }
  SRB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace srb
