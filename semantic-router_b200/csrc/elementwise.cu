// HBM-bound kernels of the encoder path: token-embedding gather + LayerNorm, row LayerNorm, pooling,
// L2 normalisation, sequence / token classification heads.  One warp per row, float4 coalesced loads,
// warp-shuffle reductions, fp32 statistics throughout.
//
// Reference semantics (paths relative to candle-binding/src/):
//   embeddings      model_architectures/traditional/candle_models/modernbert.rs:466 (tok_embeddings -> norm)
//   LayerNorm       candle_nn::LayerNorm (remove_mean, biased variance, eps inside the sqrt)
//   mean pooling    model_architectures/traditional/modernbert.rs:1146-1169, embedding/pooling.rs:57-85
//   head            model_architectures/traditional/modernbert.rs:303-329 (dense -> gelu(tanh) -> LN eps 1e-12)
//   classifier      modernbert.rs:490-497 (Linear + softmax), argmax :1184-1192 (first max);
//                   traditional/bert.rs:237-252 (pooler -> tanh -> classifier -> softmax -> max_by = last max)
//   l2 normalise    embedding/mmbert_embedding.rs:781-796 (norm + 1e-12), core/similarity.rs:338-341 (no eps)
#include "kernels.h"

#include "common.cuh"

namespace srb {
namespace {

// ---- per-warp row helpers: a row of H = 128*NV floats, lane holds float4 #(i*32+lane) for i < NV
template <int NV>
__device__ __forceinline__ void row_load(const float* row, float4 (&v)[NV]) {
  const float4* r4 = reinterpret_cast<const float4*>(row);
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = __ldg(r4 + i * 32 + lane_id());
}
template <int NV>
__device__ __forceinline__ void row_layernorm(float4 (&v)[NV], const float* w, const float* b, float eps) {
  constexpr float inv_h = 1.0f / (NV * 128);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) * inv_h;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
    q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) * inv_h + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float4 ww = __ldg(reinterpret_cast<const float4*>(w) + i * 32 + lane_id());
    v[i].x = v[i].x * rstd * ww.x; v[i].y = v[i].y * rstd * ww.y;
    v[i].z = v[i].z * rstd * ww.z; v[i].w = v[i].w * rstd * ww.w;
    if (b) {
      const float4 bb = __ldg(reinterpret_cast<const float4*>(b) + i * 32 + lane_id());
      v[i].x += bb.x; v[i].y += bb.y; v[i].z += bb.z; v[i].w += bb.w;
    }
  }
}
template <int NV>
__device__ __forceinline__ void row_store32(float* row, const float4 (&v)[NV]) {
  float4* r4 = reinterpret_cast<float4*>(row);
#pragma unroll
  for (int i = 0; i < NV; ++i) r4[i * 32 + lane_id()] = v[i];
}
template <int NV>
__device__ __forceinline__ void row_store16(__half* row, const float4 (&v)[NV]) {
  uint2* r2 = reinterpret_cast<uint2*>(row);
#pragma unroll
  for (int i = 0; i < NV; ++i)
    r2[i * 32 + lane_id()] = make_uint2(pack_half2(v[i].x, v[i].y), pack_half2(v[i].z, v[i].w));
}

constexpr int kRowThreads = 256;  // 8 rows per CTA

// group of a row in a grouped pass (RowGroups): 0 when the launch is not grouped
__device__ __forceinline__ int row_group(int row, int group_rows) { return group_rows > 0 ? row / group_rows : 0; }

template <int NV>
__global__ void __launch_bounds__(kRowThreads)
embed_ln_mb_kernel(const int* __restrict__ ids, int T, int vocab, const __grid_constant__ RowGroups table,
                   const __grid_constant__ RowGroups w, int group_rows, float eps, float* __restrict__ x,
                   __half* __restrict__ h, __half* __restrict__ lo) {
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
  if (row >= T) return;
  const int g = row_group(row, group_rows);
  int id = __ldg(ids + row);
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  float4 v[NV];
  row_load<NV>(table.p[g] + static_cast<size_t>(id) * (NV * 128), v);
  row_layernorm<NV>(v, w.p[g], nullptr, eps);
  if (x) row_store32<NV>(x + static_cast<size_t>(row) * (NV * 128), v);
  row_store16<NV>(h + static_cast<size_t>(row) * (NV * 128), v);
  if (lo) {   // residual stream as an fp16 pair (gemm.h: EPI_RESID_HL): lo = fp16(x - fp16(x))
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      v[i].x -= __half2float(__float2half_rn(v[i].x)); v[i].y -= __half2float(__float2half_rn(v[i].y));
      v[i].z -= __half2float(__float2half_rn(v[i].z)); v[i].w -= __half2float(__float2half_rn(v[i].w));
    }
    row_store16<NV>(lo + static_cast<size_t>(row) * (NV * 128), v);
  }
}

// x = pivot[row] + hi + lo: the fp32 form of a residual stream held as an fp16 pair (gemm.h: EPI_RESID_HL)
__global__ void hl_to_f32_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, const float* __restrict__ pivot,
                                 size_t n8, int h8, float* __restrict__ x) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const float pv = pivot ? __ldg(pivot + i / h8) : 0.f;
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(hi) + i), b = __ldg(reinterpret_cast<const uint4*>(lo) + i);
  const uint32_t au[4] = {a.x, a.y, a.z, a.w}, bu[4] = {b.x, b.y, b.z, b.w};
  float o[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&au[k]));
    const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&bu[k]));
    o[2 * k] = pv + (fa.x + fb.x);
    o[2 * k + 1] = pv + (fa.y + fb.y);
  }
  float4* dst = reinterpret_cast<float4*>(x) + 2 * i;
  dst[0] = make_float4(o[0], o[1], o[2], o[3]);
  dst[1] = make_float4(o[4], o[5], o[6], o[7]);
}

template <int NV>
__global__ void __launch_bounds__(kRowThreads)
embed_ln_bert_kernel(const int* __restrict__ ids, const int* __restrict__ pos, int T, int vocab, int max_pos,
                     const __grid_constant__ RowGroups word, const __grid_constant__ RowGroups pos_emb,
                     const __grid_constant__ RowGroups type0, const __grid_constant__ RowGroups w,
                     const __grid_constant__ RowGroups b, int group_rows, float eps, float* __restrict__ x,
                     __half* __restrict__ h) {
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
  if (row >= T) return;
  const int g = row_group(row, group_rows);
  int id = __ldg(ids + row);
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  int p = __ldg(pos + row);
  p = p >= max_pos ? max_pos - 1 : p;
  float4 v[NV], a[NV];
  row_load<NV>(word.p[g] + static_cast<size_t>(id) * (NV * 128), v);
  row_load<NV>(type0.p[g], a);   // reference order: word + token_type, then + position
#pragma unroll
  for (int i = 0; i < NV; ++i) { v[i].x += a[i].x; v[i].y += a[i].y; v[i].z += a[i].z; v[i].w += a[i].w; }
  row_load<NV>(pos_emb.p[g] + static_cast<size_t>(p) * (NV * 128), a);
#pragma unroll
  for (int i = 0; i < NV; ++i) { v[i].x += a[i].x; v[i].y += a[i].y; v[i].z += a[i].z; v[i].w += a[i].w; }
  row_layernorm<NV>(v, w.p[g], b.p[g], eps);
  row_store32<NV>(x + static_cast<size_t>(row) * (NV * 128), v);
  row_store16<NV>(h + static_cast<size_t>(row) * (NV * 128), v);
}

template <int NV>
__global__ void __launch_bounds__(kRowThreads)
layernorm_kernel(const float* x, int T, const __grid_constant__ RowGroups w, const __grid_constant__ RowGroups b,
                 int group_rows, float eps, float* y32, __half* __restrict__ y16) {
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
  if (row >= T) return;
  const int g = row_group(row, group_rows);
  float4 v[NV];
  const float4* r4 = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * (NV * 128));
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = r4[i * 32 + lane_id()];
  row_layernorm<NV>(v, w.p[g], b.p[g], eps);
  if (y32) row_store32<NV>(y32 + static_cast<size_t>(row) * (NV * 128), v);
  if (y16) row_store16<NV>(y16 + static_cast<size_t>(row) * (NV * 128), v);
}

// thread i < n / 4 converts float4 #i; thread n / 4 converts the last n % 4 elements one by one
__global__ void cast_f16_kernel(const float* __restrict__ x, size_t n, __half* __restrict__ y) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t n4 = n / 4;
  if (i < n4) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    reinterpret_cast<uint2*>(y)[i] = make_uint2(pack_half2(v.x, v.y), pack_half2(v.z, v.w));
  } else if (i == n4) {
    for (size_t j = 4 * n4; j < n; ++j) y[j] = __float2half_rn(__ldg(x + j));
  }
}

__global__ void positions_kernel(const int* __restrict__ cu, int* __restrict__ pos) {
  const int b = blockIdx.x;
  const int s = cu[b], e = cu[b + 1];
  for (int t = s + threadIdx.x; t < e; t += blockDim.x) pos[t] = t - s;
}

// kPoolParts CTAs per sequence (a lone 512-token prompt would otherwise walk 64 rows per warp back to back, which is
// pure latency); 64 "virtual warps" stride over the tokens, each CTA reduces its 8 warps in order into a partial row,
// and the CTA that arrives last adds the partials in index order -- the result does not depend on arrival order or on
// what else is in the batch.
template <int NV>
__global__ void __launch_bounds__(kRowThreads)
pool_kernel(const float* __restrict__ x, const int* __restrict__ cu, int mode, const float* __restrict__ w,
            const float* __restrict__ b, float eps, float* __restrict__ pooled, float* __restrict__ part,
            int* __restrict__ arrived, const int* __restrict__ div_lens) {
  constexpr int H = NV * 128;
  constexpr int kWarps = kRowThreads / 32;
  __shared__ float4 red[kRowThreads / 32][NV * 32];
  __shared__ int s_last;
  const int seq = blockIdx.x;
  const int s = cu[seq], e = cu[seq + 1];
  const int warp = threadIdx.x >> 5;
  const int vwarp = blockIdx.y * kWarps + warp;
  float4 acc[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int last = (mode == POOL_CLS) ? (s + 1 < e ? s + 1 : e) : e;
  for (int t = s + vwarp; t < last; t += kPoolParts * kWarps) {
    float4 v[NV];
    row_load<NV>(x + static_cast<size_t>(t) * H, v);
    if (w) row_layernorm<NV>(v, w, b, eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) { acc[i].x += v[i].x; acc[i].y += v[i].y; acc[i].z += v[i].z; acc[i].w += v[i].w; }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) red[warp][i * 32 + lane_id()] = acc[i];
  __syncthreads();
  float4* mine = reinterpret_cast<float4*>(part + (static_cast<size_t>(seq) * kPoolParts + blockIdx.y) * H);
  for (int c = threadIdx.x; c < NV * 32; c += kRowThreads) {
    float4 t = red[0][c];
#pragma unroll
    for (int k = 1; k < kWarps; ++k) { t.x += red[k][c].x; t.y += red[k][c].y; t.z += red[k][c].z; t.w += red[k][c].w; }
    mine[c] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(arrived + seq, 1) == kPoolParts - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // div_lens: BertSimilarity under a fixed-padding tokenizer sums EVERY position (pads included) and divides by the
  // number of real tokens (core/similarity.rs:220-222)
  const int n_div = div_lens ? div_lens[seq] : e - s;
  const float inv = (mode == POOL_CLS) ? 1.0f : 1.0f / static_cast<float>(n_div > 0 ? n_div : 1);
  const float4* all = reinterpret_cast<const float4*>(part + static_cast<size_t>(seq) * kPoolParts * H);
  for (int c = threadIdx.x; c < NV * 32; c += kRowThreads) {
    float4 t = __ldcg(all + c);
#pragma unroll
    for (int k = 1; k < kPoolParts; ++k) {
      const float4 u = __ldcg(all + k * (NV * 32) + c);
      t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
    }
    t.x *= inv; t.y *= inv; t.z *= inv; t.w *= inv;
    reinterpret_cast<float4*>(pooled + static_cast<size_t>(seq) * H)[c] = t;
  }
  if (threadIdx.x == 0) arrived[seq] = 0;   // ready for the next call on this stream
}

__global__ void l2norm_rows_kernel(const float* __restrict__ pooled, int batch, int H, int dim, float norm_eps,
                                   float* __restrict__ emb) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= batch) return;
  const float* p = pooled + static_cast<size_t>(row) * H;
  float s = 0.f;
  for (int i = lane_id(); i < dim; i += 32) { const float v = p[i]; s += v * v; }
  const float nrm = sqrtf(warp_sum(s)) + norm_eps;
  for (int i = lane_id(); i < dim; i += 32) emb[static_cast<size_t>(row) * dim + i] = p[i] / nrm;
}

// ---- sequence head: one CTA per sequence
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane_id() == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int k = 0; k < (blockDim.x >> 5); ++k) t += red[k];
  return t;
}

constexpr int kHeadThreads = 1024;   // the dense layer is a latency-bound GEMV: 32 warps x 4 rows in flight per CTA
__global__ void __launch_bounds__(kHeadThreads)
seq_head_kernel(const float* __restrict__ pooled, int H, SeqHeadWeights w, float* __restrict__ logits,
                float* __restrict__ probs, int* __restrict__ cls, float* __restrict__ conf) {
  extern __shared__ float sh[];  // [H] in, [H] hidden, [C] logits, [32] red
  float* in = sh;
  float* hid = sh + H;
  float* lg = hid + H;
  float* red = lg + w.num_classes;
  const int seq = blockIdx.x;
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int i = threadIdx.x; i < H; i += blockDim.x) in[i] = pooled[static_cast<size_t>(seq) * H + i];
  __syncthreads();
  if (w.dense_mode == 1 || w.dense_mode == 2) {  // y[o] = sum_k in[k] * W[o,k]
    for (int o = warp * 4; o < H; o += nwarps * 4) {   // four output rows per warp pass: four independent load streams
      const float* wr = w.dense_w + static_cast<size_t>(o) * H;
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
      for (int k = lane_id() * 4; k < H; k += 128) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(wr + k));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(wr + H + k));
        const float4 w2 = __ldg(reinterpret_cast<const float4*>(wr + 2 * H + k));
        const float4 w3 = __ldg(reinterpret_cast<const float4*>(wr + 3 * H + k));
        const float a0 = in[k], a1 = in[k + 1], a2 = in[k + 2], a3 = in[k + 3];
        s0 += a0 * w0.x + a1 * w0.y + a2 * w0.z + a3 * w0.w;
        s1 += a0 * w1.x + a1 * w1.y + a2 * w1.z + a3 * w1.w;
        s2 += a0 * w2.x + a1 * w2.y + a2 * w2.z + a3 * w2.w;
        s3 += a0 * w3.x + a1 * w3.y + a2 * w3.z + a3 * w3.w;
      }
      s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2); s3 = warp_sum(s3);
      if (lane_id() == 0) {
        hid[o] = s0 + (w.dense_b ? w.dense_b[o] : 0.f);
        hid[o + 1] = s1 + (w.dense_b ? w.dense_b[o + 1] : 0.f);
        hid[o + 2] = s2 + (w.dense_b ? w.dense_b[o + 2] : 0.f);
        hid[o + 3] = s3 + (w.dense_b ? w.dense_b[o + 3] : 0.f);
      }
    }
  } else if (w.dense_mode == 3) {  // y[o] = sum_k in[k] * P[k,o]  (bert.rs:107 `pooler_weight.t()`)
    for (int o = threadIdx.x; o < H; o += blockDim.x) {
      float s = 0.f;
      for (int k = 0; k < H; ++k) s += in[k] * __ldg(w.dense_w + static_cast<size_t>(k) * H + o);
      hid[o] = s + (w.dense_b ? w.dense_b[o] : 0.f);
    }
  } else {
    for (int i = threadIdx.x; i < H; i += blockDim.x) hid[i] = in[i];
  }
  __syncthreads();
  if (w.dense_mode == 1) {  // gelu(tanh) -> LayerNorm(norm_w, zero bias, eps 1e-12)
    float s = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
      hid[i] = w.gelu_erf ? gelu_erf_f(hid[i]) : gelu_tanh_f(hid[i]);
      s += hid[i];
    }
    const float mean = block_sum(s, red) / H;
    float q = 0.f;
    for (int i = threadIdx.x; i < H; i += blockDim.x) { const float d = hid[i] - mean; q += d * d; }
    const float rstd = 1.0f / sqrtf(block_sum(q, red) / H + w.head_eps);
    for (int i = threadIdx.x; i < H; i += blockDim.x) hid[i] = (hid[i] - mean) * rstd * w.norm_w[i];
    __syncthreads();
  } else if (w.dense_mode == 2 || w.dense_mode == 3) {
    for (int i = threadIdx.x; i < H; i += blockDim.x) hid[i] = tanhf(hid[i]);
    __syncthreads();
  }
  const int C = w.num_classes;
  for (int c = warp; c < C; c += nwarps) {
    const float* wr = w.cls_w + static_cast<size_t>(c) * H;
    float s = 0.f;
    for (int k = lane_id() * 4; k < H; k += 128) {
      const float4 ww = __ldg(reinterpret_cast<const float4*>(wr + k));
      s += hid[k] * ww.x + hid[k + 1] * ww.y + hid[k + 2] * ww.z + hid[k + 3] * ww.w;
    }
    s = warp_sum(s);
    if (lane_id() == 0) lg[c] = s + (w.cls_b ? w.cls_b[c] : 0.f);
  }
  __syncthreads();
  if (warp == 0) {
    float mx = -INFINITY;
    for (int c = lane_id(); c < C; c += 32) mx = fmaxf(mx, lg[c]);
    mx = warp_max(mx);
    float s = 0.f;
    for (int c = lane_id(); c < C; c += 32) s += expf(lg[c] - mx);
    s = warp_sum(s);
    for (int c = lane_id(); c < C; c += 32) {
      const float pr = expf(lg[c] - mx) / s;
      probs[static_cast<size_t>(seq) * C + c] = pr;
      logits[static_cast<size_t>(seq) * C + c] = lg[c];
      lg[c] = pr;  // reuse as probabilities for the argmax below
    }
    __syncwarp();
    if (lane_id() == 0) {
      int best = 0;
      float bv;
      if (w.argmax_last) {  // Iterator::max_by: later element wins on ties
        bv = lg[0];
        for (int c = 1; c < C; ++c) if (!(lg[c] < bv)) { bv = lg[c]; best = c; }
      } else {              // strict > starting from 0.0: first max wins
        bv = 0.f;
        for (int c = 0; c < C; ++c) if (lg[c] > bv) { bv = lg[c]; best = c; }
      }
      cls[seq] = best;
      conf[seq] = bv;
    }
  }
}

// ---- token head: one warp per token
template <int NV>
__global__ void __launch_bounds__(kRowThreads)
token_head_kernel(const float* __restrict__ hidden32, const __half* __restrict__ dense16, int T,
                  const float* __restrict__ norm_w, const float* __restrict__ pre_ln_w, float pre_ln_eps,
                  const float* __restrict__ cls_w,
                  const float* __restrict__ cls_b, int C, int argmax_last, float* __restrict__ logits,
                  float* __restrict__ probs, int* __restrict__ pred, float* __restrict__ conf, int gelu_erf,
                  float head_eps) {
  constexpr int H = NV * 128;
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5);
  if (row >= T) return;
  float4 v[NV];
  if (dense16) {
    const uint2* r2 = reinterpret_cast<const uint2*>(dense16 + static_cast<size_t>(row) * H);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const uint2 u = __ldg(r2 + i * 32 + lane_id());
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
      const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
      v[i] = gelu_erf ? make_float4(gelu_erf_f(a.x), gelu_erf_f(a.y), gelu_erf_f(b.x), gelu_erf_f(b.y))
                      : make_float4(gelu_tanh_f(a.x), gelu_tanh_f(a.y), gelu_tanh_f(b.x), gelu_tanh_f(b.y));
    }
    row_layernorm<NV>(v, norm_w, nullptr, head_eps);
  } else {
    row_load<NV>(hidden32 + static_cast<size_t>(row) * H, v);
    if (pre_ln_w) row_layernorm<NV>(v, pre_ln_w, nullptr, pre_ln_eps);
  }
  constexpr int kMaxSlots = 8;  // C <= 256
  float my[kMaxSlots];
#pragma unroll
  for (int s = 0; s < kMaxSlots; ++s) my[s] = -INFINITY;
  for (int c = 0; c < C; ++c) {
    const float4* wr = reinterpret_cast<const float4*>(cls_w + static_cast<size_t>(c) * H);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 ww = __ldg(wr + i * 32 + lane_id());
      s += v[i].x * ww.x + v[i].y * ww.y + v[i].z * ww.z + v[i].w * ww.w;
    }
    s = warp_sum(s) + (cls_b ? __ldg(cls_b + c) : 0.f);
    if ((c & 31) == static_cast<int>(lane_id())) {
#pragma unroll
      for (int k = 0; k < kMaxSlots; ++k) if (k == (c >> 5)) my[k] = s;
    }
  }
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < kMaxSlots; ++k) mx = fmaxf(mx, my[k]);
  mx = warp_max(mx);
  float se = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxSlots; ++k) if (k * 32 + static_cast<int>(lane_id()) < C) se += expf(my[k] - mx);
  se = warp_sum(se);
  // argmax over logits with the tie rule; ties resolved on the class index
  float bv = -INFINITY;
  int bi = argmax_last ? -1 : 0x7fffffff;
#pragma unroll
  for (int k = 0; k < kMaxSlots; ++k) {
    const int c = k * 32 + lane_id();
    if (c < C) {
      if (logits) logits[static_cast<size_t>(row) * C + c] = my[k];
      if (probs) probs[static_cast<size_t>(row) * C + c] = expf(my[k] - mx) / se;
      const bool better = my[k] > bv || (my[k] == bv && (argmax_last ? c > bi : c < bi));
      if (better) { bv = my[k]; bi = c; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    const bool better = ov > bv || (ov == bv && (argmax_last ? oi > bi : oi < bi));
    if (better) { bv = ov; bi = oi; }
  }
  if (lane_id() == 0) {
    pred[row] = bi;
    conf[row] = expf(bv - mx) / se;
  }
}

#define SRB_DISPATCH_H(H, ...)                                  \
  switch (H) {                                                  \
    case 384: { constexpr int NV = 3; __VA_ARGS__; break; }     \
    case 768: { constexpr int NV = 6; __VA_ARGS__; break; }     \
    case 1024: { constexpr int NV = 8; __VA_ARGS__; break; }    \
    default:                                                    \
      fprintf(stderr, "[srb200] unsupported hidden size %d (384/768/1024)\n", H); \
      return -1;                                                \
  }

inline int row_blocks(int T) { return (T + kRowThreads / 32 - 1) / (kRowThreads / 32); }

}  // namespace

int compute_positions(cudaStream_t stream, const int* cu_seqlens, int batch, int* pos) {
  if (batch <= 0) return 0;
  positions_kernel<<<batch, 128, 0, stream>>>(cu_seqlens, pos);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int embed_ln_modernbert(cudaStream_t stream, const int* ids, int T, int H, int vocab, const float* table,
                        const float* ln_w, float eps, float* x, __half* h, __half* lo) {
  return embed_ln_modernbert(stream, ids, T, H, vocab, RowGroups::one(table), RowGroups::one(ln_w), 0, eps, x, h, lo);
}

int embed_ln_modernbert(cudaStream_t stream, const int* ids, int T, int H, int vocab, const RowGroups& table,
                        const RowGroups& ln_w, int group_rows, float eps, float* x, __half* h, __half* lo) {
  if (T <= 0) return 0;
  if (group_rows < 0 || (group_rows > 0 && (T + group_rows - 1) / group_rows > kMaxRowGroups)) return -1;
  SRB_DISPATCH_H(H, (embed_ln_mb_kernel<NV><<<row_blocks(T), kRowThreads, 0, stream>>>(ids, T, vocab, table, ln_w,
                                                                                        group_rows, eps, x, h, lo)));
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int hl_to_f32(cudaStream_t stream, const __half* hi, const __half* lo, const float* pivot, int T, int H, float* x) {
  if (T <= 0) return 0;
  if (H % 8 != 0) return -1;
  const size_t n8 = static_cast<size_t>(T) * H / 8;
  hl_to_f32_kernel<<<static_cast<unsigned>((n8 + 255) / 256), 256, 0, stream>>>(hi, lo, pivot, n8, H / 8, x);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int embed_ln_bert(cudaStream_t stream, const int* ids, const int* pos, int T, int H, int vocab, int max_pos,
                  const float* word, const float* pos_emb, const float* type0, const float* ln_w,
                  const float* ln_b, float eps, float* x, __half* h) {
  return embed_ln_bert(stream, ids, pos, T, H, vocab, max_pos, RowGroups::one(word), RowGroups::one(pos_emb),
                       RowGroups::one(type0), RowGroups::one(ln_w), RowGroups::one(ln_b), 0, eps, x, h);
}

int embed_ln_bert(cudaStream_t stream, const int* ids, const int* pos, int T, int H, int vocab, int max_pos,
                  const RowGroups& word, const RowGroups& pos_emb, const RowGroups& type0, const RowGroups& ln_w,
                  const RowGroups& ln_b, int group_rows, float eps, float* x, __half* h) {
  if (T <= 0) return 0;
  if (group_rows < 0 || (group_rows > 0 && (T + group_rows - 1) / group_rows > kMaxRowGroups)) return -1;
  SRB_DISPATCH_H(H, (embed_ln_bert_kernel<NV><<<row_blocks(T), kRowThreads, 0, stream>>>(
                        ids, pos, T, vocab, max_pos, word, pos_emb, type0, ln_w, ln_b, group_rows, eps, x, h)));
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int layernorm_rows(cudaStream_t stream, const float* x, int T, int H, const float* w, const float* b, float eps,
                   float* y32, __half* y16) {
  return layernorm_rows(stream, x, T, H, RowGroups::one(w), RowGroups::one(b), 0, eps, y32, y16);
}

int layernorm_rows(cudaStream_t stream, const float* x, int T, int H, const RowGroups& w, const RowGroups& b,
                   int group_rows, float eps, float* y32, __half* y16) {
  if (T <= 0) return 0;
  if (group_rows < 0 || (group_rows > 0 && (T + group_rows - 1) / group_rows > kMaxRowGroups)) return -1;
  SRB_DISPATCH_H(H, (layernorm_kernel<NV><<<row_blocks(T), kRowThreads, 0, stream>>>(x, T, w, b, group_rows, eps, y32,
                                                                                      y16)));
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int cast_rows_f16(cudaStream_t stream, const float* x, size_t n, __half* y) {
  if (n == 0) return 0;
  const size_t threads = n / 4 + (n % 4 != 0);
  cast_f16_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, stream>>>(x, n, y);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int pool_rows(cudaStream_t stream, const float* x, const int* cu_seqlens, int batch, int H, PoolMode mode,
              const float* ln_w, const float* ln_b, float eps, float* pooled, float* part, int* arrived, const int* div_lens) {
  if (batch <= 0) return 0;
  if (!part || !arrived) return -1;
  SRB_DISPATCH_H(H, (pool_kernel<NV><<<dim3(batch, kPoolParts), kRowThreads, 0, stream>>>(
                        x, cu_seqlens, static_cast<int>(mode), ln_w, ln_b, eps, pooled, part, arrived, div_lens)));
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int l2_normalize_rows(cudaStream_t stream, const float* pooled, int batch, int H, int dim, float norm_eps,
                      float* emb) {
  if (batch <= 0) return 0;
  l2norm_rows_kernel<<<(batch + 7) / 8, 256, 0, stream>>>(pooled, batch, H, dim, norm_eps, emb);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int seq_head(cudaStream_t stream, const float* pooled, int batch, int H, const SeqHeadWeights& w, float* logits,
             float* probs, int* cls, float* conf) {
  if (batch <= 0) return 0;
  if (H % 128 != 0 || w.num_classes <= 0) return -1;
  const size_t smem = (2 * H + w.num_classes + 32) * sizeof(float);
  seq_head_kernel<<<batch, kHeadThreads, smem, stream>>>(pooled, H, w, logits, probs, cls, conf);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

int token_head(cudaStream_t stream, const float* hidden32, const __half* dense16, int T, int H,
               const float* norm_w, const float* pre_ln_w, float pre_ln_eps, const float* cls_w,
               const float* cls_b, int C, int argmax_last, float* logits, float* probs, int* pred, float* conf,
               int gelu_erf, float head_eps) {
  if (T <= 0) return 0;
  if (C > 256 || C <= 0) {
    fprintf(stderr, "[srb200] token_head: %d classes unsupported (1..256)\n", C);
    return -1;
  }
  SRB_DISPATCH_H(H, (token_head_kernel<NV><<<row_blocks(T), kRowThreads, 0, stream>>>(
                        hidden32, dense16, T, norm_w, pre_ln_w, pre_ln_eps, cls_w, cls_b, C, argmax_last, logits, probs, pred,
                        conf, gelu_erf, head_eps)));
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace srb
