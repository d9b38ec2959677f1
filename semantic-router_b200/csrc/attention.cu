// Variable-length, non-causal flash attention forward (fp16 in, fp32 softmax/accumulate, fp16 out).
//
// Replaces ModernBertAttention::compute_standard_attention + the materialised [B,12,S,S] score tensor and
// [S,S] local mask of the reference
// (candle-binding/src/model_architectures/traditional/candle_models/modernbert.rs:121-213,
//  355-393) and candle BertSelfAttention.  The padding mask ((1-mask)*f32::MIN) and the sliding-window
// mask (-inf where |i-j| > local_attention/2) are predicates here, never tensors: sequences are packed
// (cu_seqlens) so padded keys do not exist, and local layers only visit the key blocks inside the window.
//
// Data path: cp.async double-buffered K/V tiles in XOR-swizzled shared memory, ldmatrix fragments,
// mma.sync.m16n8k16.  The engine runs attention_wgmma.cu; this kernel is its independent comparator in the tests.
// One CTA = 64 query rows of one (sequence, head); 4 warps x 16 rows.
#include "kernels.h"

#include "common.cuh"

namespace srb {
namespace {

constexpr int kBQ = 64;   // query rows per CTA
constexpr int kBKV = 64;  // keys per block
constexpr int kD = 64;    // head dim

__device__ __forceinline__ uint32_t swz(int row, int chunk) {  // byte offset in a [rows][128 B] tile
  return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Load a [64 rows][64 halfs] tile (rows row0.. of this sequence, zero-filled past `len`) into swizzled smem.
__device__ __forceinline__ void load_tile(uint32_t smem_base, const __half* gbase, int ld, int row0, int len) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + i * 128;
    const int r = idx >> 3, c = idx & 7;
    const int grow = row0 + r;
    const bool ok = grow < len;
    const __half* src = gbase + static_cast<size_t>(ok ? grow : 0) * ld + c * 8;
    cp_async16(smem_base + swz(r, c), src, ok ? 16 : 0);
  }
}

__global__ void __launch_bounds__(128)
attn_fwd_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, const int* __restrict__ cu_seqlens,
                int num_heads, int window, float scale_log2) {
  __shared__ __align__(128) uint8_t smem[kBQ * 128 + 2 * 2 * kBKV * 128];
  const int b = blockIdx.z, h = blockIdx.y;
  const int seq0 = cu_seqlens[b];
  const int len = cu_seqlens[b + 1] - seq0;
  const int q0 = blockIdx.x * kBQ;
  if (q0 >= len) return;
  const int H = num_heads * kD;
  const int ld = 3 * H;
  const __half* qg = qkv + static_cast<size_t>(seq0) * ld + h * kD;
  const __half* kg = qg + H;
  const __half* vg = qg + 2 * H;

  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + kBQ * 128;
  const uint32_t sV = sK + 2 * kBKV * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  int kb_lo = 0, kb_hi = (len - 1) / kBKV;
  if (window > 0) {
    const int lo = q0 - window;
    kb_lo = lo > 0 ? lo / kBKV : 0;
    const int hi = q0 + kBQ - 1 + window;
    kb_hi = (hi < len - 1 ? hi : len - 1) / kBKV;
  }

  load_tile(sQ, qg, ld, q0, len);
  load_tile(sK, kg, ld, kb_lo * kBKV, len);
  load_tile(sV, vg, ld, kb_lo * kBKV, len);
  cp_async_commit();

  uint32_t qf[4][4];
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const int qrow0 = q0 + warp * 16 + (lane >> 2);  // this thread's rows: qrow0, qrow0+8

  for (int kb = kb_lo; kb <= kb_hi; ++kb) {
    const int buf = (kb - kb_lo) & 1;
    if (kb + 1 <= kb_hi) {
      load_tile(sK + (buf ^ 1) * kBKV * 128, kg, ld, (kb + 1) * kBKV, len);
      load_tile(sV + (buf ^ 1) * kBKV * 128, vg, ld, (kb + 1) * kBKV, len);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kb == kb_lo) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        ldsm_x4(sQ + swz(warp * 16 + (lane & 15), 2 * kk + (lane >> 4)), qf[kk][0], qf[kk][1], qf[kk][2],
                qf[kk][3]);
    }
    const uint32_t sKb = sK + buf * kBKV * 128, sVb = sV + buf * kBKV * 128;

    // ---- S = Q K^T (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        const int m = lane >> 3;
        uint32_t b0, b1, b2, b3;
        ldsm_x4(sKb + swz(8 * (2 * jp + (m >> 1)) + (lane & 7), 2 * kk + (m & 1)), b0, b1, b2, b3);
        mma16816(s[2 * jp], qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], b0, b1);
        mma16816(s[2 * jp + 1], qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], b2, b3);
      }
    }

    // ---- masking (sequence tail, sliding window)
    const int key0 = kb * kBKV + 2 * (lane & 3);
    const bool need_mask = (kb * kBKV + kBKV > len) || (window > 0);
    if (need_mask) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + 8 * j + (e & 1);
          const int qr = qrow0 + ((e >> 1) << 3);
          bool ok = key < len;
          if (window > 0) {
            const int d = key - qr;
            ok = ok && (d <= window) && (d >= -window);
          }
          if (!ok) s[j][e] = -INFINITY;
        }
      }
    }

    // ---- online softmax
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx[0] = fmaxf(mx[0], fmaxf(s[j][0], s[j][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[j][2], s[j][3]));
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[r] = exp2f((m_run[r] - m_use[r]) * scale_log2);
      m_run[r] = m_new;
      l_run[r] *= alpha[r];
    }
    uint32_t pf[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = exp2f((s[j][0] - m_use[0]) * scale_log2);
      const float p1 = exp2f((s[j][1] - m_use[0]) * scale_log2);
      const float p2 = exp2f((s[j][2] - m_use[1]) * scale_log2);
      const float p3 = exp2f((s[j][3] - m_use[1]) * scale_log2);
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pf[j >> 1][(j & 1) * 2 + 0] = pack_half2(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_half2(p2, p3);
      o[j][0] *= alpha[0]; o[j][1] *= alpha[0];
      o[j][2] *= alpha[1]; o[j][3] *= alpha[1];
    }

    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        const int m = lane >> 3;
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(sVb + swz(16 * kk + 8 * (m & 1) + (lane & 7), 2 * jp + (m >> 1)), b0, b1, b2, b3);
        mma16816(o[2 * jp], pf[kk][0], pf[kk][1], pf[kk][2], pf[kk][3], b0, b1);
        mma16816(o[2 * jp + 1], pf[kk][0], pf[kk][1], pf[kk][2], pf[kk][3], b2, b3);
      }
    }
    __syncthreads();  // all warps done with this K/V buffer before it is refilled
  }

  // ---- finalise: O /= l, stage through smem (reuse the Q tile), coalesced 16 B stores
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    l_run[r] = 1.f / l_run[r];
  }
  {
    const int r0 = warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t lo = pack_half2(o[j][0] * l_run[0], o[j][1] * l_run[0]);
      const uint32_t hi = pack_half2(o[j][2] * l_run[1], o[j][3] * l_run[1]);
      const uint32_t colb = (lane & 3) * 4;
      *reinterpret_cast<uint32_t*>(smem + swz(r0, j) + colb) = lo;
      *reinterpret_cast<uint32_t*>(smem + swz(r0 + 8, j) + colb) = hi;
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + i * 128;
    const int r = idx >> 3, c = idx & 7;
    if (q0 + r < len) {
      const uint4 v = *reinterpret_cast<const uint4*>(smem + swz(r, c));
      *reinterpret_cast<uint4*>(out + static_cast<size_t>(seq0 + q0 + r) * H + h * kD + c * 8) = v;
    }
  }
}

}  // namespace

int attention_fwd(cudaStream_t stream, const __half* qkv, __half* out, const int* cu_seqlens, int batch,
                  int max_len, int num_heads, int head_dim, int window) {
  if (head_dim != kD) {
    fprintf(stderr, "[srb200] attention_fwd: head_dim %d unsupported (64 only)\n", head_dim);
    return -1;
  }
  if (batch <= 0 || max_len <= 0) return 0;
  const dim3 grid((max_len + kBQ - 1) / kBQ, num_heads, batch);
  const float scale_log2 = 0.125f * 1.4426950408889634f;  // head_dim^-0.5 * log2(e)
  attn_fwd_kernel<<<grid, 128, 0, stream>>>(qkv, out, cu_seqlens, num_heads, window, scale_log2);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace srb
