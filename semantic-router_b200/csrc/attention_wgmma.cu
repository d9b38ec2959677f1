// Variable-length, non-causal flash attention forward on Hopper tensor cores (wgmma), head dim 64, fp16 in, fp32
// softmax / accumulate, fp16 out; optional sliding window |i - j| <= window and per-sequence key lengths (kv_lens).
//
// One CTA = one warpgroup = 64 query rows of one (sequence, head).  Per 64-key block:
//   S = Q K^T    : 4 x wgmma m64n64k16, both operands from 128B-swizzled shared memory (K-major)
//   softmax      : online, on the accumulator fragment (warp w holds rows 16w + lane/4 and +8, like mma.sync m16n8)
//   O += P V     : 4 x wgmma m64n64k16 with P as the register A operand (the S fragment repacked to fp16, no shared-memory
//                  round trip) and V as an MN-major B operand (the [keys][64] tile as it lies in memory)
// K / V blocks are double-buffered with cp.async into the same 128B-swizzle layout TMA would produce.
#include "kernels.h"

#include "common.cuh"

namespace srb {
namespace {

constexpr int kBQ = 64;   // query rows per CTA (one warpgroup)
constexpr int kBKV = 64;  // keys per block
constexpr int kD = 64;    // head dim
constexpr int kTile = 64 * 128;   // one [64 rows][64 fp16] swizzled tile

__device__ __forceinline__ uint32_t swz(int row, int chunk) {  // byte offset in a [rows][128 B] tile (= SWIZZLE_128B)
  return static_cast<uint32_t>(row * 128 + ((chunk ^ (row & 7)) << 4));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// [64 rows][64 halfs] of this sequence from row0 (zero-filled past `len`) into a swizzled tile
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

// wgmma descriptors, 128B swizzle (layout type 1 in bits [62,64)).  K-major: rows of 64 fp16, 8-row groups 1024 B apart.
// MN-major (the [k][n] tile with n contiguous, n = 64 = one swizzle atom): 8-row k groups 1024 B apart.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4) | (static_cast<uint64_t>(1) << 16) |
         (static_cast<uint64_t>(1024 >> 4) << 32) | (static_cast<uint64_t>(1) << 62);
}
__device__ __forceinline__ uint64_t desc_sw128_mn(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4) | (static_cast<uint64_t>(1024 >> 4) << 16) |
         (static_cast<uint64_t>(1024 >> 4) << 32) | (static_cast<uint64_t>(1) << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define SRB_D32(d)                                                                                                   \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),        \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),           \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),          \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// D[64 x 64] (+)= A[64 x 16] (smem, K-major) * B[64 x 16]^T (smem, K-major)
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : SRB_D32(d)
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
// D[64 x 64] += A[64 x 16] (registers: the m16n8k16 A fragment of this warp's 16 rows) * B[16 x 64] (smem, MN-major)
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : SRB_D32(d)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db)
      : "memory");
}
#undef SRB_D32

__global__ void __launch_bounds__(128)
attn_wgmma_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, const int* __restrict__ cu_seqlens,
                  int num_heads, int window, float scale_log2, const int* __restrict__ kv_lens) {
  __shared__ __align__(1024) uint8_t smem[5 * kTile];   // Q, K[2], V[2]
  const int b = blockIdx.z, h = blockIdx.y;
  const int seq0 = cu_seqlens[b];
  const int len = cu_seqlens[b + 1] - seq0;
  const int q0 = blockIdx.x * kBQ;
  if (q0 >= len) return;
  // keys >= klen are masked for every query row (kv_lens: right-padded sequences whose pads are queries)
  const int klen = kv_lens ? min(len, kv_lens[b]) : len;
  const int H = num_heads * kD;
  const int ld = 3 * H;
  const __half* qg = qkv + static_cast<size_t>(seq0) * ld + h * kD;
  const __half* kg = qg + H;
  const __half* vg = qg + 2 * H;

  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK = sQ + kTile;
  const uint32_t sV = sK + 2 * kTile;
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

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const int qrow0 = q0 + warp * 16 + (lane >> 2);  // this thread's rows: qrow0, qrow0 + 8

  for (int kb = kb_lo; kb <= kb_hi; ++kb) {
    const int buf = (kb - kb_lo) & 1;
    if (kb + 1 <= kb_hi) {
      load_tile(sK + (buf ^ 1) * kTile, kg, ld, (kb + 1) * kBKV, len);
      load_tile(sV + (buf ^ 1) * kTile, vg, ld, (kb + 1) * kBKV, len);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();   // cp.async (generic proxy) writes -> wgmma (async proxy) reads
    __syncthreads();
    const uint32_t sKb = sK + buf * kTile, sVb = sV + buf * kTile;

    // ---- S = Q K^T (64 x 64 per warpgroup; s[4j + e] = mma.sync fragment element (j, e))
    float s[32];
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_ss(s, desc_sw128(sQ + 32 * kk), desc_sw128(sKb + 32 * kk), kk > 0 ? 1u : 0u);
    wg_commit();
    wg_wait0();

    // ---- masking (sequence tail, key lengths, sliding window)
    const int key0 = kb * kBKV + 2 * (lane & 3);
    const bool need_mask = (kb * kBKV + kBKV > klen) || (window > 0);
    if (need_mask) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = key0 + 8 * j + (e & 1);
          const int qr = qrow0 + ((e >> 1) << 3);
          bool ok = key < klen;
          if (window > 0) {
            const int dd = key - qr;
            ok = ok && (dd <= window) && (dd >= -window);
          }
          if (!ok) s[4 * j + e] = -INFINITY;
        }
      }
    }

    // ---- online softmax
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * j], s[4 * j + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * j + 2], s[4 * j + 3]));
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
    uint32_t pf[4][4];   // P as the A operand of the PV product: k-chunk kk = keys [16 kk, 16 kk + 16)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = exp2f((s[4 * j] - m_use[0]) * scale_log2);
      const float p1 = exp2f((s[4 * j + 1] - m_use[0]) * scale_log2);
      const float p2 = exp2f((s[4 * j + 2] - m_use[1]) * scale_log2);
      const float p3 = exp2f((s[4 * j + 3] - m_use[1]) * scale_log2);
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pf[j >> 1][(j & 1) * 2 + 0] = pack_half2(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_half2(p2, p3);
      o[4 * j] *= alpha[0]; o[4 * j + 1] *= alpha[0];
      o[4 * j + 2] *= alpha[1]; o[4 * j + 3] *= alpha[1];
    }

    // ---- O += P V
    wg_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs(o, pf[kk], desc_sw128_mn(sVb + kk * 16 * 128));
    wg_commit();
    wg_wait0();
    __syncthreads();  // every warp done with this K/V buffer before it is refilled
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
      const uint32_t lo = pack_half2(o[4 * j] * l_run[0], o[4 * j + 1] * l_run[0]);
      const uint32_t hi = pack_half2(o[4 * j + 2] * l_run[1], o[4 * j + 3] * l_run[1]);
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

int attention_wgmma_fwd(cudaStream_t stream, const __half* qkv, __half* out, const int* cu_seqlens, int batch,
                        int max_len, int num_heads, int head_dim, int window, const int* kv_lens) {
  if (kv_lens && window > 0) {
    fprintf(stderr, "[srb200] attention_wgmma_fwd: kv_lens applies to global attention only\n");
    return -1;
  }
  if (head_dim != kD) {
    fprintf(stderr, "[srb200] attention_wgmma_fwd: head_dim %d unsupported (64 only)\n", head_dim);
    return -1;
  }
  if (batch <= 0 || max_len <= 0) return 0;
  const dim3 grid((max_len + kBQ - 1) / kBQ, num_heads, batch);
  const float scale_log2 = 0.125f * 1.4426950408889634f;  // head_dim^-0.5 * log2(e)
  attn_wgmma_kernel<<<grid, 128, 0, stream>>>(qkv, out, cu_seqlens, num_heads, window, scale_log2, kv_lens);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace srb
