// Common device helpers for the sm_90a kernels: mbarrier, TMA, warp reductions, vector loads, device math.
// Everything here is raw inline PTX or CUDA C++ -- no CUTLASS/CuTe.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace srb {

#define SRB_CUDA_CHECK(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      fprintf(stderr, "[srb200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, \
              __LINE__, cudaGetErrorString(_e));                                               \
      return srb::fail_cuda(_e);                                                               \
    }                                                                                          \
  } while (0)

inline int fail_cuda(cudaError_t) { return -1; }

constexpr int kWarp = 32;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ------------------------------------------------------------------------------------------
// warp reductions
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may
// become resident while its predecessor in the stream is still running; everything before griddep_wait() (barrier
// init, TMEM allocation, descriptor prefetch) then overlaps the predecessor's tail.  griddep_wait() returns once the
// predecessor grid has completed and its writes are visible; without the launch attribute both are no-ops.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Non-blocking probe (mbarrier.try_wait may suspend the thread for a hardware time slice when the phase is not
// complete; test_wait never does) -- for event loops that poll several barriers.
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Wait with a watchdog: a protocol bug traps (launch error) instead of hanging the GPU box.  The watchdog reads
// the clock only every 64K failed probes so the spin itself stays a two-instruction loop; kSleepNs > 0 backs the
// warp off between probes (producer-side waits) so it does not steal issue slots from the math warps.
// No printf on the trap path: inlined at every wait site it cost ~80 SASS instructions each -- a quarter of the
// attention kernel, which is instruction-cache bound -- and an out-of-line call would spill the caller's live
// registers at every site.  cuda-gdb / compute-sanitizer locate a trapped wait.
template <int kSleepNs = 0>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (kSleepNs > 0) __nanosleep(kSleepNs);
    if ((++spins & 0xFFFFu) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 8000000000LL) __trap();  // ~4 s at 2 GHz
    }
  }
}

// ------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) -- 2D tile load into 128B-swizzled shared memory
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
      "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                                 int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
      "r"(c1), "l"(policy)
      : "memory");
}
// The same load, delivered to every CTA of the cluster whose bit is set in `cta_mask`: the box lands at the same shared
// offset in each of them and signals the mbarrier at the same offset in each of them (complete_tx of the box bytes).
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0),
      "r"(c1), "h"(cta_mask)
      : "memory");
}
// Arrive on the mbarrier at the same shared offset as `bar` in CTA `cta` of the cluster (cluster rank; may be this CTA).
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}
// Every thread of every CTA of the cluster (a plain CTA barrier when the kernel runs without clusters).
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;

// ---- TMA store / bulk-group helpers (epilogue) -----------------------------------------------------
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// 16-byte chunk `c` of row `r` inside a 32-row x 128-byte box written/read by TMA with SWIZZLE_128B
__device__ __forceinline__ uint32_t box_off(int r, int c) { return static_cast<uint32_t>(r * 128 + ((c ^ (r & 7)) << 4)); }
__device__ __forceinline__ void sts16(uint8_t* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  *reinterpret_cast<uint4*>(p) = make_uint4(a, b, c, d);
}
__device__ __forceinline__ void sts_b32(uint8_t* p, uint32_t a) { *reinterpret_cast<uint32_t*>(p) = a; }


// ------------------------------------------------------------------------------------------
// explicit shared-memory vector accesses (avoid generic ST/LD through a converted pointer)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void sts128(uint32_t saddr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ float4 lds128f(uint32_t saddr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr));
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t saddr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(saddr), "f"(v) : "memory");
}
__device__ __forceinline__ float lds_f32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr) : "memory");
  return v;
}
__device__ __forceinline__ void sts128f(uint32_t saddr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 2^x on the FMA pipe (x <= 0 here; clamped at -125): round-to-nearest integer part through the magic-number add, 2^f on
// f in [-0.5, 0.5] by a degree-3 polynomial, exponent spliced in with an integer add.  Max relative error 8.4e-5 (minimax
// fit, tests/test_device_math_constants.py checks it) -- a sixth of the fp16 rounding (4.9e-4) a softmax probability gets before
// the PV MMA.  An alternative to the MUFU exp2 for kernels whose softmax is bounded by that unit.
__device__ __forceinline__ float ex2_poly(float x) {
  x = fmaxf(x, -125.0f);
  const float t = x + 12582912.0f;                    // 1.5 * 2^23
  const float f = x - (t - 12582912.0f);
  float p = fmaf(f, 0.055212993174791336f, 0.24271413683891296f);
  p = fmaf(p, f, 0.6932621598243713f);
  p = fmaf(p, f, 0.999919593334198f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
// three-input maximum
__device__ __forceinline__ float fmax3(float a, float b, float c) {
  return fmaxf(fmaxf(a, b), c);
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float gelu_erf_f(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
// Branch-free erf-GELU for the GEMM epilogues (the libdevice erff above costs two divergent polynomial branches per
// element, which made the GeGLU epilogue as long as its mainloop): erf(t) = 1 - 2^(-t P6(t)) on t = min(|z|, 4),
// P6 a weighted least-squares fit (tools/fit_erf.py); max |erf error| 3.3e-7, max |gelu error| 5e-7 over [-12, 12]
// (fp32 emulation) -- far below the fp16 rounding of the stored result.
__device__ __forceinline__ float gelu_erf_fast_f(float x) {
  const float z = x * 0.70710678118654752440f;
  const float t = fminf(fabsf(z), 4.0f);
  float p = -3.6191246181260794e-05f;
  p = fmaf(p, t, 5.4603693570243195e-05f);
  p = fmaf(p, t, 0.0032821965869516134f);
  p = fmaf(p, t, -0.03057790733873844f);
  p = fmaf(p, t, 0.14959882199764252f);
  p = fmaf(p, t, 0.9181672930717468f);
  p = fmaf(p, t, 1.6279274225234985f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-t * p));
  const float r = copysignf(1.0f - e, z);
  const float h = 0.5f * x;
  return fmaf(h, r, h);
}
// GeGLU with the LayerNorm-fold scale folded in: gelu_erf(a r) * (b r) with kz = r / sqrt(2), kh = r^2 / 2 -- thirteen
// instructions per output (the separate rstd multiplies and gelu_erf_fast_f took nineteen; the GeGLU epilogue is the
// bottleneck of its GEMM: 1.5 ms of 9.1 per step in the decomposition runs).  erf(t) = 1 - 2^(-t P4(t)), P4 the weighted fit of
// tools/fit_erf.py at degree 4: max |erf error| 1.4e-6, max |gelu error| 1.3e-6 -- two orders below the fp16 rounding of
// the stored product.
__device__ __forceinline__ float geglu_fold_f(float a, float b, float kz, float kh) {
  const float z = a * kz;
  const float t = fminf(fabsf(z), 4.0f);
  float p = 0.002819528104737401f;
  p = fmaf(p, t, -0.029150057584047318f);
  p = fmaf(p, t, 0.14815378189086914f);
  p = fmaf(p, t, 0.9187344908714294f);
  p = fmaf(p, t, 1.6278589963912964f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-t * p));
  const float r = copysignf(1.0f - e, z);
  const float hb = (a * b) * kh;
  return fmaf(hb, r, hb);
}
__device__ __forceinline__ float gelu_tanh_f(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  return 0.5f * x * (1.0f + tanhf(k0 * (x + k1 * x * x * x)));
}

}  // namespace srb
