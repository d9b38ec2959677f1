// Mainloop-only microbenchmark of the projection GEMM's tile shapes (sm_90a).
//
// Question it answers: at the ModernBERT-base projection shape (M = 131072, N = 2304, K = 768) is the mainloop of a
// 128 x 192 tile fed to TWO MMA warpgroups (m64n192k16, one 64-row half each) faster than today's 128 x 128 tile on ONE
// warpgroup (two m64n128k16 per k-step), and how does 128 x 256 on two warpgroups compare?  Each kernel is the
// projection GEMM's persistent, contiguous schedule and TMA ring (128B swizzle, 64-wide k-blocks, optional 1 x 2
// cluster with the A box multicast, as gemm_wgmma.cu), with NO epilogue: the accumulators are only stored behind a
// predicate that is false at run time, so the time is the operand feed and the tensor cores alone.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Xptxas -v \
//        -I semantic-router_b200/csrc tools/micro/wgmma_mainloop.cu -o /tmp/wgmma_mainloop
//   /tmp/wgmma_mainloop [M N K iters]
//
// Prints one line per (tile, warpgroups, cluster) configuration: ms per GEMM (CUDA events over `iters` launches after
// a warm-up) and TFLOP/s.  Read the card, its power limit and SM clock in the same run
// (nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"

using namespace srb;

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kStages = 4;

__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

__device__ __forceinline__ void wgmma_m64n128k16(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n192k16(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %98, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, "
      "%96, %97, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_m64n256k16(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db, uint32_t acc) {
  if constexpr (BN == 128) wgmma_m64n128k16(d, da, db, acc);
  else if constexpr (BN == 192) wgmma_m64n192k16(d, da, db, acc);
  else wgmma_m64n256k16(d, da, db, acc);
}

// BN: tile width.  NWG: MMA warpgroups -- 1: one warpgroup issues both 64-row halves (today's kernel), 2: warpgroup w
// owns rows 64 w .. 64 w + 63.  CN: cluster size along N (A box multicast).  Warpgroup 0 is the producer.
template <int BN, int NWG, int CN>
__global__ void __launch_bounds__(128 * (NWG + 1), 1)
mainloop_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, int M, int N,
                int K, int flag, float* sink) {
  constexpr int kABytes = BM * BK * 2, kBBytes = BN * BK * 2, kStageBytes = kABytes + kBBytes;
  constexpr int kAccRegs = BN / 2;        // fp32 accumulators per thread per 64-row half
  constexpr int kHalves = NWG == 1 ? 2 : 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_blocks = (M + BM - 1) / BM, n_blocks = (N + BN - 1) / BN, k_blocks = (K + BK - 1) / BK;
  const int rn = blockIdx.x % CN;
  const int n_cblocks = (n_blocks + CN - 1) / CN;
  const int num_tiles = m_blocks * n_cblocks;
  const int num_workers = gridDim.x / CN, bid = blockIdx.x / CN;
  const int base = num_tiles / num_workers, rem = num_tiles % num_workers;
  const int t_begin = bid * base + (bid < rem ? bid : rem);
  const int t_end = t_begin + base + (bid < rem ? 1 : 0);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4 * NWG * CN);
    }
    mbar_fence_init();
  }
  if constexpr (CN > 1) cluster_sync();
  else __syncthreads();

  if (warp < 4) {
    if constexpr (NWG == 2) setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      const int a_rows = BM / CN;
      for (int t = t_begin; t < t_end; ++t) {
        const int m_blk = t / n_cblocks, n_blk = (t % n_cblocks) * CN + rn;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], kStageBytes);
          uint8_t* da = smem_a + s * kABytes + rn * a_rows * (BK * 2);
          if (CN > 1) tma_load_2d_multicast(da, &tmap_a, &full_bar[s], kb * BK, m_blk * BM + rn * a_rows, (1u << CN) - 1);
          else tma_load_2d(da, &tmap_a, &full_bar[s], kb * BK, m_blk * BM);
          tma_load_2d(smem_b + s * kBBytes, &tmap_b, &full_bar[s], kb * BK, n_blk * BN);
          if (++s == kStages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    if constexpr (NWG == 2) setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;
    float acc[kHalves][kAccRegs];
    int s = 0;
    uint32_t ph = 0;
    auto release = [&](int st) {
      if (CN == 1) {
        if (lane == 0) mbar_arrive(&empty_bar[st]);
      } else if (lane < CN) {
        mbar_arrive_cluster(&empty_bar[st], lane);
      }
    };
    for (int t = t_begin; t < t_end; ++t) {
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[s], ph);
        wgmma_fence();
        const uint32_t a0 = smem_u32(smem_a + s * kABytes) + (NWG == 2 ? wg * 64 * 128 : 0);
        const uint32_t b0 = smem_u32(smem_b + s * kBBytes);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t db = gmma_desc_sw128(b0 + 32 * k);
          const uint32_t accum = (kb > 0 || k > 0) ? 1u : 0u;
#pragma unroll
          for (int h = 0; h < kHalves; ++h) wgmma_tile<BN>(acc[h], gmma_desc_sw128(a0 + h * 64 * 128 + 32 * k), db, accum);
        }
        wgmma_commit();
        wgmma_wait<1>();
        __syncwarp();
        if (prev >= 0) release(prev);
        prev = s;
        if (++s == kStages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (prev >= 0) release(prev);
      if (flag) {   // never at run time: keeps the accumulators live without an epilogue
        float v = 0.f;
#pragma unroll
        for (int h = 0; h < kHalves; ++h)
#pragma unroll
          for (int i = 0; i < kAccRegs; ++i) v += acc[h][i];
        sink[threadIdx.x] = v;
      }
    }
  }
  if constexpr (CN > 1) cluster_sync();
  else __syncthreads();
}

__global__ void fill_f16(__half* p, size_t n, uint32_t seed) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint32_t h = static_cast<uint32_t>(i) * 2654435761u ^ seed;
    h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12;
    p[i] = __float2half((static_cast<float>(h & 0xFFFF) / 32768.0f - 1.0f) * 0.5f);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

bool kmajor_map(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t k, uint32_t box_rows) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return false;
    fn = reinterpret_cast<EncodeTiledFn>(f);
  }
  cuuint64_t gdim[2] = {k, rows}, gstride[1] = {k * 2};
  cuuint32_t box[2] = {BK, box_rows}, estr[2] = {1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

#define CHECK(x)                                                                                 \
  do {                                                                                           \
    cudaError_t e_ = (x);                                                                        \
    if (e_ != cudaSuccess) {                                                                     \
      fprintf(stderr, "%s:%d: %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));                \
      exit(1);                                                                                   \
    }                                                                                            \
  } while (0)

template <int BN, int NWG, int CN>
void run(const __half* A, const __half* W, float* sink, int M, int N, int K, int iters) {
  constexpr int kSmem = kStages * (BM + BN) * BK * 2 + 1024 + 2 * kStages * 8;
  auto kern = mainloop_kernel<BN, NWG, CN>;
  CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  CUtensorMap ta, tb;
  if (!kmajor_map(&ta, A, M, K, BM / CN) || !kmajor_map(&tb, W, N, K, BN)) {
    fprintf(stderr, "tensor map encode failed\n");
    exit(1);
  }
  int sms = 0;
  CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(128 * (NWG + 1));
  cfg.dynamicSmemBytes = kSmem;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = CN;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  int workers = sms;
  if (CN > 1) {
    cfg.gridDim = dim3(CN * sms);
    CHECK(cudaOccupancyMaxActiveClusters(&workers, kern, &cfg));
  }
  const int tiles = ((M + BM - 1) / BM) * ((N + BN * CN - 1) / (BN * CN));
  cfg.gridDim = dim3(CN * (tiles < workers ? tiles : workers));
  for (int i = 0; i < 5; ++i) CHECK(cudaLaunchKernelEx(&cfg, kern, ta, tb, M, N, K, 0, sink));
  CHECK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1;
  CHECK(cudaEventCreate(&e0));
  CHECK(cudaEventCreate(&e1));
  CHECK(cudaEventRecord(e0));
  for (int i = 0; i < iters; ++i) CHECK(cudaLaunchKernelEx(&cfg, kern, ta, tb, M, N, K, 0, sink));
  CHECK(cudaEventRecord(e1));
  CHECK(cudaEventSynchronize(e1));
  float ms = 0.f;
  CHECK(cudaEventElapsedTime(&ms, e0, e1));
  ms /= iters;
  printf("tile 128x%d  mma_warpgroups %d  cluster 1x%d  workers %3d  smem %6d B  %7.4f ms  %6.1f TFLOP/s\n", BN, NWG, CN,
         workers, kSmem, ms, 2.0 * M * N * K / ms / 1e9);
  CHECK(cudaEventDestroy(e0));
  CHECK(cudaEventDestroy(e1));
}

}  // namespace

int main(int argc, char** argv) {
  const int M = argc > 1 ? atoi(argv[1]) : 131072;
  const int N = argc > 2 ? atoi(argv[2]) : 2304;
  const int K = argc > 3 ? atoi(argv[3]) : 768;
  const int iters = argc > 4 ? atoi(argv[4]) : 50;
  __half *A, *W;
  float* sink;
  CHECK(cudaMalloc(&A, static_cast<size_t>(M) * K * 2));
  CHECK(cudaMalloc(&W, static_cast<size_t>(N) * K * 2));
  CHECK(cudaMalloc(&sink, 1024 * sizeof(float)));
  fill_f16<<<1024, 256>>>(A, static_cast<size_t>(M) * K, 1u);
  fill_f16<<<1024, 256>>>(W, static_cast<size_t>(N) * K, 2u);
  CHECK(cudaDeviceSynchronize());
  printf("M %d  N %d  K %d  iters %d\n", M, N, K, iters);
  // two rounds, alternating the configurations, so that clock drift shows up as a difference between rounds
  for (int round = 0; round < 2; ++round) {
    run<128, 1, 1>(A, W, sink, M, N, K, iters);
    run<128, 1, 2>(A, W, sink, M, N, K, iters);
    run<192, 2, 1>(A, W, sink, M, N, K, iters);
    run<192, 2, 2>(A, W, sink, M, N, K, iters);
    run<256, 2, 1>(A, W, sink, M, N, K, iters);
  }
  CHECK(cudaFree(A));
  CHECK(cudaFree(W));
  CHECK(cudaFree(sink));
  return 0;
}
