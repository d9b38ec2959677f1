// Persistent, warp-specialised wgmma GEMM for sm_90a (Hopper) with fused epilogues.
//
//   C[M,N] = A[M,K] (fp16, K-major)  x  W[N,K]^T (fp16, K-major == nn.Linear layout), fp32 accumulate.
//
// Replaces the dense f32 `gemm`+rayon matmuls behind candle's Linear on the reference's hot loop
// (candle-binding/src/model_architectures/traditional/candle_models/modernbert.rs
//  :123 Wqkv, :196 Wo, :236-238 Wi/GeGLU/Wo) with one kernel family on 128 x 128 tiles:
//   * warp 8      : TMA producer  (cp.async.bulk.tensor 2D, 128B swizzle, mbarrier complete_tx)
//   * warps 4..7  : one MMA warpgroup -- wgmma.mma_async m64n128k16 twice per k-step (rows 0-63, 64-127), fp32
//                   accumulators in registers; at the end of a tile they go to a swizzled fp32 tile in shared memory
//   * warps 0..3  : epilogue (shared fp32 tile -> registers, one row per lane -> fused math -> swizzled box -> TMA store)
//   * the accumulator tile in shared memory is the hand-off: the epilogue of tile i overlaps the mainloop of tile i+1,
//     whose accumulators live in the MMA warpgroup's registers until the epilogue has released the shared tile.
// Fused epilogues: bias, RoPE (rotate-half, modernbert.rs:61-85), fp32 residual add (:300-303),
// GeGLU = gelu_erf(a)*b (:238), erf-GELU (BERT intermediate).
#include "gemm.h"

#include <cstdlib>
#include <mutex>

#include "common.cuh"
#include "kernels.h"

namespace srb {

namespace {

constexpr int BM = 128;
constexpr int BN = 128;
constexpr int BK = 64;  // 64 fp16 = 128 B = one swizzle-128B row
constexpr int kEpiWarps = 4;       // one per 32-row quarter of the tile
constexpr int kMmaWarp0 = 4;       // warps 4..7: the MMA warpgroup (warpgroup-aligned)
constexpr int kProducerWarp = 8;
constexpr int kGemmThreads = 32 * (kProducerWarp + 1);
constexpr int kStageBufBytes = 4096;   // one epilogue staging box: 32 rows x 128 B
constexpr int kBarrierBytes = 512;
constexpr int kSmemLimit = 232448;     // 227 KB opt-in limit per CTA (sm_90)
constexpr int kAccBytes = BM * BN * 4; // fp32 accumulator tile handed from the MMA warpgroup to the epilogue
// staging boxes per epilogue warp.  The fp32-residual epilogue keeps one residual load in flight next to the box being
// computed; the fp16-pair residual epilogue keeps two (hi, lo) box pairs (one loading while the other computes).
// Shared memory is what limits this on sm_90: the 64 KB accumulator tile plus these boxes leave 3-4 mainloop stages.
__host__ __device__ constexpr int stage_bufs(int epi) { return epi == EPI_RESID_HL ? 4 : 2; }

template <int EPI>
struct GemmCfg {
  static constexpr int kBufs = stage_bufs(EPI);
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRawBufs = EPI == EPI_RESID ? 2 : 0;   // fp16 copy of the residual stream (LayerNorm fold)
  static constexpr int kEpiBytes = kEpiWarps * (kBufs + kRawBufs) * kStageBufBytes;
  static constexpr int kFit = (kSmemLimit - kAccBytes - kEpiBytes - 1024 /*align slack*/ - kBarrierBytes) / kStageBytes;
  static constexpr int kStages = kFit < 6 ? kFit : 6;   // as deep as shared memory allows, 6 at most
  static constexpr int kSmemBytes = kStages * kStageBytes + kAccBytes + kEpiBytes + 1024 + kBarrierBytes;
  static_assert(kStages >= 3, "mainloop ring too shallow");
};

struct KArgs {
  int M, N, K;
  const float* bias;
  int has_resid;
  const int* pos;
  const float* rope_cos;
  const float* rope_sin;
  int rope_cols;
  float* row_stats;          // EPI_RESID: accumulate (sum, sumsq) per row
  int has_raw16;             // EPI_RESID: tmap_aux is the fp16 copy of the output
  const float* fold_stats;   // EPI_ROPE / EPI_GEGLU: per-row (sum, sumsq) of the A rows (null: no fold)
  float fold_eps;
  float fold_inv_h;
  int fold_parts;            // 128-column slices the row statistics come in
  float* pivot_out;          // EPI_RESID: row pivots (see gemm.h)
  const float* pivot_in;
  const float* pivot_in_stats;
  int* topk_idx;             // EPI_TOPK
  float* topk_score;
  const uint8_t* topk_valid;
  int topk_n;
  int grouped;               // EPI_TOPK: grouped tile schedule (see the kernel)
  int interleave;            // tiles w, w + W, ... per worker instead of a contiguous range
  int K2;                    // K extension: k-blocks beyond K come from (tmap_a2, tmap_b2) -- low-rank adapters (gemm.h)
  int mask_block, mask_rows; // EPI_F16: keep column c of row r only when c / mask_block == r / mask_rows (0: off)
  int grp_rows;              // > 0: W is a stack of [N, K] matrices, rows [g * grp_rows, (g + 1) * grp_rows) of A multiply matrix g
};
constexpr int kTopK = 8;

// ---- wgmma (sm_90a) ---------------------------------------------------------------------------------
// K-major, 128B-swizzled operand descriptor (rows x 64 fp16; 8-row groups 1024 B apart):
//   start address >> 4 [0,14) | LBO (unused for swizzled K-major, 1) [16,30) | SBO = 1024 B >> 4 [32,46)
//   | layout = SWIZZLE_128B (1) [62,64)
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
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both operands K-major in shared memory.  Fragment of D: warp w of the
// warpgroup holds rows 16w + lane/4 (d[4j], d[4j+1]) and 16w + 8 + lane/4 (d[4j+2], d[4j+3]) at columns 8j + 2(lane%4) + {0,1}.
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
// Byte offset of fp32 column `col` of row `row` in the shared accumulator tile: [BM][BN] fp32 rows, 16-byte units
// XOR-swizzled by (row & 7) inside each 128-byte group, so that a warp reading one row per lane (8 units each) and the
// MMA warpgroup writing its fragments both stay at the minimum number of shared-memory wavefronts.
__device__ __forceinline__ uint32_t acc_off(int row, int col) {
  const int u = col >> 2;
  return static_cast<uint32_t>(row * (BN * 4) + (((u & ~7) | ((u & 7) ^ (row & 7))) << 4) + (col & 3) * 4);
}

// LayerNorm fold, consumer side.  W'' = (W diag(gamma)) with every row re-centred to sum zero, so that
// sum_k x[r,k] W''[n,k] = sum_k (x[r,k] - mean_r) W'[n,k]: the mean subtraction of the LayerNorm happens inside the GEMM
// (the centring matrix I - 11^T/H commutes into the weights) and the epilogue is left with the per-row rstd factor --
// which the RoPE epilogue folds into the row's cos / sin registers (the rotation is linear), so q and k cost nothing.
__device__ __forceinline__ void fold_scale(float rstd, uint32_t* a, uint32_t* b) {
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    a[i] = __float_as_uint(__uint_as_float(a[i]) * rstd);
    b[i] = __float_as_uint(__uint_as_float(b[i]) * rstd);
  }
}

template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_aux,
            const __grid_constant__ CUtensorMap tmap_a2, const __grid_constant__ CUtensorMap tmap_b2, const KArgs p) {
  using Cfg = GemmCfg<EPI>;
  static_assert(Cfg::kSmemBytes <= kSmemLimit, "over the 227 KB shared-memory opt-in limit");
  constexpr bool kHL = EPI == EPI_RESID_HL;
  constexpr int kStageBufs = Cfg::kBufs;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;
  uint8_t* smem_acc = smem + Cfg::kStages * Cfg::kStageBytes;
  uint8_t* smem_epi = smem_acc + kAccBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_epi + Cfg::kEpiBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + Cfg::kStages;
  uint64_t* tfull_bar = bars + 2 * Cfg::kStages;   // accumulator tile written (MMA warpgroup -> epilogue)
  uint64_t* tempty_bar = tfull_bar + 1;            // accumulator tile read out (epilogue -> MMA warpgroup)
  uint64_t* resid_bar = tempty_bar + 1;            // [kEpiWarps][kStageBufs]
  static_assert((2 * Cfg::kStages + 2 + kEpiWarps * kStageBufs) * 8 <= kBarrierBytes, "barrier block too small");

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_blocks = (p.M + BM - 1) / BM;
  const int n_blocks = (p.N + BN - 1) / BN;
  const int k1_blocks = (p.K + BK - 1) / BK;
  // K extension: the accumulator also takes A2[M, K2] x W2[N, K2]^T -- same stages, same MMAs, other tensor maps
  const int k_blocks = k1_blocks + (p.K2 + BK - 1) / BK;
  const int num_tiles = m_blocks * n_blocks;
  auto row_base = [&](int m_blk) { return m_blk * BM; };
  // contiguous tile range per CTA (n fastest): one CTA walks all N tiles of an M block back to back, so the
  // A row-block stays hot in L2 and per-row epilogue state (RoPE cos/sin) is reused across tiles
  const int num_workers = gridDim.x;
  const int base = num_tiles / num_workers, rem = num_tiles % num_workers;
  const int bid = blockIdx.x;
  int t_begin = bid * base + (bid < rem ? bid : rem);
  int t_end = t_begin + base + (bid < rem ? 1 : 0);
  // EPI_TOPK, grouped schedule (p.grouped): worker w owns query block w % m_blocks for its whole life (its running
  // top-8 lists live in registers) and walks the stored-row tiles g, g + G, g + 2G, ... with g = w / m_blocks,
  // G = workers / m_blocks.  The m_blocks workers of a group therefore ask for the SAME stored-row tile at about the
  // same time: one HBM read, the rest L2 hits -- the store streams once per batch instead of once per query block.
  // Tiles are numbered t = m_blk * n_blocks + n_blk as everywhere else; `t_step` is the distance between two tiles of
  // this worker (1 for the contiguous ranges).
  int t_step = 1;
  // Interleaved schedule (p.interleave; the residual GEMMs): worker w takes tiles w, w + W, w + 2W, ...  With
  // n fastest in the tile numbering the N / BN tiles of one row block run AT THE SAME TIME on neighbouring workers, so
  // each A k-block is pulled from HBM once and hit in L2 by the others, where the contiguous ranges could lose the row
  // block from L2 to the residual stream passing through between two tiles of one worker.
  if (p.interleave) {
    t_begin = bid;
    t_end = num_tiles;
    t_step = num_workers;
  }
  if constexpr (EPI == EPI_TOPK) {
    if (p.grouped) {
      const int groups = num_workers / m_blocks;
      const int m_own = bid % m_blocks, g_own = bid / m_blocks;
      t_begin = m_own * n_blocks + g_own;
      t_end = (m_own + 1) * n_blocks;
      t_step = groups;
      if (g_own >= groups) t_end = t_begin;   // workers beyond the last full group stay idle
    }
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    tma_prefetch_desc(&tmap_out);
#pragma unroll
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);        // one arrival per MMA warp
    }
    mbar_init(tfull_bar, 128);            // every thread of the MMA warpgroup, after its fragment stores
    mbar_init(tempty_bar, kEpiWarps);
    for (int i = 0; i < kEpiWarps * kStageBufs; ++i) mbar_init(&resid_bar[i], 1);
    mbar_fence_init();
  }
  __syncthreads();
  // PDL: everything above overlapped the previous kernel's tail; nothing below may start before its writes are visible
  griddep_launch_dependents();
  griddep_wait();

  if (warp == kProducerWarp) {
    // ================= TMA producer =================
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int t = t_begin; t < t_end; t += t_step) {
        const int m_blk = t / n_blocks, n_blk = t % n_blocks;
        // grouped weights (one matrix per task, stacked along N): the row block picks its matrix; blocks never straddle
        // two groups (grp_rows is a multiple of the block height, checked on the host)
        const int w_row0 = p.grp_rows > 0 ? ((m_blk * BM) / p.grp_rows) * p.N : 0;
        for (int kb = 0; kb < k_blocks; ++kb) {
          mbar_wait(&empty_bar[s], ph ^ 1);
          const bool ext = kb >= k1_blocks;
          const CUtensorMap* ma = ext ? &tmap_a2 : &tmap_a;
          const CUtensorMap* mb = ext ? &tmap_b2 : &tmap_b;
          const int kc = (ext ? kb - k1_blocks : kb) * BK;
          mbar_expect_tx(&full_bar[s], Cfg::kStageBytes);
          tma_load_2d(smem_a + s * Cfg::kABytes, ma, &full_bar[s], kc, m_blk * BM);
          tma_load_2d(smem_b + s * Cfg::kBBytes, mb, &full_bar[s], kc, (ext ? 0 : w_row0) + n_blk * BN);
          if (++s == Cfg::kStages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else if (warp >= kMmaWarp0) {
    // ================= MMA warpgroup =================
    const int wq = warp - kMmaWarp0;   // warp of the warpgroup: fragment rows 16 wq .. 16 wq + 15 of each 64-row half
    float acc[2][64];
    int s = 0;
    uint32_t ph = 0;
    uint32_t eph = 0;   // tempty phase
    for (int t = t_begin; t < t_end; t += t_step) {
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[s], ph);
        wgmma_fence();
        const uint32_t a0 = smem_u32(smem_a + s * Cfg::kABytes);
        const uint32_t b0 = smem_u32(smem_b + s * Cfg::kBBytes);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          // advance 16 fp16 = 32 B along K inside the swizzle atom; rows 64..127 of A start 64 x 128 B further
          const uint64_t db = gmma_desc_sw128(b0 + 32 * k);
          const uint32_t accum = (kb > 0 || k > 0) ? 1u : 0u;
          wgmma_m64n128k16(acc[0], gmma_desc_sw128(a0 + 32 * k), db, accum);
          wgmma_m64n128k16(acc[1], gmma_desc_sw128(a0 + 64 * 128 + 32 * k), db, accum);
        }
        wgmma_commit();
        // the previous stage's MMAs have completed once at most this stage's group is pending: free that stage
        wgmma_wait<1>();
        __syncwarp();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == Cfg::kStages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      // hand the tile to the epilogue once it has read out the previous one
      mbar_wait(tempty_bar, eph ^ 1);
      eph ^= 1;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = 64 * h + 16 * wq + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = 8 * j + 2 * (lane & 3);
          *reinterpret_cast<float2*>(smem_acc + acc_off(r, col)) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
          *reinterpret_cast<float2*>(smem_acc + acc_off(r + 8, col)) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
        }
      }
      mbar_arrive(tfull_bar);
    }
  } else {
    // ================= epilogue warps: shared fp32 tile -> registers -> swizzled smem box -> TMA store =================
    const int quad = warp;  // 32-row quarter of the tile this warp owns (one row per lane)
    uint8_t* my_bufs = smem_epi + warp * ((kStageBufs + Cfg::kRawBufs) * kStageBufBytes);
    uint8_t* my_raw = my_bufs + kStageBufs * kStageBufBytes;   // [kRawBufs] fp16 boxes (32 rows x 64 columns)
    const bool want_raw = (EPI == EPI_RESID) && p.has_raw16;
    const bool want_stats = (EPI == EPI_RESID || kHL) && p.row_stats != nullptr;
    const bool fold = (EPI == EPI_ROPE || EPI == EPI_GEGLU) && p.fold_stats != nullptr;
    float f_rstd = 1.f;   // fold: rstd of this thread's row
    float pv = 0.f;       // fold producer: this thread's row pivot (EPI_RESID_HL: the pivot SHIFT of this GEMM)
    float pv_prev = 0.f;  // EPI_RESID_HL: the pivot the stored pair is relative to
    int pv_mblk = -1;
    int fold_mblk = -1;
    uint64_t* my_rbar = resid_bar + warp * kStageBufs;
    uint32_t aph = 0;
    int cb = 0;                 // staging buffer to use next
    uint32_t rph = 0;           // phase bit per staging buffer (residual loads)
    const uint8_t* acc_row = smem_acc + (quad * 32 + lane) * (BN * 4);
    // this thread's row, accumulator columns [col, col + 32) (col a multiple of 32)
    auto acc_ld32 = [&](int col, uint32_t* r) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint4 v = *reinterpret_cast<const uint4*>(acc_row + ((((col >> 2) + (i ^ (lane & 7)))) << 4));
        r[4 * i] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
      }
    };
    // chunk geometry: a chunk is one 32-row x 128-byte output box of this warp
    constexpr int kAccPerChunk = (EPI == EPI_RESID || EPI == EPI_TOPK) ? 32 : (EPI == EPI_GEGLU ? 128 : 64);  // accumulator columns
    constexpr int kOutPerChunk = (EPI == EPI_RESID || EPI == EPI_TOPK) ? 32 : 64;                                // output columns
    constexpr int kChunks = BN / kAccPerChunk;
    constexpr int kPairs = kStageBufs / 2;   // EPI_RESID_HL: (hi, lo) box pairs of this warp
    const int n_out = (EPI == EPI_GEGLU) ? p.N / 2 : p.N;
    const bool use_resid = (EPI == EPI_RESID) && p.has_resid;

    // EPI_RESID: residual boxes are TMA-loaded one chunk ahead (flat over (tile, chunk) of this CTA)
    auto out_col = [&](int t, int c) { return (t % n_blocks) * (BN / kAccPerChunk * kOutPerChunk) + c * kOutPerChunk; };
    auto chunk_valid = [&](int t, int c) { return t < t_end && out_col(t, c) < n_out; };
    auto issue_resid = [&](int t, int c, int buf) {  // lane 0 only
      if constexpr (kHL) {   // buf = pair index: hi box, then lo box, one barrier for both
        uint8_t* pb = my_bufs + buf * 2 * kStageBufBytes;
        mbar_expect_tx(&my_rbar[buf], 2 * kStageBufBytes);
        tma_load_2d(pb, &tmap_out, &my_rbar[buf], out_col(t, c), row_base(t / n_blocks) + quad * 32);
        tma_load_2d(pb + kStageBufBytes, &tmap_aux, &my_rbar[buf], out_col(t, c), row_base(t / n_blocks) + quad * 32);
      } else {
        mbar_expect_tx(&my_rbar[buf], kStageBufBytes);
        tma_load_2d(my_bufs + buf * kStageBufBytes, &tmap_out, &my_rbar[buf], out_col(t, c),
                    row_base(t / n_blocks) + quad * 32);
      }
    };
    // residual prefetch cursor: runs kAhead chunks in front of the chunk being processed (flat over this CTA's
    // (tile, chunk) sequence)
    constexpr int kRing = kHL ? kPairs : kStageBufs;   // residual-load ring: boxes, or box pairs
    constexpr int kAhead = kHL ? 1 : (kStageBufs - 2 > 0 ? kStageBufs - 2 : 1);
    int pf_t = t_begin, pf_c = 0, pf_buf = 0;
    auto pf_issue = [&]() {  // lane 0 only
      if (!chunk_valid(pf_t, pf_c)) return;
      issue_resid(pf_t, pf_c, pf_buf);
      if (++pf_buf == kRing) pf_buf = 0;
      if (++pf_c >= kChunks || !chunk_valid(pf_t, pf_c)) { pf_t += t_step; pf_c = 0; }
    };
    if ((use_resid || kHL) && lane == 0) {
#pragma unroll
      for (int i = 0; i < kAhead; ++i) pf_issue();
    }

    // EPI_ROPE: this thread's cos/sin row, reloaded only when the M block changes
    float cs[EPI == EPI_ROPE ? 32 : 1], sn[EPI == EPI_ROPE ? 32 : 1];
    int rope_mblk = -1;

    // EPI_TOPK: this thread's running top-8 (descending) over the columns this CTA walks for its current row
    float tk_v[EPI == EPI_TOPK ? kTopK : 1];
    int tk_i[EPI == EPI_TOPK ? kTopK : 1];
    int tk_mblk = -1;
    auto tk_reset = [&]() {
#pragma unroll
      for (int i = 0; i < (EPI == EPI_TOPK ? kTopK : 1); ++i) { tk_v[i] = -INFINITY; tk_i[i] = -1; }
    };
    auto tk_flush = [&](int m_blk_done) {   // this CTA's list for the row it has just left
      const int row = row_base(m_blk_done) + quad * 32 + lane;
      if (row < p.M) {
        const size_t at = (static_cast<size_t>(row) * gridDim.x + bid) * kTopK;
#pragma unroll
        for (int i = 0; i < (EPI == EPI_TOPK ? kTopK : 1); ++i) { p.topk_idx[at + i] = tk_i[i]; p.topk_score[at + i] = tk_v[i]; }
      }
    };
    for (int t = t_begin; t < t_end; t += t_step) {
      const int m_blk = t / n_blocks, n_blk = t % n_blocks;
      const int row0 = row_base(m_blk) + quad * 32;
      if constexpr (EPI == EPI_TOPK) {
        if (m_blk != tk_mblk) {
          if (tk_mblk >= 0) tk_flush(tk_mblk);
          tk_reset();
          tk_mblk = m_blk;
        }
      }
      if constexpr (EPI == EPI_ROPE || EPI == EPI_GEGLU) {
        if (fold && m_blk != fold_mblk) {
          const int row = row0 + lane < p.M ? row0 + lane : p.M - 1;
          float s1 = 0.f, s2 = 0.f;
          for (int k = 0; k < p.fold_parts; ++k) {   // fixed slice order: reproducible
            const float2 st = __ldg(reinterpret_cast<const float2*>(p.fold_stats) + static_cast<size_t>(k) * p.M + row);
            s1 += st.x;
            s2 += st.y;
          }
          const float mean = s1 * p.fold_inv_h;
          const float var = fmaxf(s2 * p.fold_inv_h - mean * mean, 0.f);
          f_rstd = rsqrtf(var + p.fold_eps);
          fold_mblk = m_blk;
          rope_mblk = -1;   // the row's cos / sin registers carry rstd: reload them for this M block
        }
      }
      if constexpr (EPI == EPI_ROPE) {
        if (m_blk != rope_mblk && n_blk * BN < p.rope_cols) {
          const int row = row0 + lane;
          const int pos = __ldg(p.pos + (row < p.M ? row : p.M - 1));   // rows past M: any valid table row (never stored)
          const float4* c4 = reinterpret_cast<const float4*>(p.rope_cos + static_cast<size_t>(pos) * 32);
          const float4* s4 = reinterpret_cast<const float4*>(p.rope_sin + static_cast<size_t>(pos) * 32);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 a = __ldg(c4 + i), b = __ldg(s4 + i);
            cs[4 * i] = a.x; cs[4 * i + 1] = a.y; cs[4 * i + 2] = a.z; cs[4 * i + 3] = a.w;
            sn[4 * i] = b.x; sn[4 * i + 1] = b.y; sn[4 * i + 2] = b.z; sn[4 * i + 3] = b.w;
          }
          if (fold) {   // LayerNorm fold: the rstd factor of the row rides on the (linear) rotation
#pragma unroll
            for (int i = 0; i < 32; ++i) { cs[i] *= f_rstd; sn[i] *= f_rstd; }
          }
          rope_mblk = m_blk;
        }
      }
      float st1 = 0.f, st2 = 0.f;   // EPI_RESID: this row's (sum, sum of squares) over the current 128-column slice
      if constexpr (kHL) {
        // pivot shift of this row: the stored pair is x - pivot_in; the new pivot is pivot_in + (mean of x - pivot_in),
        // read from the previous residual GEMM's statistics (0 for the first one: the embedding's pair is x itself)
        if (m_blk != pv_mblk) {
          pv = 0.f;
          pv_prev = 0.f;
          if (p.pivot_in_stats) {
            const int row = row0 + lane < p.M ? row0 + lane : p.M - 1;
            float s1 = 0.f;
            const int parts = p.N >> 7;
            for (int k = 0; k < parts; ++k)
              s1 += __ldg(reinterpret_cast<const float2*>(p.pivot_in_stats) + static_cast<size_t>(k) * p.M + row).x;
            pv = s1 / static_cast<float>(p.N);
            pv_prev = __ldg(p.pivot_in + row);
          }
          pv_mblk = m_blk;
        }
      }
      if constexpr (EPI == EPI_RESID) {
        if (want_stats && m_blk != pv_mblk) {   // the row's pivot: its mean after the previous residual GEMM
          pv = 0.f;
          if (p.pivot_in_stats) {
            const int row = row0 + lane < p.M ? row0 + lane : p.M - 1;
            float s1 = 0.f;
            const int parts = p.N >> 7;
            for (int k = 0; k < parts; ++k)
              s1 += __ldg(reinterpret_cast<const float2*>(p.pivot_in_stats) + static_cast<size_t>(k) * p.M + row).x;
            pv = __ldg(p.pivot_in + row) + s1 / static_cast<float>(p.N);
          }
          pv_mblk = m_blk;
        }
      }
      mbar_wait(tfull_bar, aph);
      aph ^= 1;

      if constexpr (EPI == EPI_TOPK) {
        // This warp scans the tile's columns 32 at a time.  The common path per chunk is the maximum of 32 scores and
        // one compare against the list's tail; validity (invalidated rows, padding rows >= topk_n) is only looked up
        // for a score that would enter the list -- after the first tiles that is rare.
        auto topk_chunk = [&](uint32_t* r, int ocol0) {
          float m0 = -INFINITY, m1 = -INFINITY, m2 = -INFINITY, m3 = -INFINITY;
#pragma unroll
          for (int i = 0; i < 32; i += 8) {
            m0 = fmax3(m0, __uint_as_float(r[i]), __uint_as_float(r[i + 1]));
            m1 = fmax3(m1, __uint_as_float(r[i + 2]), __uint_as_float(r[i + 3]));
            m2 = fmax3(m2, __uint_as_float(r[i + 4]), __uint_as_float(r[i + 5]));
            m3 = fmax3(m3, __uint_as_float(r[i + 6]), __uint_as_float(r[i + 7]));
          }
          // Take the chunk's maximum while it beats the list's tail (usually zero or one round): a round is ~150
          // instructions, against ~1300 for trying all 32 scores in turn.
          float cm = fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
          while (cm > tk_v[kTopK - 1]) {   // strict: an equal score at a higher column never displaces
            int ci = 31;
#pragma unroll
            for (int i = 30; i >= 0; --i)
              if (__uint_as_float(r[i]) == cm) ci = i;          // lowest column holding the maximum
            ci = __uint_as_float(r[31]) == cm && ci == 31 ? 31 : ci;
            float cv = cm;
            int cidx = ocol0 + ci;
            const bool ok = cidx < p.topk_n && (!p.topk_valid || __ldg(p.topk_valid + (cidx < p.topk_n ? cidx : 0)));
            if (ok) {
#pragma unroll
              for (int j = 0; j < kTopK; ++j) {   // insertion into the descending list
                if (cv > tk_v[j]) {
                  const float tv = tk_v[j]; const int ti = tk_i[j];
                  tk_v[j] = cv; tk_i[j] = cidx;
                  cv = tv; cidx = ti;
                }
              }
            }
            float n0 = -INFINITY, n1 = -INFINITY;
#pragma unroll
            for (int i = 0; i < 32; i += 2) {   // drop it and find the next maximum
              if (i == ci) r[i] = 0xff800000u;
              if (i + 1 == ci) r[i + 1] = 0xff800000u;
              n0 = fmaxf(n0, __uint_as_float(r[i]));
              n1 = fmaxf(n1, __uint_as_float(r[i + 1]));
            }
            cm = fmaxf(n0, n1);
          }
        };
#pragma unroll 1
        for (int c = 0; c < kChunks; ++c) {
          uint32_t r[32];
          acc_ld32(c * 32, r);
          topk_chunk(r, out_col(t, c));
        }
      }
      if constexpr (kHL) {
        // 64-column chunks: the (hi, lo) boxes of the chunk arrive by TMA one chunk ahead, are updated in place in
        // shared memory and leave by TMA; statistics per 128-column slice as in EPI_RESID
#pragma unroll 1
        for (int c = 0; c < kChunks; ++c) {
          const int ocol0 = out_col(t, c);
          if (ocol0 >= n_out) break;
          uint8_t* hb = my_bufs + cb * 2 * kStageBufBytes;
          uint8_t* lb = hb + kStageBufBytes;
          if (lane == 0) {
            // the pair the prefetch cursor points at was stored kPairs - 1 chunks ago: all but the newest store group read out
            bulk_wait_read<kPairs - kAhead - 1>();
            pf_issue();
          }
          mbar_wait(&my_rbar[cb], (rph >> cb) & 1u);
          rph ^= 1u << cb;
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            uint32_t r[32];
            acc_ld32(c * 64 + hf * 32, r);
#pragma unroll
            for (int u = 0; u < 4; ++u) {   // 16-byte units: 8 columns each
              const uint32_t off = box_off(lane, hf * 4 + u);
              uint4 hv = *reinterpret_cast<const uint4*>(hb + off);
              uint4 lv = *reinterpret_cast<const uint4*>(lb + off);
              uint32_t hw[4] = {hv.x, hv.y, hv.z, hv.w}, lw[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&hw[k]));
                const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&lw[k]));
                float x0 = (fh.x + fl.x) + (__uint_as_float(r[8 * u + 2 * k]) - pv);
                float x1 = (fh.y + fl.y) + (__uint_as_float(r[8 * u + 2 * k + 1]) - pv);
                if (p.bias) {
                  const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + ocol0 + hf * 32 + 8 * u) + k);
                  x0 += b.x; x1 += b.y;
                }
                st1 += x0 + x1;
                st2 += x0 * x0 + x1 * x1;
                const __half2 nh = __floats2half2_rn(x0, x1);
                const float2 fb = __half22float2(nh);
                hw[k] = *reinterpret_cast<const uint32_t*>(&nh);
                lw[k] = pack_half2(x0 - fb.x, x1 - fb.y);
              }
              sts16(hb + off, hw[0], hw[1], hw[2], hw[3]);
              sts16(lb + off, lw[0], lw[1], lw[2], lw[3]);
            }
          }
          if (c & 1) {   // a 128-column slice is complete: its partial goes out, once
            if (row0 + lane < p.M) {
              const size_t part = static_cast<size_t>((ocol0 - 64) >> 7);
              *reinterpret_cast<float2*>(p.row_stats + 2 * (part * p.M + row0 + lane)) = make_float2(st1, st2);
              if (part == 0) p.pivot_out[row0 + lane] = pv_prev + pv;
            }
            st1 = 0.f;
            st2 = 0.f;
          }
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            tma_store_2d(&tmap_out, hb, ocol0, row0);
            tma_store_2d(&tmap_aux, lb, ocol0, row0);
            bulk_commit();
          }
          if (++cb == kPairs) cb = 0;
        }
      }
#pragma unroll 1
      for (int c = 0; c < ((EPI == EPI_TOPK || kHL) ? 0 : kChunks); ++c) {
        const int ocol0 = out_col(t, c);
        if (ocol0 >= n_out) break;
        uint8_t* buf = my_bufs + cb * kStageBufBytes;
        uint8_t* my_row = buf;  // + box_off(lane, chunk16)
        if (use_resid) {
          // the box the prefetch cursor points at was last used kStageBufs - kAhead chunks ago: its store must have
          // been read out (all but the newest kStageBufs - kAhead - 1 store groups complete)
          if (lane == 0) {
            bulk_wait_read<(kStageBufs - kAhead - 1 > 0 ? kStageBufs - kAhead - 1 : 0)>();
            pf_issue();
          }
          mbar_wait(&my_rbar[cb], (rph >> cb) & 1u);
          rph ^= 1u << cb;
        } else {
          if (lane == 0) bulk_wait_read<kStageBufs - 1>();  // this buffer's previous store has been read out
          __syncwarp();
        }

        if constexpr (EPI == EPI_RESID) {
          uint32_t r[32];
          acc_ld32(c * 32, r);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float4* q = reinterpret_cast<float4*>(my_row + box_off(lane, i));
            float4 x = use_resid ? *q : make_float4(0.f, 0.f, 0.f, 0.f);
            x.x += __uint_as_float(r[4 * i]);
            x.y += __uint_as_float(r[4 * i + 1]);
            x.z += __uint_as_float(r[4 * i + 2]);
            x.w += __uint_as_float(r[4 * i + 3]);
            if (p.bias) {
              const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + ocol0) + i);
              x.x += b.x; x.y += b.y; x.z += b.z; x.w += b.w;
            }
            *q = x;
            x.x -= pv; x.y -= pv; x.z -= pv; x.w -= pv;   // statistics and the fp16 copy are taken of x - pivot
            st1 += (x.x + x.y) + (x.z + x.w);
            st2 += (x.x * x.x + x.y * x.y) + (x.z * x.z + x.w * x.w);
            if (want_raw) {   // fp16 copy: chunk c fills 16-byte units (c & 1) * 4 + i / 2 of the 64-column box
              r[2 * i] = pack_half2(x.x, x.y);
              r[2 * i + 1] = pack_half2(x.z, x.w);
            }
          }
          if (want_stats && (c & 3) == 3) {   // a 128-column slice is complete: its partial goes out, once
            if (row0 + lane < p.M) {
              const size_t part = static_cast<size_t>((ocol0 - 96) >> 7);
              *reinterpret_cast<float2*>(p.row_stats + 2 * (part * p.M + row0 + lane)) = make_float2(st1, st2);
              if (part == 0 && p.pivot_out) p.pivot_out[row0 + lane] = pv;
            }
            st1 = 0.f;
            st2 = 0.f;
          }
          if (want_raw) {
            uint8_t* rb = my_raw + ((c >> 1) & 1) * kStageBufBytes;
#pragma unroll
            for (int i = 0; i < 4; ++i)
              sts16(rb + box_off(lane, (c & 1) * 4 + i), r[4 * i], r[4 * i + 1], r[4 * i + 2], r[4 * i + 3]);
          }
        } else if constexpr (EPI == EPI_F16 || EPI == EPI_GELU) {
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            uint32_t r[32];
            acc_ld32(c * 64 + hf * 32, r);
            uint32_t h[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              float v0 = __uint_as_float(r[2 * i]), v1 = __uint_as_float(r[2 * i + 1]);
              if (p.bias) {
                const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + ocol0 + hf * 32) + i);
                v0 += b.x; v1 += b.y;
              }
              if constexpr (EPI == EPI_GELU) { v0 = gelu_erf_fast_f(v0); v1 = gelu_erf_fast_f(v1); }
              if constexpr (EPI == EPI_F16) {
                if (p.mask_block > 0) {   // adapter projections: a row keeps the column block of its own task only
                  const int own = (row0 + lane) / p.mask_rows, col = ocol0 + hf * 32 + 2 * i;
                  if (col / p.mask_block != own) v0 = 0.f;
                  if ((col + 1) / p.mask_block != own) v1 = 0.f;
                }
              }
              h[i] = pack_half2(v0, v1);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
              sts16(my_row + box_off(lane, hf * 4 + i), h[4 * i], h[4 * i + 1], h[4 * i + 2], h[4 * i + 3]);
          }
        } else if constexpr (EPI == EPI_ROPE) {
          uint32_t r1[32], r2[32];
          acc_ld32(c * 64, r1);
          acc_ld32(c * 64 + 32, r2);
          if (fold && ocol0 >= p.rope_cols) fold_scale(f_rstd, r1, r2);   // v columns: no rotation to carry rstd
          if (ocol0 < p.rope_cols) {  // q and k heads: rotate-half over the 64-wide head (in place, packed)
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const float a0 = __uint_as_float(r1[2 * i]), a1 = __uint_as_float(r1[2 * i + 1]);
              const float b0 = __uint_as_float(r2[2 * i]), b1 = __uint_as_float(r2[2 * i + 1]);
              r1[i] = pack_half2(a0 * cs[2 * i] - b0 * sn[2 * i], a1 * cs[2 * i + 1] - b1 * sn[2 * i + 1]);
              r2[i] = pack_half2(a0 * sn[2 * i] + b0 * cs[2 * i], a1 * sn[2 * i + 1] + b1 * cs[2 * i + 1]);
            }
          } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              r1[i] = pack_half2(__uint_as_float(r1[2 * i]), __uint_as_float(r1[2 * i + 1]));
              r2[i] = pack_half2(__uint_as_float(r2[2 * i]), __uint_as_float(r2[2 * i + 1]));
            }
          }
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            sts16(my_row + box_off(lane, i), r1[4 * i], r1[4 * i + 1], r1[4 * i + 2], r1[4 * i + 3]);
            sts16(my_row + box_off(lane, 4 + i), r2[4 * i], r2[4 * i + 1], r2[4 * i + 2], r2[4 * i + 3]);
          }
        } else if constexpr (EPI == EPI_GEGLU) {
          // W rows are pre-interleaved in 32-row groups [a(32j..32j+31) | b(32j..32j+31)]: accumulator columns
          // [64j, 64j+32) hold `a`, [64j+32, 64j+64) the matching `b`; one output chunk = two such groups
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            uint32_t ra[32], rb[32];
            acc_ld32(c * 128 + hf * 64, ra);
            acc_ld32(c * 128 + hf * 64 + 32, rb);
            const float rs = fold ? f_rstd : 1.0f;
            const float kz = rs * 0.70710678118654752440f, kh = 0.5f * rs * rs;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const float g0 = geglu_fold_f(__uint_as_float(ra[2 * i]), __uint_as_float(rb[2 * i]), kz, kh);
              const float g1 = geglu_fold_f(__uint_as_float(ra[2 * i + 1]), __uint_as_float(rb[2 * i + 1]), kz, kh);
              ra[i] = pack_half2(g0, g1);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
              sts16(my_row + box_off(lane, hf * 4 + i), ra[4 * i], ra[4 * i + 1], ra[4 * i + 2], ra[4 * i + 3]);
          }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          tma_store_2d(&tmap_out, buf, ocol0, row0);  // rows >= M / cols >= N are clipped by the TMA unit
          if constexpr (EPI == EPI_RESID) {
            // the fp16 box completes every second chunk and rides in the same bulk group as that chunk's fp32 store
            // (its staging box is next written two chunks later, after the wait_group.read above)
            if (want_raw && (c & 1)) tma_store_2d(&tmap_aux, my_raw + ((c >> 1) & 1) * kStageBufBytes, ocol0 - 32, row0);
          }
          bulk_commit();
        }
        if (++cb == kStageBufs) cb = 0;
      }
      // release the accumulator tile back to the MMA warpgroup
      __syncwarp();
      if (lane == 0) mbar_arrive(tempty_bar);
    }
    if constexpr (EPI == EPI_TOPK) {
      if (tk_mblk >= 0) tk_flush(tk_mblk);
    }
    if (lane == 0) bulk_wait_read<0>();  // smem must outlive the last stores' reads
    __syncwarp();
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
  });
  return fn;
}

template <int EPI>
int launch(cudaStream_t stream, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
           const CUtensorMap& tx, const CUtensorMap& ta2, const CUtensorMap& tb2, const KArgs& ka, int num_sms,
           int grid_override = 0) {
  using Cfg = GemmCfg<EPI>;
  // per-device attribute; cheap enough to set on every launch (multi-GPU processes switch devices)
  SRB_CUDA_CHECK(cudaFuncSetAttribute(gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  const int m_blocks = (ka.M + BM - 1) / BM, n_blocks = (ka.N + BN - 1) / BN;
  const int tiles = m_blocks * n_blocks;
  const int grid = grid_override > 0 ? grid_override : (tiles < num_sms ? tiles : num_sms);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  SRB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, gemm_kernel<EPI>, ta, tb, tc, tx, ta2, tb2, ka));
  note_launch();
  return 0;
}

}  // namespace

static int make_tmap_2d(CUtensorMap* out, CUtensorMapDataType dt, int elem_bytes, const void* ptr, uint64_t cols,
                        uint64_t rows, uint64_t ld_elems, uint32_t box_cols, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    fprintf(stderr, "[srb200] cuTensorMapEncodeTiled entry point unavailable\n");
    return -1;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld_elems * elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, dt, 2, const_cast<void*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[srb200] cuTensorMapEncodeTiled failed: %d (cols=%llu rows=%llu ld=%llu box=%ux%u)\n", (int)r,
            (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)ld_elems, box_cols, box_rows);
    return -1;
  }
  return 0;
}

int make_tmap_2d_f16(CUtensorMap* out, const void* ptr, uint64_t cols, uint64_t rows, uint64_t ld_elems,
                     uint32_t box_cols, uint32_t box_rows) {
  return make_tmap_2d(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptr, cols, rows, ld_elems, box_cols, box_rows);
}

int make_tmap_f16_kmajor(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t k, uint32_t box_rows) {
  return make_tmap_2d(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, ptr, k, rows, k, BK, box_rows);
}

int gemm_f16(cudaStream_t stream, const GemmDesc& g) {
  if (g.M <= 0) return 0;
  if (g.K % 8 != 0 || g.N % 64 != 0 || g.ldo % 8 != 0) {
    fprintf(stderr, "[srb200] gemm_f16: unsupported shape M=%d N=%d K=%d ldo=%d\n", g.M, g.N, g.K, g.ldo);
    return -1;
  }
  if (g.epi == EPI_RESID && g.resid && (g.resid != g.out || g.ldr != g.ldo)) {
    fprintf(stderr, "[srb200] gemm_f16: EPI_RESID runs in place (resid must alias out) or without residual\n");
    return -1;
  }
  const bool is_hl = g.epi == EPI_RESID_HL;
  if (is_hl && (!g.lo16 || !g.row_stats || !g.pivot_out || g.N % 128 != 0 || g.ldo != g.N || g.raw16 || g.resid)) {
    fprintf(stderr, "[srb200] gemm_f16: EPI_RESID_HL needs out (hi) + lo16 with ld = N, row_stats, pivot_out, N %% 128 == 0\n");
    return -1;
  }
  if (g.epi == EPI_GEGLU && g.N % 128 != 0) {
    fprintf(stderr, "[srb200] gemm_f16: EPI_GEGLU needs N %% 128 == 0\n");
    return -1;
  }
  static int num_sms = 0;  // all devices of one box are the same part
  if (!num_sms) {
    int dev = 0, n = 0;
    SRB_CUDA_CHECK(cudaGetDevice(&dev));
    SRB_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    num_sms = n;
  }
  CUtensorMap ta, tb, tc;
  if (make_tmap_f16_kmajor(&ta, g.A, static_cast<uint64_t>(g.a_rows > 0 ? g.a_rows : g.M), g.K, BM)) return -1;
  const int w_groups = g.w_groups > 1 ? g.w_groups : 1;
  if (w_groups > 1 && (g.w_group_rows <= 0 || g.w_group_rows % BM != 0 || g.N % BN != 0 || g.epi == EPI_TOPK)) {
    fprintf(stderr, "[srb200] gemm_f16: grouped weights need w_group_rows %% %d == 0 and whole column tiles\n", BM);
    return -1;
  }
  if (make_tmap_f16_kmajor(&tb, g.W, static_cast<uint64_t>(g.N) * w_groups, g.K, BN)) return -1;
  // output boxes: 32 rows x 128 bytes (64 fp16 or 32 fp32 columns), clipped at M rows / n_out columns
  if (g.epi == EPI_TOPK) {
    tc = ta;   // no matrix output
  } else if (g.epi == EPI_RESID) {
    if (make_tmap_2d(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, g.out, g.N, g.M, g.ldo, 32, 32)) return -1;
  } else if (is_hl) {
    if (make_tmap_2d(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.out, g.N, g.M, g.N, 64, 32)) return -1;
  } else {
    const uint64_t n_out = g.epi == EPI_GEGLU ? g.N / 2 : g.N;
    if (make_tmap_2d(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.out, n_out, g.M, g.ldo, 64, 32)) return -1;
  }
  KArgs ka;
  ka.M = g.M; ka.N = g.N; ka.K = g.K;
  ka.bias = g.bias; ka.has_resid = g.resid != nullptr;
  ka.pos = g.pos; ka.rope_cos = g.rope_cos; ka.rope_sin = g.rope_sin; ka.rope_cols = g.rope_cols;
  ka.row_stats = nullptr; ka.has_raw16 = 0;
  ka.pivot_out = g.pivot_out; ka.pivot_in = g.pivot_in; ka.pivot_in_stats = g.pivot_in_stats;
  ka.topk_idx = g.topk_idx; ka.topk_score = g.topk_score; ka.topk_valid = g.topk_valid; ka.topk_n = g.topk_n;
  ka.grouped = 0;
  // SRB_RESID_INTERLEAVE=0 restores the contiguous ranges for the residual GEMMs (A/B measurements); =2 interleaves
  // the fp32-residual GEMMs for every K (by default only K > 768, whose row block is too large to survive in L2)
  static const bool resid_interleave = [] { const char* e = getenv("SRB_RESID_INTERLEAVE"); return !(e && e[0] == '0'); }();
  static const int interleave_min_k = [] { const char* e = getenv("SRB_RESID_INTERLEAVE"); return (e && e[0] == '2') ? 0 : 768; }();
  ka.interleave = (((g.epi == EPI_RESID && g.resid != nullptr) || is_hl) && resid_interleave && (is_hl || g.K > interleave_min_k) &&
                   g.N / BN > 1) ? 1 : 0;
  if ((g.pivot_in != nullptr) != (g.pivot_in_stats != nullptr) || ((g.pivot_out || g.pivot_in) && !g.row_stats)) {
    fprintf(stderr, "[srb200] gemm_f16: pivots come with row_stats, pivot_in with pivot_in_stats\n");
    return -1;
  }
  ka.fold_stats = nullptr; ka.fold_eps = 0.f; ka.fold_inv_h = 0.f; ka.fold_parts = 0;
  ka.K2 = 0; ka.mask_block = 0; ka.mask_rows = 0;
  ka.grp_rows = w_groups > 1 ? g.w_group_rows : 0;
  CUtensorMap ta2 = ta, tb2 = tb;   // K extension (low-rank adapters): unused copies otherwise
  if (g.K2 > 0) {
    if (!g.A2 || !g.W2 || g.K2 % 8 != 0 || g.epi == EPI_TOPK) {
      fprintf(stderr, "[srb200] gemm_f16: K extension needs A2, W2 and K2 %% 8 == 0\n");
      return -1;
    }
    if (make_tmap_f16_kmajor(&ta2, g.A2, static_cast<uint64_t>(g.a_rows > 0 ? g.a_rows : g.M), g.K2, BM)) return -1;
    if (make_tmap_f16_kmajor(&tb2, g.W2, g.N, g.K2, BN)) return -1;
    ka.K2 = g.K2;
  }
  if (g.mask_block > 0) {
    if (g.epi != EPI_F16 || g.mask_rows <= 0) {
      fprintf(stderr, "[srb200] gemm_f16: the column-block mask belongs to EPI_F16\n");
      return -1;
    }
    ka.mask_block = g.mask_block; ka.mask_rows = g.mask_rows;
  }
  CUtensorMap tx = tc;   // auxiliary output map (fp16 copy of the residual stream); unused otherwise
  if (is_hl) {
    if (make_tmap_2d(&tx, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.lo16, g.N, g.M, g.N, 64, 32)) return -1;
    ka.row_stats = g.row_stats;
  } else if (g.row_stats || g.raw16) {
    if (g.epi != EPI_RESID || g.N % 128 != 0) {
      fprintf(stderr, "[srb200] gemm_f16: row_stats / raw16 belong to EPI_RESID with N %% 128 == 0\n");
      return -1;
    }
    ka.row_stats = g.row_stats;
    if (g.raw16) {
      if (make_tmap_2d(&tx, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.raw16, g.N, g.M, g.N, 64, 32)) return -1;
      ka.has_raw16 = 1;
    }
  }
  if (g.fold_stats) {
    if ((g.epi != EPI_ROPE && g.epi != EPI_GEGLU) || g.fold_h <= 0 || g.fold_h % 128 != 0) {
      fprintf(stderr, "[srb200] gemm_f16: LayerNorm fold belongs to EPI_ROPE / EPI_GEGLU with the row length\n");
      return -1;
    }
    ka.fold_stats = g.fold_stats; ka.fold_eps = g.fold_eps;
    ka.fold_inv_h = 1.0f / static_cast<float>(g.fold_h);
    ka.fold_parts = g.fold_h / 128;
  }
  switch (g.epi) {
    case EPI_F16: return launch<EPI_F16>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms);
    case EPI_ROPE: return launch<EPI_ROPE>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms);
    case EPI_RESID: return launch<EPI_RESID>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms);
    case EPI_RESID_HL: return launch<EPI_RESID_HL>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms);
    case EPI_GEGLU: return launch<EPI_GEGLU>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms);
    case EPI_GELU: return launch<EPI_GELU>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms);
    case EPI_TOPK: {
      if (!g.topk_idx || !g.topk_score || !g.topk_lists || g.N % 256 != 0) {
        fprintf(stderr, "[srb200] gemm_f16: EPI_TOPK needs list buffers and N %% 256 == 0\n");
        return -1;
      }
      // the query batch is the short dimension here, the stored rows stream as N; one list per worker and query row
      const int m_blocks = (g.M + BM - 1) / BM, n_blocks = g.N / BN;
      const long long tiles = static_cast<long long>(m_blocks) * n_blocks;
      // grouped schedule (kernel comment at t_step): whole groups of m_blocks workers, each group at least one tile.
      // SRB_TOPK_GROUPED=0 restores the contiguous ranges (A/B measurements).
      static const bool grouped_on = [] { const char* e = getenv("SRB_TOPK_GROUPED"); return !(e && e[0] == '0'); }();
      const int groups = m_blocks > 0 ? num_sms / m_blocks : 0;
      if (grouped_on && m_blocks > 1 && groups >= 1 && n_blocks >= groups) {
        ka.grouped = 1;
        *g.topk_lists = groups * m_blocks;
        return launch<EPI_TOPK>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms, groups * m_blocks);
      }
      *g.topk_lists = static_cast<int>(tiles < num_sms ? tiles : num_sms);
      return launch<EPI_TOPK>(stream, ta, tb, tc, tx, ta2, tb2, ka, num_sms);
    }
  }
  return -1;
}

}  // namespace srb
