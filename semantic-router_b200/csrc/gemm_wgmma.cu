// Persistent, warp-specialised wgmma GEMM for sm_90a (Hopper) with fused epilogues.
//
//   C[M,N] = A[M,K] (fp16, K-major)  x  W[N,K]^T (fp16, K-major == nn.Linear layout), fp32 accumulate.
//
// Replaces the dense f32 `gemm`+rayon matmuls behind candle's Linear on the reference's hot loop
// (candle-binding/src/model_architectures/traditional/candle_models/modernbert.rs
//  :123 Wqkv, :196 Wo, :236-238 Wi/GeGLU/Wo) with two persistent kernels.  In this file, in order:
//   * what both kernels share: the wgmma wrappers, the operand-ring position (Ring), the tile schedule (tile_range),
//     the TMA producer (produce_operands), the prologue (kernel_prologue) and the closing barrier (cta_sync).
//   * gemm_kernel's epilogues, one Epilogue<EPI> per output form with only its own state: EPI_F16 / EPI_GELU (bias,
//     erf-GELU for BERT's intermediate), EPI_RESID (fp32 residual add, :300-303), EPI_RESID_HL (the fp16-pair residual
//     stream) and EPI_TOPK (the cache scan's running top-8).
//   * gemm_kernel, 128 x 128 tiles, for those epilogues
//     - warp 8      : TMA producer  (cp.async.bulk.tensor 2D, 128B swizzle, mbarrier complete_tx)
//     - warps 4..7  : one MMA warpgroup -- wgmma.mma_async m64n128k16 twice per k-step (rows 0-63, 64-127), fp32
//                     accumulators in registers; at the end of a tile they go to a swizzled fp32 tile in shared memory
//     - warps 0..3  : epilogue (shared fp32 tile -> registers, one row per lane -> fused math -> swizzled box -> TMA store)
//     - the accumulator tile in shared memory is the hand-off: the epilogue of tile i overlaps the mainloop of tile i+1,
//       whose accumulators live in the MMA warpgroup's registers until the epilogue has released the shared tile.
//   * gemm_wide_kernel, 128 x 192 tiles: the LayerNorm-fold projections, EPI_ROPE (rotate-half, modernbert.rs:61-85)
//     and EPI_GEGLU (gelu_erf(a)*b, :238), with two MMA warpgroups and the epilogue from their registers.  It is the
//     only kernel that runs in thread-block clusters (see there); results are bitwise those without clusters.
//   * the host side: tensor maps, the one list of kernel instances (with_kernel) and the launch.
#include "gemm.h"

#include <atomic>
#include <cstdlib>
#include <mutex>
#include <type_traits>

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
// staging boxes per epilogue warp: the fp32-residual epilogue's two-box ring, or the fp16-pair residual epilogue's one
// (hi, lo) box pair, loaded at the start of the chunk that uses it.  Shared memory is what limits this on sm_90: the
// 64 KB accumulator tile plus these boxes leave 4 mainloop stages.  A second pair (to load a chunk ahead) costs the
// fourth stage, and the residual GEMMs are bound by their operand feed, not by the epilogue's load latency: at
// T = 131072 on an H100 80GB HBM3 (700 W), two pairs and 3 stages ran Wo in 0.518 ms and Wo2 in 0.651-0.662 ms, one
// pair and 4 stages 0.443-0.444 and 0.528-0.536 ms (tools/gemm_prof.py).
constexpr int kStageBufs = 2;

// gemm_kernel's shared memory: the operand ring, the accumulator tile, the staging boxes and the barriers
struct GemmCfg {
  static constexpr int kBN = BN;   // W box height
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiBytes = kEpiWarps * kStageBufs * kStageBufBytes;
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
  float* row_stats;          // EPI_RESID_HL: (sum, sumsq) per row and 128-column slice
  const float* fold_stats;   // EPI_ROPE / EPI_GEGLU: per-row (sum, sumsq) of the A rows (null: no fold)
  float fold_eps;
  float fold_inv_h;
  int fold_parts;            // 128-column slices the row statistics come in
  float* pivot_out;          // EPI_RESID_HL: row pivots (see gemm.h)
  const float* pivot_in;
  const float* pivot_in_stats;
  int* topk_idx;             // EPI_TOPK
  float* topk_score;
  const uint8_t* topk_valid;
  int topk_n;
  int grouped;               // EPI_TOPK: grouped tile schedule (see the kernel)
  int interleave;            // tiles w, w + W, ... per worker instead of a contiguous range
  int grp_rows;              // > 0: W is a stack of [N, K] matrices, rows [g * grp_rows, (g + 1) * grp_rows) of A multiply matrix g
  int bias_stride;           // grp_rows > 0: group g's bias starts at bias + g * bias_stride (0: one bias for every group)
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
// D[64 x 192] (+)= A[64 x 16] * B[192 x 16]^T: the same fragment layout as m64n128k16, with j = 0..23 (gemm_wide_kernel)
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

// Byte offset of fp32 column `col` of row `row` in the shared accumulator tile: [BM][BN] fp32 rows, 16-byte units
// XOR-swizzled by (row & 7) inside each 128-byte group, so that a warp reading one row per lane (8 units each) and the
// MMA warpgroup writing its fragments both stay at the minimum number of shared-memory wavefronts.
__device__ __forceinline__ uint32_t acc_off(int row, int col) {
  const int u = col >> 2;
  return static_cast<uint32_t>(row * (BN * 4) + (((u & ~7) | ((u & 7) ^ (row & 7))) << 4) + (col & 3) * 4);
}

// ---- shared by both kernels ---------------------------------------------------------------------------------------
// Position in a ring of kStages buffers: the stage and the parity of its current round (the mbarrier phase bit)
template <int kStages>
struct Ring {
  int s = 0;
  uint32_t ph = 0;
  __device__ __forceinline__ void advance() {
    if (++s == kStages) { s = 0; ph ^= 1; }
  }
};

// The tiles of one worker: t = begin, begin + step, ... < end, numbered t = m_blk * n_tiles + n_tile (n fastest).  The
// workers of gemm_wide_kernel are clusters and its tiles cluster tiles.
struct TileRange { int begin, end, step; };
__device__ __forceinline__ TileRange tile_range(int m_blocks, int n_tiles, int worker, int workers, bool interleave,
                                                bool grouped) {
  const int num_tiles = m_blocks * n_tiles;
  if (grouped) {
    // EPI_TOPK, grouped schedule (p.grouped): worker w owns query block w % m_blocks for its whole life (its running
    // top-8 lists live in registers) and walks the stored-row tiles g, g + G, g + 2G, ... with g = w / m_blocks,
    // G = workers / m_blocks.  The m_blocks workers of a group therefore ask for the SAME stored-row tile at about the
    // same time: one HBM read, the rest L2 hits -- the store streams once per batch instead of once per query block.
    const int groups = workers / m_blocks;
    const int m_own = worker % m_blocks, g_own = worker / m_blocks;
    const int begin = m_own * n_tiles + g_own;
    return {begin, g_own < groups ? (m_own + 1) * n_tiles : begin, groups};   // workers beyond the last full group idle
  }
  // Interleaved schedule (p.interleave; the residual GEMMs): worker w takes tiles w, w + W, w + 2W, ...  With
  // n fastest in the tile numbering the N / BN tiles of one row block run AT THE SAME TIME on neighbouring workers, so
  // each A k-block is pulled from HBM once and hit in L2 by the others, where the contiguous ranges could lose the row
  // block from L2 to the residual stream passing through between two tiles of one worker.
  if (interleave) return {worker, num_tiles, workers};
  // contiguous tile range per worker: one worker walks all N tiles of its M blocks back to back, so the A row-block
  // stays hot in L2 and per-row epilogue state (pivots, top-8 lists, rstd, positions) is reused across tiles
  const int base = num_tiles / workers, rem = num_tiles % workers;
  const int begin = worker * base + (worker < rem ? worker : rem);
  return {begin, begin + base + (worker < rem ? 1 : 0), 1};
}

// TMA producer (one lane): every k-block of every tile of the worker into the operand ring, W in boxes of Cfg::kBN rows.
// CTA rn of a cluster of CN (1: none) loads its slice of the shared A box (tensor-map box height BM / CN rows, a multiple
// of the 8-row swizzle atom, so the slices assemble into exactly the tile layout one full-box load would give) and
// multicasts it to the whole cluster.
template <class Cfg, int CN>
__device__ __forceinline__ void produce_operands(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b, uint8_t* smem_a,
                                                 uint8_t* smem_b, uint64_t* full_bar, uint64_t* empty_bar,
                                                 const TileRange& tr, int n_tiles, int rn, int k_blocks, const KArgs& p) {
  Ring<Cfg::kStages> ring;
  constexpr int a_rows = BM / CN;
  const uint16_t a_mask = static_cast<uint16_t>((1u << CN) - 1);
  for (int t = tr.begin; t < tr.end; t += tr.step) {
    const int m_blk = t / n_tiles, n_blk = (t % n_tiles) * CN + rn;
    // grouped weights (one matrix per task, stacked along N): the row block picks its matrix; blocks never straddle
    // two groups (grp_rows is a multiple of the block height, checked on the host)
    const int w_row0 = p.grp_rows > 0 ? ((m_blk * BM) / p.grp_rows) * p.N : 0;
    for (int kb = 0; kb < k_blocks; ++kb) {
      mbar_wait(&empty_bar[ring.s], ring.ph ^ 1);
      const int kc = kb * BK;
      // the stage fills with the A slices of every CTA of the cluster and this CTA's own W box: the whole stage
      mbar_expect_tx(&full_bar[ring.s], Cfg::kStageBytes);
      uint8_t* da = smem_a + ring.s * Cfg::kABytes + rn * a_rows * (BK * 2);
      const int ya = m_blk * BM + rn * a_rows;
      if constexpr (CN > 1) tma_load_2d_multicast(da, tmap_a, &full_bar[ring.s], kc, ya, a_mask);
      else tma_load_2d(da, tmap_a, &full_bar[ring.s], kc, ya);
      tma_load_2d(smem_b + ring.s * Cfg::kBBytes, tmap_b, &full_bar[ring.s], kc, w_row0 + n_blk * Cfg::kBN);
      ring.advance();
    }
  }
}

// Barrier of the CTA, or of its cluster for CN > 1: no CTA may multicast into another or arrive on its barriers before
// those exist (kernel start), nor leave while another of its cluster may still arrive on its own (kernel end).
template <int CN>
__device__ __forceinline__ void cta_sync() {
  if constexpr (CN > 1) cluster_sync();
  else __syncthreads();
}

// Kernel start: thread 0 prefetches the tensor maps and sets up the operand ring's barriers (full: the producer's
// arrival and the stage's bytes; empty: `empty_arrivals`) and, in `init_more`, the kernel's own; then cta_sync.
template <int CN, int kStages, class InitMore>
__device__ __forceinline__ void kernel_prologue(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b,
                                                const CUtensorMap* tmap_out, uint64_t* full_bar, uint64_t* empty_bar,
                                                uint32_t empty_arrivals, InitMore init_more) {
  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmap_a);
    tma_prefetch_desc(tmap_b);
    tma_prefetch_desc(tmap_out);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], empty_arrivals);
    }
    init_more();
    mbar_fence_init();
  }
  cta_sync<CN>();
  // PDL: everything above overlapped the previous kernel's tail; nothing below may start before its writes are visible
  griddep_launch_dependents();
  griddep_wait();
}

// ---- gemm_kernel's epilogues ---------------------------------------------------------------------------------------
// An epilogue warp of gemm_kernel: warp `quad` owns rows 32 quad .. 32 quad + 31 of the tile, one per lane, and
// kStageBufs boxes of 32 rows x 128 bytes (one chunk of output columns) with a residual-load barrier each.  Per tile
// it runs row_block before the accumulator tile is ready (per-row loads overlap the mainloop), then tile.
struct EpiWarp {
  const KArgs& p;
  const CUtensorMap *tmap_out, *tmap_aux;   // tmap_aux: the lo boxes of EPI_RESID_HL
  int lane, quad;
  const uint8_t* acc_row;   // this thread's row of the accumulator tile
  uint8_t* bufs;
  uint64_t* rbar;
  TileRange tr;             // this CTA's tiles, n_blocks to a row block
  int n_blocks;
  // this thread's row, accumulator columns [col, col + 32) (col a multiple of 32)
  __device__ __forceinline__ void acc_ld32(int col, uint32_t* r) const {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 v = *reinterpret_cast<const uint4*>(acc_row + ((((col >> 2) + (i ^ (lane & 7)))) << 4));
      r[4 * i] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
    }
  }
  // TMA-store the box(es) this warp has written, as one store group (aux_buf: the lo box of EPI_RESID_HL's pair)
  __device__ __forceinline__ void store(const uint8_t* buf, int col, int row0, const uint8_t* aux_buf = nullptr) const {
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      tma_store_2d(tmap_out, buf, col, row0);  // rows >= M / cols >= N are clipped by the TMA unit
      if (aux_buf) tma_store_2d(tmap_aux, aux_buf, col, row0);
      bulk_commit();
    }
  }
  __device__ __forceinline__ void row_block(int) {}
  __device__ __forceinline__ void finish() {}
};

// EPI_F16 / EPI_GELU: fp16 out = acc + bias, erf-GELU'd for EPI_GELU, in 64-column chunks through the two boxes in
// turn.  A box is rewritten once its previous store has been read out: all but the newest store group, bulk_wait_read<1>.
template <int EPI>
struct Epilogue : EpiWarp {
  static_assert(EPI == EPI_F16 || EPI == EPI_GELU, "no gemm_kernel epilogue of this kind");
  int cb = 0;   // box of the next chunk
  __device__ __forceinline__ void tile(int, int m_blk, int n_blk, const float* bias) {
    const int row0 = m_blk * BM + quad * 32;
#pragma unroll 1
    for (int c = 0; c < BN / 64; ++c) {
      const int ocol0 = n_blk * BN + c * 64;
      if (ocol0 >= p.N) break;   // the last column tile of an N % 128 == 64 output is half empty
      uint8_t* my_row = bufs + cb * kStageBufBytes;  // + box_off(lane, chunk16)
      if (lane == 0) bulk_wait_read<1>();
      __syncwarp();
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        uint32_t r[32];
        acc_ld32(c * 64 + hf * 32, r);
        uint32_t h[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          float v0 = __uint_as_float(r[2 * i]), v1 = __uint_as_float(r[2 * i + 1]);
          if (bias) {
            const float2 b = __ldg(reinterpret_cast<const float2*>(bias + ocol0 + hf * 32) + i);
            v0 += b.x; v1 += b.y;
          }
          if constexpr (EPI == EPI_GELU) { v0 = gelu_erf_fast_f(v0); v1 = gelu_erf_fast_f(v1); }
          h[i] = pack_half2(v0, v1);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
          sts16(my_row + box_off(lane, hf * 4 + i), h[4 * i], h[4 * i + 1], h[4 * i + 2], h[4 * i + 3]);
      }
      store(my_row, ocol0, row0);
      cb ^= 1;
    }
  }
};

// EPI_RESID: fp32 out = acc + bias, plus out itself in place (has_resid), in 32-column chunks.  With a residual the two
// boxes are a ring over this CTA's (tile, chunk) sequence: while a chunk is computed in one, the next chunk's residual
// loads into the other.  The previous chunk stored from that box, the newest store group, so the load waits for every
// store to be read out: bulk_wait_read<0>.  Without a residual the boxes alternate as in EPI_F16.
template <>
struct Epilogue<EPI_RESID> : EpiWarp {
  static constexpr int kChunks = BN / 32;
  const bool use_resid;
  int cb = 0;         // box of the next chunk
  uint32_t rph = 0;   // phase bit per box (residual loads)
  __device__ __forceinline__ Epilogue(const EpiWarp& w) : EpiWarp(w), use_resid(w.p.has_resid) {
    if (use_resid && lane == 0 && tr.begin < tr.end) load(0, tr.begin, 0);   // the first chunk
  }
  // lane 0: the residual of chunk c of tile t into box b
  __device__ __forceinline__ void load(int b, int t, int c) {
    mbar_expect_tx(&rbar[b], kStageBufBytes);
    tma_load_2d(bufs + b * kStageBufBytes, tmap_out, &rbar[b], (t % n_blocks) * BN + c * 32, (t / n_blocks) * BM + quad * 32);
  }
  __device__ __forceinline__ void tile(int t, int m_blk, int n_blk, const float* bias) {
    const int row0 = m_blk * BM + quad * 32;
#pragma unroll 1
    for (int c = 0; c < kChunks; ++c) {
      const int ocol0 = n_blk * BN + c * 32;
      if (ocol0 >= p.N) break;   // the last column tile of an N % 128 == 64 output is half empty
      uint8_t* my_row = bufs + cb * kStageBufBytes;  // + box_off(lane, chunk16)
      if (use_resid) {
        if (lane == 0) {
          bulk_wait_read<0>();
          if (c + 1 < kChunks && ocol0 + 32 < p.N) load(cb ^ 1, t, c + 1);
          else if (t + tr.step < tr.end) load(cb ^ 1, t + tr.step, 0);
        }
        mbar_wait(&rbar[cb], (rph >> cb) & 1u);
        rph ^= 1u << cb;
      } else {
        if (lane == 0) bulk_wait_read<1>();  // this box's previous store has been read out
        __syncwarp();
      }
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
        if (bias) {
          const float4 b = __ldg(reinterpret_cast<const float4*>(bias + ocol0) + i);
          x.x += b.x; x.y += b.y; x.z += b.z; x.w += b.w;
        }
        *q = x;
      }
      store(my_row, ocol0, row0);
      cb ^= 1;
    }
  }
};

// EPI_RESID_HL: the fp16-pair residual stream, hi (tmap_out) + lo (tmap_aux) = x - pivot.  Per 64-column chunk the
// warp's one (hi, lo) box pair is loaded once its previous store has been read out (bulk_wait_read<0>), updated in
// place and stored.  Row statistics go out per 128-column slice (N % 128 == 0: no chunk is past N), in chunk order.
template <>
struct Epilogue<EPI_RESID_HL> : EpiWarp {
  float pv = 0.f;       // the pivot SHIFT of this GEMM for this thread's row
  float pv_prev = 0.f;  // the pivot the stored pair is relative to
  int pv_mblk = -1;
  uint32_t rph = 0;     // phase bit of the pair's barrier
  __device__ __forceinline__ void row_block(int m_blk) {
    // pivot shift of this row: the stored pair is x - pivot_in; the new pivot is pivot_in + (mean of x - pivot_in),
    // read from the previous residual GEMM's statistics (0 for the first one: the embedding's pair is x itself)
    if (m_blk == pv_mblk) return;
    pv = 0.f;
    pv_prev = 0.f;
    if (p.pivot_in_stats) {
      const int row0 = m_blk * BM + quad * 32;
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

  __device__ __forceinline__ void tile(int, int m_blk, int n_blk, const float* bias) {
    const int row0 = m_blk * BM + quad * 32;
    uint8_t* hb = bufs;
    uint8_t* lb = hb + kStageBufBytes;
    float st1 = 0.f, st2 = 0.f;   // this row's (sum, sum of squares) over the current 128-column slice
#pragma unroll 1
    for (int c = 0; c < BN / 64; ++c) {
      const int ocol0 = n_blk * BN + c * 64;
      if (lane == 0) {
        bulk_wait_read<0>();
        mbar_expect_tx(&rbar[0], 2 * kStageBufBytes);
        tma_load_2d(hb, tmap_out, &rbar[0], ocol0, row0);
        tma_load_2d(lb, tmap_aux, &rbar[0], ocol0, row0);
      }
      mbar_wait(&rbar[0], rph);
      rph ^= 1u;
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
            if (bias) {
              const float2 b = __ldg(reinterpret_cast<const float2*>(bias + ocol0 + hf * 32 + 8 * u) + k);
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
      store(hb, ocol0, row0, lb);
    }
  }
};

// EPI_TOPK: this thread's running top-8 (descending) over the columns this CTA walks for its current row, written out
// as this CTA's list for the row when the row block changes and after the last tile.
template <>
struct Epilogue<EPI_TOPK> : EpiWarp {
  float tk_v[kTopK];   // set at the first row block
  int tk_i[kTopK];
  int tk_mblk = -1;
  __device__ __forceinline__ Epilogue(const EpiWarp& w) : EpiWarp(w) {}
  __device__ __forceinline__ void flush() {   // this CTA's list for the row it has just left
    const int row = tk_mblk * BM + quad * 32 + lane;
    if (row < p.M) {
      const size_t at = (static_cast<size_t>(row) * gridDim.x + blockIdx.x) * kTopK;
#pragma unroll
      for (int i = 0; i < kTopK; ++i) { p.topk_idx[at + i] = tk_i[i]; p.topk_score[at + i] = tk_v[i]; }
    }
  }
  __device__ __forceinline__ void row_block(int m_blk) {
    if (m_blk == tk_mblk) return;
    if (tk_mblk >= 0) flush();
#pragma unroll
    for (int i = 0; i < kTopK; ++i) { tk_v[i] = -INFINITY; tk_i[i] = -1; }
    tk_mblk = m_blk;
  }
  __device__ __forceinline__ void finish() {
    if (tk_mblk >= 0) flush();
  }
  // This warp scans the tile's columns 32 at a time.  The common path per chunk is the maximum of 32 scores and
  // one compare against the list's tail; validity (invalidated rows, padding rows >= topk_n) is only looked up
  // for a score that would enter the list -- after the first tiles that is rare.
  __device__ __forceinline__ void topk_chunk(uint32_t* r, int ocol0) {
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
        // insertion into the descending list: strict > finds the slot (after any equal score, which has the lower
        // column), and from there every entry shifts down one, ties included, so the tail is the one dropped
        bool shift = false;
#pragma unroll
        for (int j = 0; j < kTopK; ++j) {
          if (shift || cv > tk_v[j]) {
            shift = true;
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
  }

  __device__ __forceinline__ void tile(int, int, int n_blk, const float*) {
#pragma unroll 1
    for (int c = 0; c < BN / 32; ++c) {
      uint32_t r[32];
      acc_ld32(c * 32, r);
      topk_chunk(r, n_blk * BN + c * 32);
    }
  }
};

// ================= gemm_kernel: 128 x 128 tiles, epilogue warps fed through the shared accumulator tile =================
template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
            const __grid_constant__ CUtensorMap tmap_out, const __grid_constant__ CUtensorMap tmap_aux, const KArgs p) {
  static_assert(EPI != EPI_ROPE && EPI != EPI_GEGLU, "the LayerNorm-fold projections run on gemm_wide_kernel");
  using Cfg = GemmCfg;
  static_assert(Cfg::kSmemBytes <= kSmemLimit, "over the 227 KB shared-memory opt-in limit");
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
  const int k_blocks = (p.K + BK - 1) / BK;
  const TileRange tr = tile_range(m_blocks, n_blocks, blockIdx.x, gridDim.x, p.interleave, EPI == EPI_TOPK && p.grouped);

  kernel_prologue<1, Cfg::kStages>(&tmap_a, &tmap_b, &tmap_out, full_bar, empty_bar, 4 /*one arrival per MMA warp*/, [&] {
    mbar_init(tfull_bar, 128);            // every thread of the MMA warpgroup, after its fragment stores
    mbar_init(tempty_bar, kEpiWarps);
    for (int i = 0; i < kEpiWarps * kStageBufs; ++i) mbar_init(&resid_bar[i], 1);
  });

  if (warp == kProducerWarp) {
    // ================= TMA producer =================
    if (lane == 0) produce_operands<Cfg, 1>(&tmap_a, &tmap_b, smem_a, smem_b, full_bar, empty_bar, tr, n_blocks, 0, k_blocks, p);
  } else if (warp >= kMmaWarp0) {
    // ================= MMA warpgroup =================
    const int wq = warp - kMmaWarp0;   // warp of the warpgroup: fragment rows 16 wq .. 16 wq + 15 of each 64-row half
    float acc[2][64];
    Ring<Cfg::kStages> ring;
    uint32_t eph = 0;   // tempty phase
    for (int t = tr.begin; t < tr.end; t += tr.step) {
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[ring.s], ring.ph);
        wgmma_fence();
        const uint32_t a0 = smem_u32(smem_a + ring.s * Cfg::kABytes);
        const uint32_t b0 = smem_u32(smem_b + ring.s * Cfg::kBBytes);
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
        prev = ring.s;
        ring.advance();
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
    Epilogue<EPI> epi{EpiWarp{p, &tmap_out, &tmap_aux, lane, warp, smem_acc + (warp * 32 + lane) * (BN * 4),
                              smem_epi + warp * (kStageBufs * kStageBufBytes), resid_bar + warp * kStageBufs, tr, n_blocks}};
    uint32_t aph = 0;
    for (int t = tr.begin; t < tr.end; t += tr.step) {
      const int m_blk = t / n_blocks, n_blk = t % n_blocks;
      // grouped weights with a bias per matrix (stacked like the matrices): the row block adds its matrix's
      const float* bias = (p.bias && p.grp_rows > 0) ? p.bias + static_cast<size_t>((m_blk * BM) / p.grp_rows) * p.bias_stride : p.bias;
      epi.row_block(m_blk);
      mbar_wait(tfull_bar, aph);
      aph ^= 1;
      epi.tile(t, m_blk, n_blk, bias);
      // release the accumulator tile back to the MMA warpgroup
      __syncwarp();
      if (lane == 0) mbar_arrive(tempty_bar);
    }
    epi.finish();
    if (lane == 0) bulk_wait_read<0>();  // smem must outlive the last stores' reads
    __syncwarp();
  }
  cta_sync<1>();
}

// ================= the LayerNorm-fold projections (EPI_ROPE, EPI_GEGLU) on 128 x 192 tiles =================
// gemm_wide_kernel runs
//   * warps 0..7 : two MMA warpgroups; warpgroup w owns rows 64 w .. 64 w + 63 of the tile: m64n192k16 per k-step,
//     then the epilogue straight from its accumulator fragment (fold rstd, RoPE or GeGLU, fp16 pack) into a swizzled
//     16-row box per warp, stored by TMA.  There is no fp32 hand-off through shared memory to separate epilogue warps:
//     for these two large projections that hand-off, and the single MMA warpgroup stalling on it, cost about a quarter
//     of the GEMM.
//   * warp 8     : TMA producer; it fills the ring for the next tile while the warpgroups run the epilogue.
// 288 threads: nine warps, three on one SM sub-partition, so ptxas allocates at most 16384 / 96 -> 168 registers per
// thread.  The 96 accumulators and the epilogue fit in that without spilling (-Xptxas -v: 166-168).
// 192 = three 64-wide heads, and in the fragment columns c and c + 32 sit in the same thread, which is the pairing of
// both rotate-half RoPE and the 32-row (a | b) interleave of the GeGLU weights.
// Thread-block clusters of CN CTAs along N (1: none): the schedule (contiguous ranges) hands out CLUSTER tiles -- cn neighbouring tiles of
// one row block -- and CTA rn of the cluster computes tile (m_c, cn n_c + rn) of cluster tile (m_c, n_c).  The cn CTAs
// share the A row block: each loads a 1/cn slice of the A box and multicasts it to all of them, so an A k-block is read
// out of L2 once per cluster instead of once per CTA.  All CTAs of a cluster walk the same cluster tiles and k-blocks in
// lockstep.  (Sharing W across row blocks as well was measured slower at every projection shape.)
// LayerNorm fold, consumer side.  W'' = (W diag(gamma)) with every row re-centred to sum zero, so that
// sum_k x[r,k] W''[n,k] = sum_k (x[r,k] - mean_r) W'[n,k]: the mean subtraction of the LayerNorm happens inside the GEMM
// (the centring matrix I - 11^T/H commutes into the weights) and the epilogue is left with the per-row rstd factor --
// which the RoPE epilogue folds into the row's cos / sin (the rotation is linear), so q and k cost nothing.
constexpr int BNW = 192;
constexpr int kWideThreads = 32 * 9;

template <int EPI>
struct WideCfg {
  static constexpr int kBN = BNW;   // W box height
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BNW * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // output box per warp and 64-column accumulator group: 16 rows x 64 fp16 (RoPE, 128B swizzle) or x 32 fp16 (GeGLU's
  // halved width, 64B swizzle)
  static constexpr int kBoxCols = EPI == EPI_GEGLU ? 32 : 64;
  static constexpr int kBoxBytes = 16 * kBoxCols * 2;
  static constexpr int kEpiBytes = 8 * 3 * kBoxBytes;
  static constexpr int kFit = (kSmemLimit - kEpiBytes - 1024 /*align slack*/ - kBarrierBytes) / kStageBytes;
  static constexpr int kStages = kFit < 6 ? kFit : 6;
  static constexpr int kSmemBytes = kStages * kStageBytes + kEpiBytes + 1024 + kBarrierBytes;
  static_assert(kStages >= 3, "mainloop ring too shallow");
};

template <int EPI, int CN>
__global__ void __launch_bounds__(kWideThreads, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_out, const KArgs p) {
  static_assert(EPI == EPI_ROPE || EPI == EPI_GEGLU, "the wide kernel serves the LayerNorm-fold projections");
  using Cfg = WideCfg<EPI>;
  static_assert(Cfg::kSmemBytes <= kSmemLimit, "over the 227 KB shared-memory opt-in limit");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + Cfg::kStages * Cfg::kABytes;
  uint8_t* smem_epi = smem + Cfg::kStages * Cfg::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_epi + Cfg::kEpiBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_blocks = (p.M + BM - 1) / BM;
  const int n_blocks = (p.N + BNW - 1) / BNW;
  const int k_blocks = (p.K + BK - 1) / BK;
  constexpr int cn = CN;
  const int rn = blockIdx.x % cn;
  const int n_cblocks = (n_blocks + cn - 1) / cn;   // cluster tiles per row block (see above)
  const TileRange tr = tile_range(m_blocks, n_cblocks, blockIdx.x / cn, gridDim.x / cn, false, false);

  // one arrival per MMA warp of every CTA of the cluster frees a stage
  kernel_prologue<CN, Cfg::kStages>(&tmap_a, &tmap_b, &tmap_out, full_bar, empty_bar, 8 * cn, [] {});

  if (warp == 8) {
    // ================= TMA producer =================
    if (lane == 0) produce_operands<Cfg, CN>(&tmap_a, &tmap_b, smem_a, smem_b, full_bar, empty_bar, tr, n_cblocks, rn, k_blocks, p);
  } else {
    // ================= MMA warpgroups, epilogue from the accumulator fragment =================
    const int wg = warp >> 2;         // 64-row half of the tile
    const int wq = warp & 3;          // fragment rows 16 wq .. 16 wq + 15 of that half
    const int q = lane & 3;
    const int fr = lane >> 2;         // this thread's rows: fr and fr + 8 of the warp's 16
    const bool fold = p.fold_stats != nullptr;
    const int n_out = (EPI == EPI_GEGLU) ? p.N / 2 : p.N;
    uint8_t* my_boxes = smem_epi + warp * 3 * Cfg::kBoxBytes;
    float acc[96];
    float rstd[2] = {1.f, 1.f};   // per row of the thread: the fold's rstd and (EPI_ROPE) the position
    int pos[2] = {0, 0};
    int row_mblk = -1;
    Ring<Cfg::kStages> ring;
    // a stage of this CTA is written by the producers of every CTA of its cluster (A slices): freeing it is one
    // arrival on the empty barrier of each of them, lane i for CTA i, so that the arrivals go out side by side on the
    // MMA warp's critical path
    auto release = [&](int st) {
      if (cn == 1) {
        if (lane == 0) mbar_arrive(&empty_bar[st]);
      } else if (lane < cn) {
        mbar_arrive_cluster(&empty_bar[st], lane);
      }
    };
    for (int t = tr.begin; t < tr.end; t += tr.step) {
      const int m_blk = t / n_cblocks, n_blk = (t % n_cblocks) * cn + rn;
      const int row0 = m_blk * BM + 64 * wg + 16 * wq;   // first row of this warp's boxes
      if (m_blk != row_mblk) {   // per-row state, reloaded only when the row block changes
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row0 + fr + 8 * h < p.M ? row0 + fr + 8 * h : p.M - 1;   // rows past M: never stored
          if (fold) {
            float s1 = 0.f, s2 = 0.f;
            for (int k = 0; k < p.fold_parts; ++k) {
              const float2 st = __ldg(reinterpret_cast<const float2*>(p.fold_stats) + static_cast<size_t>(k) * p.M + row);
              s1 += st.x;
              s2 += st.y;
            }
            const float mean = s1 * p.fold_inv_h;
            const float var = fmaxf(s2 * p.fold_inv_h - mean * mean, 0.f);
            rstd[h] = rsqrtf(var + p.fold_eps);
          }
          if constexpr (EPI == EPI_ROPE) {
            if (p.rope_cols > 0) pos[h] = __ldg(p.pos + row);
          }
        }
        row_mblk = m_blk;
      }
      int prev = -1;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&full_bar[ring.s], ring.ph);
        wgmma_fence();
        const uint32_t a0 = smem_u32(smem_a + ring.s * Cfg::kABytes) + wg * 64 * 128;
        const uint32_t b0 = smem_u32(smem_b + ring.s * Cfg::kBBytes);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_m64n192k16(acc, gmma_desc_sw128(a0 + 32 * k), gmma_desc_sw128(b0 + 32 * k), (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        __syncwarp();
        if (prev >= 0) release(prev);
        prev = ring.s;
        ring.advance();
      }
      wgmma_wait<0>();
      __syncwarp();
      if (prev >= 0) release(prev);

      const bool rotate = EPI == EPI_ROPE && n_blk * BNW < p.rope_cols;   // the tile holds rotated (q, k) heads
      // this warp's boxes of the previous tile have been read out by the TMA unit
      if (lane == 0) bulk_wait_read<0>();
      __syncwarp();
#pragma unroll
      for (int h = 0; h < 2; ++h) {   // the thread's two rows
        const int br = fr + 8 * h;     // row inside the boxes
        // EPI_ROPE: cos / sin of the row's first-half head columns 8 jj + 2 q + {0, 1}, carrying its rstd -- loaded once
        // per row and tile, after the mainloop.  Holding them across the mainloop, or both rows' at once, spills: at 288
        // threads ptxas gives this kernel 168 registers (three of the nine warps share a sub-partition: 16384 / 96), and
        // the 96 accumulators take most of them.
        float c[EPI == EPI_ROPE ? 8 : 1], sv[EPI == EPI_ROPE ? 8 : 1];
        if constexpr (EPI == EPI_ROPE) {
          if (rotate) {
            const float2* c2 = reinterpret_cast<const float2*>(p.rope_cos + static_cast<size_t>(pos[h]) * 32);
            const float2* s2 = reinterpret_cast<const float2*>(p.rope_sin + static_cast<size_t>(pos[h]) * 32);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const float2 cv = __ldg(c2 + 4 * jj + q), svv = __ldg(s2 + 4 * jj + q);
              c[2 * jj] = cv.x; c[2 * jj + 1] = cv.y;
              sv[2 * jj] = svv.x; sv[2 * jj + 1] = svv.y;
            }
            if (fold) {   // LayerNorm fold: the rstd factor of the row rides on the (linear) rotation
#pragma unroll
              for (int i = 0; i < 8; ++i) { c[i] *= rstd[h]; sv[i] *= rstd[h]; }
            }
          }
        }
#pragma unroll
        for (int g = 0; g < 3; ++g) {   // 64-column accumulator group: one head (RoPE) or one (a | b) pair of 32 (GeGLU)
          uint8_t* box = my_boxes + g * Cfg::kBoxBytes;
          const int col0 = n_blk * BNW + 64 * g;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            // columns 64 g + 8 jj + 2 q + {0, 1} (a) and the same + 32 (b) of the tile: fragment entries j, j + 4
            const int ja = 8 * g + jj, jb = ja + 4;
            const float a0 = acc[4 * ja + 2 * h], a1 = acc[4 * ja + 2 * h + 1];
            const float b0 = acc[4 * jb + 2 * h], b1 = acc[4 * jb + 2 * h + 1];
            if constexpr (EPI == EPI_ROPE) {
              uint32_t oa, ob;
              if (rotate && col0 < p.rope_cols) {   // q and k heads: rotate-half over the 64-wide head
                oa = pack_half2(a0 * c[2 * jj] - b0 * sv[2 * jj], a1 * c[2 * jj + 1] - b1 * sv[2 * jj + 1]);
                ob = pack_half2(a0 * sv[2 * jj] + b0 * c[2 * jj], a1 * sv[2 * jj + 1] + b1 * c[2 * jj + 1]);
              } else if (fold) {   // v columns: no rotation to carry rstd
                oa = pack_half2(a0 * rstd[h], a1 * rstd[h]);
                ob = pack_half2(b0 * rstd[h], b1 * rstd[h]);
              } else {
                oa = pack_half2(a0, a1);
                ob = pack_half2(b0, b1);
              }
              sts_b32(box + br * 128 + ((jj ^ (br & 7)) << 4) + 4 * q, oa);
              sts_b32(box + br * 128 + (((jj + 4) ^ (br & 7)) << 4) + 4 * q, ob);
            } else {
              const float rs = fold ? rstd[h] : 1.0f;
              const float kz = rs * 0.70710678118654752440f, kh = 0.5f * rs * rs;
              const float g0 = geglu_fold_f(a0, b0, kz, kh);
              const float g1 = geglu_fold_f(a1, b1, kz, kh);
              sts_b32(box + br * 64 + ((jj ^ ((br >> 1) & 3)) << 4) + 4 * q, pack_half2(g0, g1));
            }
          }
        }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          // output columns of the group; a group wholly past N (a partial last tile) is not stored, rows >= M and
          // columns >= n_out inside a box are clipped by the TMA unit
          const int ocol0 = EPI == EPI_GEGLU ? n_blk * (BNW / 2) + 32 * g : n_blk * BNW + 64 * g;
          if (ocol0 < n_out) tma_store_2d(&tmap_out, my_boxes + g * Cfg::kBoxBytes, ocol0, row0);
        }
        bulk_commit();
      }
    }
    if (lane == 0) bulk_wait_read<0>();   // smem must outlive the last stores' reads
    __syncwarp();
  }
  cta_sync<CN>();
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

// The kernel instance of an epilogue and cluster size: gemm_wide_kernel for the LayerNorm-fold projections, in clusters
// of CN CTAs; gemm_kernel, which has no clusters, for every other epilogue.
template <int EPI, int CN>
struct Kernel {
  static constexpr bool kWide = EPI == EPI_ROPE || EPI == EPI_GEGLU;
  static_assert(kWide || CN == 1, "gemm_kernel runs without clusters");
  static constexpr int kCN = CN;
  using Cfg = std::conditional_t<kWide, WideCfg<EPI>, GemmCfg>;
  static constexpr int kThreads = kWide ? kWideThreads : kGemmThreads;
  static constexpr auto fn() {
    if constexpr (kWide) return gemm_wide_kernel<EPI, CN>;
    else return gemm_kernel<EPI>;
  }
};

// f(Kernel<EPI, CN>{}) for the kernel instance of (epi, cn): the one list of the instances gemm_f16 launches
template <class F>
int with_kernel(int epi, int cn, F&& f) {
  switch (epi) {
    case EPI_F16: return f(Kernel<EPI_F16, 1>{});
    case EPI_ROPE: return cn == 2 ? f(Kernel<EPI_ROPE, 2>{}) : f(Kernel<EPI_ROPE, 1>{});
    case EPI_RESID: return f(Kernel<EPI_RESID, 1>{});
    case EPI_RESID_HL: return f(Kernel<EPI_RESID_HL, 1>{});
    case EPI_GEGLU: return cn == 2 ? f(Kernel<EPI_GEGLU, 2>{}) : f(Kernel<EPI_GEGLU, 1>{});
    case EPI_GELU: return f(Kernel<EPI_GELU, 1>{});
    case EPI_TOPK: return f(Kernel<EPI_TOPK, 1>{});
  }
  return -1;
}

// Launch configuration of kernel instance Kn but its grid, the cluster shape in attr[0].  The shared-memory opt-in is a
// per-device attribute, cheap enough to set before every use (multi-GPU processes switch devices).
template <class Kn>
int kernel_config(cudaLaunchConfig_t& cfg, cudaLaunchAttribute* attr) {
  SRB_CUDA_CHECK(cudaFuncSetAttribute(Kn::fn(), cudaFuncAttributeMaxDynamicSharedMemorySize, Kn::Cfg::kSmemBytes));
  cfg = {};
  cfg.blockDim = dim3(Kn::kThreads);
  cfg.dynamicSmemBytes = Kn::Cfg::kSmemBytes;
  cfg.attrs = attr;
  if (Kn::kCN > 1) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = Kn::kCN;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.numAttrs = 1;
  }
  return 0;
}

// Clusters of the kernel instance that are co-resident on the device.  A GPC holds a whole number of clusters, so
// this is the occupancy query's answer, not num_sms / CN.  Asked once per instance (all devices of one box are the
// same part).
template <class Kn>
int max_clusters(int num_sms) {
  static std::atomic<int> cached{0};
  int n = cached.load(std::memory_order_relaxed);
  if (n > 0) return n;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[1];
  if (kernel_config<Kn>(cfg, attr)) return -1;
  cfg.gridDim = dim3(Kn::kCN * num_sms);
  SRB_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&n, Kn::fn(), &cfg));
  if (n <= 0) {
    fprintf(stderr, "[srb200] gemm_f16: no %d-CTA cluster of this kernel fits the device\n", Kn::kCN);
    return -1;
  }
  cached.store(n, std::memory_order_relaxed);
  return n;
}

template <class Kn>
int launch(cudaStream_t stream, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc,
           const CUtensorMap& tx, const KArgs& ka, int num_sms, int grid_override) {
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  if (kernel_config<Kn>(cfg, attr)) return -1;
  cfg.stream = stream;
  if (pdl_enabled()) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[cfg.numAttrs++].val.programmaticStreamSerializationAllowed = 1;
  }
  constexpr int tile_n = Kn::Cfg::kBN * Kn::kCN;   // cluster tiles
  const int tiles = ((ka.M + BM - 1) / BM) * ((ka.N + tile_n - 1) / tile_n);
  // persistent grid: one worker per co-resident cluster (one per SM without clusters)
  const int workers = Kn::kCN > 1 ? max_clusters<Kn>(num_sms) : num_sms;
  if (workers <= 0) return -1;
  cfg.gridDim = dim3(grid_override > 0 ? grid_override : Kn::kCN * (tiles < workers ? tiles : workers));
  if constexpr (Kn::kWide) SRB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, Kn::fn(), ta, tb, tc, ka));
  else SRB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, Kn::fn(), ta, tb, tc, tx, ka));
  note_launch();
  return 0;
}

}  // namespace

static int make_tmap_2d(CUtensorMap* out, CUtensorMapDataType dt, int elem_bytes, const void* ptr, uint64_t cols,
                        uint64_t rows, uint64_t ld_elems, uint32_t box_cols, uint32_t box_rows,
                        CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
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
                  swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
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

// Measured at T = 131072 (ModernBERT-base, tools/gemm_prof.py), ms per GEMM, every GEMM on 128 x 128 tiles.  H100 80GB
// HBM3 at a 400 W power limit (power-capped SM clock), clusters of 1 x 1 / 2 x 1 (two row blocks share W) / 1 x 2 (two
// column tiles share A) / 2 x 2:  Wqkv (EPI_ROPE, N 2304, K 768) 1.46 / 1.52 / 1.31 / 1.29;  Wi (EPI_GEGLU, N 2304)
// 1.39 / 1.39 / 1.28 / 1.46;  Wo2 (EPI_RESID_HL, N 768, K 1152) 0.93 / 1.00 / 0.89 / 0.98;  Wo (EPI_RESID_HL, K 768)
// 0.59 / 0.63 / 0.64 / 0.67.  The same card at 700 W, 1 x 1 / 1 x 2:  Wqkv 1.08 / 0.96;  Wi 1.00 / 0.94;  Wo2 0.69 / 0.74.
// Only sharing A helps, so clusters are 1 x cn only, and only the two large LayerNorm-fold projections
// (gemm_wide_kernel) use them.  The residual GEMMs run without clusters (a deeper operand ring sped them up instead:
// GemmCfg, Wo 0.52 -> 0.44 ms, Wo2 0.66 -> 0.53 ms at 700 W); so do the epilogues not measured here (EPI_F16, EPI_GELU, EPI_RESID) and EPI_TOPK, whose
// grouped schedule gives each worker its own query block.
// A pair forms only where N's column-tile count is even both in 128-wide and in 192-wide tiles.  The 192-wide kernel
// needs the second condition: with an odd count, every other cluster would carry a CTA that computes a tile wholly past
// N.  The first condition is kept because this rule is the configuration the clustered 192-wide kernel was measured in.
// A rule on 192-wide tiles alone would pair shapes that run unpaired today (ModernBERT-large's Wi at N = 5248: 41 tiles
// of 128, 28 of 192), and its speed there has not been measured.
int gemm_cluster_size(int epi, int N, int K) {
  (void)K;
  const bool share_a = epi == EPI_ROPE || epi == EPI_GEGLU;
  return share_a && ((N + BN - 1) / BN) % 2 == 0 && ((N + BNW - 1) / BNW) % 2 == 0 ? 2 : 1;
}

int device_sms() {
  static int num_sms = 0;
  if (!num_sms) {
    int dev = 0, n = 0;
    SRB_CUDA_CHECK(cudaGetDevice(&dev));
    SRB_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    num_sms = n;
  }
  return num_sms;
}

int gemm_cluster_workers(int epi, int N, int K) {
  const int cn = gemm_cluster_size(epi, N, K);
  const int num_sms = device_sms();
  if (num_sms <= 0 || cn == 1) return num_sms;
  return with_kernel(epi, cn, [&](auto kn) { return max_clusters<decltype(kn)>(num_sms); });
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
  if (is_hl && (!g.lo16 || !g.row_stats || !g.pivot_out || g.N % 128 != 0 || g.ldo != g.N || g.resid ||
                (g.pivot_in != nullptr) != (g.pivot_in_stats != nullptr))) {
    fprintf(stderr, "[srb200] gemm_f16: EPI_RESID_HL needs out (hi) + lo16 with ld = N, row_stats, pivot_out, "
                    "pivot_in with pivot_in_stats, N %% 128 == 0\n");
    return -1;
  }
  if (!is_hl && (g.lo16 || g.row_stats || g.pivot_out || g.pivot_in || g.pivot_in_stats)) {
    fprintf(stderr, "[srb200] gemm_f16: lo16, row_stats and pivots belong to EPI_RESID_HL\n");
    return -1;
  }
  if (g.epi == EPI_GEGLU && g.N % 128 != 0) {
    fprintf(stderr, "[srb200] gemm_f16: EPI_GEGLU needs N %% 128 == 0\n");
    return -1;
  }
  const int num_sms = device_sms();
  if (num_sms <= 0) return -1;
  const int cn = gemm_cluster_size(g.epi, g.N, g.K);
  const bool wide = g.epi == EPI_ROPE || g.epi == EPI_GEGLU;   // gemm_wide_kernel
  // operand boxes: each CTA of a cluster loads 1/cn of the A box (kernel: TMA producer)
  CUtensorMap ta, tb, tc;
  if (make_tmap_f16_kmajor(&ta, g.A, static_cast<uint64_t>(g.a_rows > 0 ? g.a_rows : g.M), g.K, BM / cn)) return -1;
  const int w_groups = g.w_groups > 1 ? g.w_groups : 1;
  if (w_groups > 1 && (g.w_group_rows <= 0 || g.w_group_rows % BM != 0 || g.N % BN != 0 || g.epi == EPI_TOPK)) {
    fprintf(stderr, "[srb200] gemm_f16: grouped weights need w_group_rows %% %d == 0 and whole column tiles\n", BM);
    return -1;
  }
  if (make_tmap_f16_kmajor(&tb, g.W, static_cast<uint64_t>(g.N) * w_groups, g.K, wide ? BNW : BN)) return -1;
  // output boxes, clipped at M rows / n_out columns.  gemm_kernel: 32 rows x 128 bytes (64 fp16 or 32 fp32 columns)
  if (g.epi == EPI_TOPK) {
    tc = ta;   // no matrix output
  } else if (g.epi == EPI_RESID) {
    if (make_tmap_2d(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, g.out, g.N, g.M, g.ldo, 32, 32)) return -1;
  } else if (is_hl) {
    if (make_tmap_2d(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.out, g.N, g.M, g.N, 64, 32)) return -1;
  } else if (wide) {
    // gemm_wide_kernel: one box per warp (16 rows) and 64-column accumulator group (see WideCfg)
    const bool geglu = g.epi == EPI_GEGLU;
    if (make_tmap_2d(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.out, geglu ? g.N / 2 : g.N, g.M, g.ldo, geglu ? 32 : 64, 16,
                     geglu ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B))
      return -1;
  } else {
    if (make_tmap_2d(&tc, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.out, g.N, g.M, g.ldo, 64, 32)) return -1;
  }
  KArgs ka;
  ka.M = g.M; ka.N = g.N; ka.K = g.K;
  ka.bias = g.bias; ka.has_resid = g.resid != nullptr;
  ka.pos = g.pos; ka.rope_cos = g.rope_cos; ka.rope_sin = g.rope_sin; ka.rope_cols = g.rope_cols;
  ka.row_stats = g.row_stats;
  ka.pivot_out = g.pivot_out; ka.pivot_in = g.pivot_in; ka.pivot_in_stats = g.pivot_in_stats;
  ka.topk_idx = g.topk_idx; ka.topk_score = g.topk_score; ka.topk_valid = g.topk_valid; ka.topk_n = g.topk_n;
  ka.grouped = 0;
  // SRB_RESID_INTERLEAVE=0 restores the contiguous ranges for the residual GEMMs (A/B measurements); =2 interleaves
  // the fp32-residual GEMMs for every K (by default only K > 768, whose row block is too large to survive in L2)
  static const bool resid_interleave = [] { const char* e = getenv("SRB_RESID_INTERLEAVE"); return !(e && e[0] == '0'); }();
  static const int interleave_min_k = [] { const char* e = getenv("SRB_RESID_INTERLEAVE"); return (e && e[0] == '2') ? 0 : 768; }();
  ka.interleave = (((g.epi == EPI_RESID && g.resid != nullptr) || is_hl) && resid_interleave && (is_hl || g.K > interleave_min_k) &&
                   g.N / BN > 1) ? 1 : 0;
  ka.fold_stats = nullptr; ka.fold_eps = 0.f; ka.fold_inv_h = 0.f; ka.fold_parts = 0;
  ka.grp_rows = w_groups > 1 ? g.w_group_rows : 0;
  ka.bias_stride = (w_groups > 1 && g.bias_per_group) ? g.N : 0;
  CUtensorMap tx = tc;   // gemm_kernel's auxiliary map (EPI_RESID_HL: the low halves of the pair); unused otherwise
  if (is_hl && make_tmap_2d(&tx, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, g.lo16, g.N, g.M, g.N, 64, 32)) return -1;
  if (g.fold_stats) {
    if ((g.epi != EPI_ROPE && g.epi != EPI_GEGLU) || g.fold_h <= 0 || g.fold_h % 128 != 0) {
      fprintf(stderr, "[srb200] gemm_f16: LayerNorm fold belongs to EPI_ROPE / EPI_GEGLU with the row length\n");
      return -1;
    }
    ka.fold_stats = g.fold_stats; ka.fold_eps = g.fold_eps;
    ka.fold_inv_h = 1.0f / static_cast<float>(g.fold_h);
    ka.fold_parts = g.fold_h / 128;
  }
  int grid = 0;   // 0: the persistent grid of launch
  if (g.epi == EPI_TOPK) {
    if (!g.topk_idx || !g.topk_score || !g.topk_lists || g.N % 256 != 0) {
      fprintf(stderr, "[srb200] gemm_f16: EPI_TOPK needs list buffers and N %% 256 == 0\n");
      return -1;
    }
    // the query batch is the short dimension here, the stored rows stream as N; one list per worker and query row
    const int m_blocks = (g.M + BM - 1) / BM, n_blocks = g.N / BN;
    const long long tiles = static_cast<long long>(m_blocks) * n_blocks;
    // grouped schedule (tile_range): whole groups of m_blocks workers, each group at least one tile.
    // SRB_TOPK_GROUPED=0 restores the contiguous ranges (A/B measurements).
    static const bool grouped_on = [] { const char* e = getenv("SRB_TOPK_GROUPED"); return !(e && e[0] == '0'); }();
    const int groups = m_blocks > 0 ? num_sms / m_blocks : 0;
    if (grouped_on && m_blocks > 1 && groups >= 1 && n_blocks >= groups) {
      ka.grouped = 1;
      grid = groups * m_blocks;
    }
    *g.topk_lists = ka.grouped ? grid : static_cast<int>(tiles < num_sms ? tiles : num_sms);
  }
  return with_kernel(g.epi, cn, [&](auto kn) { return launch<decltype(kn)>(stream, ta, tb, tc, tx, ka, num_sms, grid); });
}

}  // namespace srb
