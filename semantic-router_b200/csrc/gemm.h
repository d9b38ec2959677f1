// Host interface of the wgmma GEMM (see gemm_wgmma.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace srb {

enum GemmEpilogue {
  EPI_F16 = 0,    // out fp16 [M,N] = acc (+bias)
  EPI_ROPE = 1,   // out fp16 [M,N]; columns < rope_cols are 64-wide heads rotated by pos[row] (rotate-half)
  EPI_RESID = 2,  // out fp32 [M,N] = resid + acc (+bias)   (out may alias resid; resid == null => plain fp32 store)
  EPI_GEGLU = 3,  // out fp16 [M,N/2] = gelu_erf(a) * b, W rows pre-interleaved in 32-row (a|b) groups
  EPI_GELU = 4,   // out fp16 [M,N] = gelu_erf(acc + bias)
  EPI_TOPK = 5,   // no matrix output: every A row keeps the running top-8 of its accumulator row (cache scan)
  // The residual stream as an fp16 PAIR, in place: with x - pivot = hi + lo (hi = fp16(x - pivot), lo = fp16 of the rest),
  // out (hi) and lo16 [M,N] fp16 are read, updated to (x - pivot) + acc (+bias) re-centred on the new pivot, and written
  // back, together with the row statistics of the LayerNorm fold.  hi IS the raw fp16 copy the next projection
  // multiplies, so the residual GEMM moves 4 + 4 bytes per element; the pair carries 22 significant bits of
  // x - pivot.  row_stats and pivot_out are required.
  EPI_RESID_HL = 6,
};

struct GemmDesc {
  int M = 0, N = 0, K = 0;
  const void* A = nullptr;  // fp16 [a_rows >= M, K] row-major
  int a_rows = 0;           // rows addressable behind A (0 => M)
  const void* W = nullptr;  // fp16 [N, K] row-major (nn.Linear weight)
  void* out = nullptr;
  int ldo = 0;
  GemmEpilogue epi = EPI_F16;
  const float* bias = nullptr;   // fp32 [N] or null (bias_per_group: [w_groups * N])
  const float* resid = nullptr;  // fp32 [M, ldr] (EPI_RESID)
  int ldr = 0;
  const int* pos = nullptr;      // int32 [M] (EPI_ROPE)
  const float* rope_cos = nullptr;  // fp32 [max_pos, 32]
  const float* rope_sin = nullptr;
  int rope_cols = 0;
  // ---- LayerNorm folded into the GEMMs around it (pre-LN models): LN(x) W^T = rstd * (x - mean 1) (W diag(gamma))^T
  // = rstd * x W''^T with W'' = W diag(gamma) re-centred so that every row sums to zero (the centring matrix commutes
  // into the weights).  The residual GEMM that finishes x (EPI_RESID_HL) leaves the fp16 pair, whose high half is the
  // fp16 copy of x, and the per-row (sum, sum of squares); the consuming projection (EPI_ROPE / EPI_GEGLU) multiplies
  // the RAW fp16 rows with W'' and scales by the row's rstd in its epilogue.  No LayerNorm pass, no mean subtraction.
  // Statistics are kept as PARTIALS over fixed 128-column slices, [N/128][M][2] fp32, each written exactly once and
  // summed by the consumer in slice order: bitwise reproducible whatever the tile shape, schedule or batch
  // composition (atomics would make the result depend on arrival order).
  // ---- EPI_TOPK (semantic-cache scan): A = queries [M, K], W = stored rows [N, K]; the scores never leave the SM.
  // Each epilogue thread owns one query row and keeps the best kTopK = 8 (score, column) pairs of the columns its CTA
  // walks (strict >, columns visited in increasing order: the lower index wins ties inside a list); lists go to
  // topk_idx / topk_score [M][lists][8] (lists = workers launched, returned in *topk_lists; unused slots idx -1) and
  // are merged per query afterwards.  topk_valid (bytes, null: all valid) masks stored rows; columns >= topk_n are
  // padding.
  int* topk_idx = nullptr;
  float* topk_score = nullptr;
  const uint8_t* topk_valid = nullptr;
  int topk_n = 0;
  int* topk_lists = nullptr;        // host out
  float* row_stats = nullptr;       // EPI_RESID_HL: fp32 [N/128][M][2] (sum, sum of squares) per 128-column slice
  void* lo16 = nullptr;             // EPI_RESID_HL: fp16 [M, N] low halves (ld = N); `out` holds the high halves (ldo = N)
  // Row pivot: LayerNorm is shift-invariant and the zero-sum rows of W'' cancel any per-row constant, so the pair
  // and the statistics are taken of x - pivot_r, with pivot_r = the row's mean after the PREVIOUS residual GEMM (read
  // from that GEMM's statistics).  Rounding x - pivot instead of x keeps the fold exact-ish for rows whose common
  // offset dwarfs their spread (fp16(x) alone would lose (x - mean) there); variances are also better conditioned.
  // gemm_f16 refuses row_stats and pivots on every other epilogue.
  float* pivot_out = nullptr;          // EPI_RESID_HL: fp32 [M], this GEMM's pivots (written next to row_stats)
  const float* pivot_in = nullptr;     // EPI_RESID_HL: fp32 [M] pivots of the previous residual GEMM (null: pivot 0)
  const float* pivot_in_stats = nullptr;  // its statistics partials [N/128][M][2]
  const float* fold_stats = nullptr;   // EPI_ROPE / EPI_GEGLU: fp32 [fold_h/128][M][2] partials of the A rows
  float fold_eps = 0.f;
  int fold_h = 0;                      // row length the statistics were taken over
  // ---- grouped weights: W = w_groups matrices [N, K] stacked along N; rows [g * w_group_rows, (g + 1) * w_group_rows) of A are
  // multiplied with matrix g (w_group_rows a multiple of 128, the row-block height: a row block never straddles two
  // groups; gemm_f16 refuses anything else).  One launch serves
  // several tasks' weights (engine.h: Grouped).
  int w_groups = 0, w_group_rows = 0;
  // with w_groups > 1: `bias` holds one [N] vector per matrix, stacked like them, and the rows of group g add bias + g * N
  // (otherwise every group adds the one [N] bias)
  bool bias_per_group = false;
};

int gemm_f16(cudaStream_t stream, const GemmDesc& g);
// Thread-block cluster size gemm_f16 launches for a GEMM: that many CTAs, on neighbouring column tiles of one row block,
// share each A k-block (1: no clusters).
int gemm_cluster_size(int epi, int N, int K);
// Workers of its persistent grid: co-resident clusters of that shape on the current device (SMs without clusters).
int gemm_cluster_workers(int epi, int N, int K);
int make_tmap_f16_kmajor(CUtensorMap* out, const void* ptr, uint64_t rows, uint64_t k, uint32_t box_rows);

}  // namespace srb
