// Semantic-cache lookup: cosine scores of a query batch against a device-resident fp16 matrix of unit
// vectors, then per-query top-k with the reference tie rule.
//
// Replaces the Go scalar loop `embeddingDotProduct` + `scanLinearForSimilarity`
// (src/semantic-router/pkg/cache/inmemory_cache_search.go:14-20,65-89; first max wins) and
// the stable-sort top-k of `calculate_similarity_batch`
// (candle-binding/src/ffi/embedding.rs:1640-1681; lower index first on ties).
//
// v1 pipeline: scores[B, chunk] = Q . C^T on the wgmma GEMM (fp16 operands, fp32 accumulate, fp32 store;
// HBM-bound for small B, tensor-bound for B >= ~256), then a two-stage selection:
//   stage 1: one CTA per (query, 8192-score segment): each warp takes the top-k of its 1024 register-resident scores with
//            warp shuffles, warp 0 merges the eight lists
//   stage 2: one CTA per query: same selection over the segment winners.
#include "kernels.h"

#include <algorithm>
#include <initializer_list>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "gemm.h"

namespace srb {
namespace {

constexpr int kSelThreads = 256;
constexpr int kPerThread = 32;
constexpr int kSegment = kSelThreads * kPerThread;  // 8192 scores per stage-1 CTA

struct Cand {
  float v;
  int i;
};
// A launch gets 48 KB of shared memory without opting in, the kernel's static shared memory included.
constexpr size_t kDefaultSmem = 48 * 1024;
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) {
  // larger score wins; equal score: lower (non-negative) index wins; index -1 = nothing
  if (i < 0) return false;
  if (bi < 0) return true;
  return v > bv || (v == bv && i < bi);
}
__device__ __forceinline__ Cand warp_argmax(Cand c) {   // every lane ends up with the winner
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, c.v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, c.i, o);
    if (better(ov, oi, c.v, c.i)) { c.v = ov; c.i = oi; }
  }
  return c;
}
__device__ __forceinline__ Cand block_argmax(Cand c) {   // every thread ends up with the winner
  __shared__ Cand red[kSelThreads / 32];
  c = warp_argmax(c);
  const int warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane_id() == 0) red[warp] = c;
  __syncthreads();
  Cand b = red[0];
#pragma unroll
  for (int k = 1; k < kSelThreads / 32; ++k)
    if (better(red[k].v, red[k].i, b.v, b.i)) b = red[k];
  return b;
}

// k rounds of argmax over the n entries (v[t], i[t]) of a shared-memory list, each winner removed from the list; out(r, b)
// receives rank r's winner b (b.i -1: the list ran out).  warp_select: one warp, out called on lane 0; block_select: the
// whole CTA, out called on thread 0, every round ending on a barrier.
template <class Out>
__device__ __forceinline__ void warp_select(float* v, int* i, int n, int k, Out out) {
  const int lane = lane_id();
  for (int r = 0; r < k; ++r) {
    Cand c{-INFINITY, -1};
    int where = -1;
    for (int t = lane; t < n; t += 32)
      if (better(v[t], i[t], c.v, c.i)) { c.v = v[t]; c.i = i[t]; where = t; }
    const Cand b = warp_argmax(c);
    if (where >= 0 && b.i >= 0 && c.i == b.i) i[where] = -1;   // indices are unique: exactly one owner
    __syncwarp();
    if (lane == 0) out(r, b);
  }
}
template <class Out>
__device__ __forceinline__ void block_select(float* v, int* i, int n, int k, Out out) {
  for (int r = 0; r < k; ++r) {
    Cand c{-INFINITY, -1};
    int where = -1;
    for (int t = threadIdx.x; t < n; t += kSelThreads)
      if (better(v[t], i[t], c.v, c.i)) { c.v = v[t]; c.i = i[t]; where = t; }
    const Cand b = block_argmax(c);
    if (where >= 0 && c.i == b.i && b.i >= 0) i[where] = -1;   // indices are unique: exactly one owner
    if (threadIdx.x == 0) out(r, b);
    __syncthreads();
  }
}

// scores: [B, ld] fp32 for local rows [row0, row0 + n); out: cand_idx/cand_score [B, total_segments, k]
// One CTA per (query, 8192-score segment); each of its eight warps owns 1024 scores in registers (32 per lane).
// Exact top-k of a warp's 1024 scores without k full passes: the k-th largest of the 32 LANE MAXIMA is a lower bound L of
// the k-th largest score (at least k scores are >= L), so only scores >= L can be winners -- typically k..2k of them.
// They are compacted into a per-warp list (ballot + popc) and the k rounds of warp argmax run over that short list.
// A warp whose list would overflow (hundreds of tied scores) falls back to k passes over its registers.  Warp 0 then
// merges the eight lists.  (The first version -- k block-wide argmax rounds over all 8192 scores -- took 3.4x the time
// of the score GEMM it follows.)
constexpr int kListCap = 128;   // candidates per warp

// stage 1 of one (query, segment)
__device__ __forceinline__ void stage1_item(const float* __restrict__ scores, int ld, int n, int row0,
                                            const uint8_t* __restrict__ valid, int k, int seg0, int total_segments,
                                            int* __restrict__ cand_idx, float* __restrict__ cand_score, int q, int seg) {
  constexpr int kWarps = kSelThreads / 32;
  __shared__ float lv[kWarps][kListCap];
  __shared__ int li[kWarps][kListCap];
  __shared__ float wv[kWarps * 64];   // warp w's k winners at [w * k, (w + 1) * k): one list of kWarps * k for warp 0
  __shared__ int wi[kWarps * 64];
  const int warp = threadIdx.x >> 5, lane = lane_id();
  const int base = seg * kSegment + warp * (kSegment / kWarps);   // first local row of this warp's 1024 scores
  const float* s = scores + static_cast<size_t>(q) * ld + base;
  float v[kPerThread];
  float lm = -INFINITY;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    const int c = base + j * 32 + lane;  // coalesced
    const bool ok = c < n && (!valid || valid[row0 + c]);
    v[j] = ok ? s[j * 32 + lane] : -INFINITY;
    lm = fmaxf(lm, v[j]);
  }
  // rank of this lane's maximum among the 32 (ties by lane): the lane of rank min(k,32)-1 holds the bound L
  int rank = 0;
#pragma unroll
  for (int o = 0; o < 32; ++o) {
    const float ov = __shfl_sync(0xffffffffu, lm, o);
    rank += (ov > lm || (ov == lm && o < lane)) ? 1 : 0;
  }
  const int want = (k < 32 ? k : 32) - 1;
  const unsigned who = __ballot_sync(0xffffffffu, rank == want);
  float L = __shfl_sync(0xffffffffu, lm, __ffs(who) - 1);
  if (k > 32) L = -INFINITY;   // more winners than lanes: every finite score is a candidate
  // compact the candidates (score >= L, finite) into this warp's list
  int count = 0;
  const unsigned lt = (1u << lane) - 1u;
#pragma unroll
  for (int j = 0; j < kPerThread; ++j) {
    const bool cand = v[j] >= L && v[j] != -INFINITY;
    const unsigned m = __ballot_sync(0xffffffffu, cand);
    const int at = count + __popc(m & lt);
    if (cand && at < kListCap) { lv[warp][at] = v[j]; li[warp][at] = row0 + base + j * 32 + lane; }
    count += __popc(m);
  }
  __syncwarp();
  float* mv = wv + warp * k;
  int* mi = wi + warp * k;
  if (count <= kListCap) {
    warp_select(lv[warp], li[warp], count, k, [&](int r, Cand b) { mv[r] = b.i >= 0 ? b.v : -INFINITY; mi[r] = b.i; });
  } else {   // pathological ties: k passes over the registers
    uint32_t removed = 0;
    for (int r = 0; r < k; ++r) {
      Cand c{-INFINITY, -1};
      int cj = -1;
#pragma unroll
      for (int j = 0; j < kPerThread; ++j) {
        const bool live = !((removed >> j) & 1u) && v[j] != -INFINITY;
        const int idx = row0 + base + j * 32 + lane;
        if (live && better(v[j], idx, c.v, c.i)) { c.v = v[j]; c.i = idx; cj = j; }
      }
      const Cand b = warp_argmax(c);
      if (b.i >= 0 && b.i == c.i) removed |= 1u << cj;
      if (lane == 0) { mv[r] = b.i >= 0 ? b.v : -INFINITY; mi[r] = b.i; }
    }
  }
  __syncthreads();
  if (warp == 0) {
    int* oi = cand_idx + (static_cast<size_t>(q) * total_segments + seg0 + seg) * k;
    float* os = cand_score + (static_cast<size_t>(q) * total_segments + seg0 + seg) * k;
    warp_select(wv, wi, kWarps * k, k, [&](int r, Cand b) { oi[r] = b.i; os[r] = b.i >= 0 ? b.v : -INFINITY; });
  }
}

// one CTA per (query, segment): grid (segments of the chunk, B)
__global__ void __launch_bounds__(kSelThreads)
select_stage1(const float* __restrict__ scores, int ld, int n, int row0, const uint8_t* __restrict__ valid,
              int k, int seg0, int total_segments, int* __restrict__ cand_idx, float* __restrict__ cand_score) {
  stage1_item(scores, ld, n, row0, valid, k, seg0, total_segments, cand_idx, cand_score, blockIdx.y, blockIdx.x);
}

// The same over *nq queries, a number read on the device: the CTAs of a fixed grid stride over its (query, segment)
// pairs.  The exact scan's fallback, whose query count the host never learns.
__global__ void __launch_bounds__(kSelThreads)
select_stage1_counted(const float* __restrict__ scores, int ld, int n, int row0, const uint8_t* __restrict__ valid,
                      int k, int seg0, int total_segments, int* __restrict__ cand_idx, float* __restrict__ cand_score,
                      const int* __restrict__ nq) {
  const int nseg = (n + kSegment - 1) / kSegment, items = *nq * nseg;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    stage1_item(scores, ld, n, row0, valid, k, seg0, total_segments, cand_idx, cand_score, item / nseg, item % nseg);
    __syncthreads();   // warp 0 has read wv / wi before the next item rewrites them
  }
}

// ---- scores for a handful of queries (the reference's operating mode is ONE query per lookup): a GEMV, not a GEMM.
// HBM-bound by construction: every stored row is read once (D * 2 bytes), one warp per row, the queries sit in shared
// memory as fp32.  fp16 x fp16 products are exact in fp32, accumulation is fp32 in a fixed order (lane-strided chunks,
// then an xor-shuffle tree): deterministic.  The 128-row MMA tile would spend 127/128 of its work on padding here.
template <int NB>
__global__ void __launch_bounds__(256)
scores_small_kernel(const __half* __restrict__ queries, const __half* __restrict__ cache, int n, int D, int ld,
                    float* __restrict__ scores) {
  extern __shared__ float qs[];   // [NB][D]
  for (int i = threadIdx.x; i < NB * D; i += blockDim.x) qs[i] = __half2float(queries[i]);
  __syncthreads();
  const int lane = lane_id();
  const int warps = gridDim.x * (blockDim.x >> 5);
  const int chunks = D >> 3;   // 16-byte units per row
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < n; row += warps) {
    const uint4* r4 = reinterpret_cast<const uint4*>(cache + static_cast<size_t>(row) * D);
    float acc[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) acc[b] = 0.f;
    for (int c = lane; c < chunks; c += 32) {
      const uint4 u = __ldg(r4 + c);
      const float2 x0 = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
      const float2 x1 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
      const float2 x2 = __half22float2(*reinterpret_cast<const __half2*>(&u.z));
      const float2 x3 = __half22float2(*reinterpret_cast<const __half2*>(&u.w));
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 qa = *reinterpret_cast<const float4*>(qs + b * D + 8 * c);
        const float4 qb = *reinterpret_cast<const float4*>(qs + b * D + 8 * c + 4);
        float t = acc[b];
        t = fmaf(x0.x, qa.x, t); t = fmaf(x0.y, qa.y, t); t = fmaf(x1.x, qa.z, t); t = fmaf(x1.y, qa.w, t);
        t = fmaf(x2.x, qb.x, t); t = fmaf(x2.y, qb.y, t); t = fmaf(x3.x, qb.z, t); t = fmaf(x3.y, qb.w, t);
        acc[b] = t;
      }
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float t = warp_sum(acc[b]);
      if (lane == 0) scores[static_cast<size_t>(b) * ld + row] = t;
    }
  }
}

// per query: top-k over `ncand` candidates; writes global ids (local + id_offset)
__device__ __forceinline__ void stage2_item(const int* __restrict__ cand_idx, const float* __restrict__ cand_score,
                                            int ncand, int k, int id_offset, int* __restrict__ out_idx,
                                            float* __restrict__ out_score, int q) {
  extern __shared__ uint8_t dyn[];
  float* sv = reinterpret_cast<float*>(dyn);
  int* si = reinterpret_cast<int*>(sv + ncand);
  for (int c = threadIdx.x; c < ncand; c += kSelThreads) {
    sv[c] = cand_score[static_cast<size_t>(q) * ncand + c];
    si[c] = cand_idx[static_cast<size_t>(q) * ncand + c];
  }
  __syncthreads();
  block_select(sv, si, ncand, k, [&](int r, Cand b) {
    out_idx[static_cast<size_t>(q) * k + r] = b.i >= 0 ? b.i + id_offset : -1;
    out_score[static_cast<size_t>(q) * k + r] = b.i >= 0 ? b.v : -INFINITY;
  });
}

// one CTA per query
__global__ void __launch_bounds__(kSelThreads)
select_stage2(const int* __restrict__ cand_idx, const float* __restrict__ cand_score, int ncand, int k, int id_offset,
              int* __restrict__ out_idx, float* __restrict__ out_score) {
  stage2_item(cand_idx, cand_score, ncand, k, id_offset, out_idx, out_score, blockIdx.x);
}

// over *nq queries, read on the device, by a fixed grid (the exact scan's fallback, as select_stage1_counted); the last
// round's barrier of one query lets the next one's loads overwrite sv / si
__global__ void __launch_bounds__(kSelThreads)
select_stage2_counted(const int* __restrict__ cand_idx, const float* __restrict__ cand_score, int ncand, int k,
                      int id_offset, int* __restrict__ out_idx, float* __restrict__ out_score, const int* __restrict__ nq) {
  const int queries = *nq;
  for (int q = blockIdx.x; q < queries; q += gridDim.x)
    stage2_item(cand_idx, cand_score, ncand, k, id_offset, out_idx, out_score, q);
}

// Exchange format of a sharded cache (SURVEY 8e): one 8-byte entry per (query, rank) = {fp32 score, int32 GLOBAL id}.
// Each rank packs its [B,k] result into this form, ONE all-gather moves B * k * 8 bytes per rank, and the merge below
// reads the G gathered lists directly.
__global__ void pack_pairs_kernel(const int* __restrict__ idx, const float* __restrict__ score, int n, int2* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = make_int2(__float_as_int(score[i]), idx[i]);
}
// merge of G per-shard lists in the packed form: pairs [G][B][k]; global ids are unique across shards
__global__ void __launch_bounds__(kSelThreads)
merge_packed_kernel(const int2* __restrict__ pairs, int G, int B, int k, int* __restrict__ out_idx,
                    float* __restrict__ out_score) {
  extern __shared__ uint8_t dyn[];
  float* sv = reinterpret_cast<float*>(dyn);
  int* si = reinterpret_cast<int*>(sv + G * k);
  const int q = blockIdx.x;
  for (int c = threadIdx.x; c < G * k; c += kSelThreads) {
    const int g = c / k, j = c % k;
    const int2 e = pairs[(static_cast<size_t>(g) * B + q) * k + j];
    sv[c] = __int_as_float(e.x);
    si[c] = e.y;
  }
  __syncthreads();
  block_select(sv, si, G * k, k, [&](int r, Cand b) {
    out_idx[static_cast<size_t>(q) * k + r] = b.i;
    out_score[static_cast<size_t>(q) * k + r] = b.i >= 0 ? b.v : -INFINITY;
  });
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
int sm_count() { return std::max(1, device_sms()); }   // a launch takes at least one CTA

// static shared memory of a kernel, asked of the runtime once per kernel
int static_smem(const void* kernel, size_t* bytes) {
  static std::mutex mu;
  static std::unordered_map<const void*, size_t> known;
  std::lock_guard<std::mutex> lk(mu);
  auto it = known.find(kernel);
  if (it == known.end()) {
    cudaFuncAttributes a;
    SRB_CUDA_CHECK(cudaFuncGetAttributes(&a, kernel));
    it = known.emplace(kernel, a.sharedSizeBytes).first;
  }
  *bytes = it->second;
  return 0;
}

// Launches kernel<<<grid, block, smem, stream>>>(args...), checks it and counts it.  A kernel whose static and smem
// bytes of dynamic shared memory exceed 48 KB is opted in first (static shared memory alone never does).  Nothing here
// synchronises or allocates, so the launches of a scan can be captured into a CUDA graph.
template <typename... P, typename... A>
int launch(void (*kernel)(P...), dim3 grid, int block, size_t smem, cudaStream_t stream, A... args) {
  size_t fixed = 0;
  if (smem > 0 && static_smem(reinterpret_cast<const void*>(kernel), &fixed)) return -1;
  if (smem + fixed > kDefaultSmem)
    SRB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  kernel<<<grid, block, smem, stream>>>(args...);
  SRB_CUDA_CHECK(cudaGetLastError());
  note_launch();
  return 0;
}
inline int chunk_rows(int B, int N) {
  // keep the score buffer <= 1 GiB; multiple of the stage-1 segment
  size_t rows = (static_cast<size_t>(1) << 30) / (static_cast<size_t>(B > 0 ? B : 1) * 4);
  rows = rows / kSegment * kSegment;
  if (rows < static_cast<size_t>(kSegment)) rows = kSegment;
  const size_t need = align_up(static_cast<size_t>(N), kSegment);
  return static_cast<int>(rows < need ? rows : need);
}

// Workspace of the two-stage route, byte offsets: the score chunk [B, chunk_rows] at 0, then cand_idx and cand_score
// [B, candidates]
struct TwoStageLayout {
  size_t cand_idx = 0, cand_score = 0, total = 0;
};
TwoStageLayout two_stage_layout(const CachePlan& p, int B) {
  const size_t cands = align_up(static_cast<size_t>(B) * p.candidates * 4, 256);
  TwoStageLayout L;
  L.cand_idx = align_up(static_cast<size_t>(B) * p.chunk_rows * 4, 256);
  L.cand_score = L.cand_idx + cands;
  L.total = L.cand_score + cands;
  return L;
}

}  // namespace

constexpr int kFusedK = 8;        // list length of the GEMM's top-k epilogue (gemm.h EPI_TOPK)
constexpr int kFusedLists = 320;  // upper bound of the lists per query (= 2 x CTAs launched <= 2 x SMs)
constexpr int kMaxK = 64;         // stage 1 keeps 64 entries per warp (wv / wi)
constexpr size_t kStage2SmemMax = 200 * 1024;   // stage 2 holds every candidate of its query in shared memory

// The two-stage part of a plan (score chunks, segments, stage-2 candidates, workspace); false, with the route left
// refused, where stage 2 would hold more than kStage2SmemMax of candidates per query.
static bool plan_two_stage(CachePlan& p, int B, int N, int k) {
  p.chunk_rows = chunk_rows(B, N);
  p.chunks = (N + p.chunk_rows - 1) / p.chunk_rows;
  p.segments = (N + kSegment - 1) / kSegment;
  p.candidates = p.segments * k;
  p.stage2_smem = static_cast<size_t>(p.candidates) * 8;
  if (p.stage2_smem > kStage2SmemMax) return false;
  p.workspace_bytes = two_stage_layout(p, B).total;
  return true;
}

CachePlan cache_topk_plan(int B, int N, int D, int k) {
  CachePlan p;
  if (B <= 0 || k <= 0 || k > kMaxK || N < 0) return p;
  if (N == 0) {
    p.route = CACHE_EMPTY;
    return p;
  }
  if (B > 4 && k <= kFusedK && D % 8 == 0) {
    p.route = CACHE_FUSED;
    p.candidates = kFusedLists * kFusedK;
    p.workspace_bytes = 2 * align_up(static_cast<size_t>(B) * kFusedLists * kFusedK * 4, 256);
    return p;
  }
  if (!plan_two_stage(p, B, N, k)) return p;
  p.route = (B <= 4 && D % 8 == 0 && static_cast<size_t>(B) * D * 4 <= 48 * 1024) ? CACHE_GEMV : CACHE_GEMM;
  return p;
}

size_t cache_topk_workspace_bytes(int B, int N, int D, int k) { return cache_topk_plan(B, N, D, k).workspace_bytes; }

int cache_topk(cudaStream_t stream, const __half* queries, int B, const __half* cache, const uint8_t* valid, int N,
               int D, int k, int id_offset, int* out_idx, float* out_score, void* workspace, size_t workspace_bytes) {
  if (B <= 0 || k <= 0) return 0;
  const CachePlan plan = cache_topk_plan(B, N, D, k);
  if (plan.route == CACHE_REFUSED) {
    fprintf(stderr, "[srb200] cache_topk: k=%d over %d rows unsupported (k <= %d, ceil(rows / %d) * k <= %d)\n", k, N,
            kMaxK, kSegment, static_cast<int>(kStage2SmemMax / 8));
    return -1;
  }
  if (workspace_bytes < plan.workspace_bytes) {
    fprintf(stderr, "[srb200] cache_topk: workspace too small\n");
    return -1;
  }
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  if (plan.route == CACHE_EMPTY)
    return launch(select_stage2, B, kSelThreads, 0, stream, nullptr, nullptr, 0, k, id_offset, out_idx, out_score);
  if (plan.route == CACHE_FUSED) {
    // Scores never leave the SM: the GEMM's epilogue keeps a running top-8 per (query, CTA) and only those short lists
    // are written (B x <= 148 x 8 pairs); no 1 GiB score chunks, no selection pass over them.
    int* l_idx = reinterpret_cast<int*>(ws);
    float* l_score = reinterpret_cast<float*>(ws + align_up(static_cast<size_t>(B) * kFusedLists * kFusedK * 4, 256));
    int lists = 0;
    GemmDesc g;
    g.M = B; g.N = static_cast<int>(align_up(N, 256)); g.K = D; g.A = queries; g.W = cache;   // the store is padded to 256 rows
    g.epi = EPI_TOPK; g.topk_idx = l_idx; g.topk_score = l_score; g.topk_valid = valid; g.topk_n = N; g.topk_lists = &lists;
    // a CTA only writes the lists of the query rows it walked: every other slot must read "nothing" (idx -1)
    SRB_CUDA_CHECK(cudaMemsetAsync(l_idx, 0xFF, static_cast<size_t>(B) * kFusedLists * kFusedK * 4, stream));
    if (gemm_f16(stream, g)) return -1;
    if (lists <= 0 || lists > kFusedLists) { fprintf(stderr, "[srb200] cache_topk: %d lists\n", lists); return -1; }
    const int ncand = lists * kFusedK;
    return launch(select_stage2, B, kSelThreads, static_cast<size_t>(ncand) * 8, stream, l_idx, l_score, ncand, k,
                  id_offset, out_idx, out_score);
  }
  const int chunk = plan.chunk_rows, segs = plan.segments;
  const TwoStageLayout W = two_stage_layout(plan, B);
  float* scores = reinterpret_cast<float*>(ws);
  int* cand_idx = reinterpret_cast<int*>(ws + W.cand_idx);
  float* cand_score = reinterpret_cast<float*>(ws + W.cand_score);
  for (int row0 = 0; row0 < N; row0 += chunk) {
    const int n = (N - row0) < chunk ? (N - row0) : chunk;
    const int n_pad = static_cast<int>(align_up(n, 64));  // cache allocation is padded to 256 rows
    if (plan.route == CACHE_GEMV) {
      const int grid = sm_count() * 8;   // 8 CTAs x 8 warps per SM: enough loads in flight to cover the HBM latency
      const auto gemv = B == 1 ? scores_small_kernel<1> : B == 2 ? scores_small_kernel<2>
                      : B == 3 ? scores_small_kernel<3> : scores_small_kernel<4>;
      if (launch(gemv, grid, 256, static_cast<size_t>(B) * D * 4, stream, queries, cache + static_cast<size_t>(row0) * D,
                 n, D, chunk, scores))
        return -1;
    } else {
      GemmDesc g;
      g.M = B; g.N = n_pad; g.K = D; g.A = queries; g.W = cache + static_cast<size_t>(row0) * D;
      g.out = scores; g.ldo = chunk; g.epi = EPI_RESID; g.resid = nullptr; g.ldr = chunk;
      if (gemm_f16(stream, g)) return -1;
    }
    if (launch(select_stage1, dim3((n + kSegment - 1) / kSegment, B), kSelThreads, 0, stream, scores, chunk, n, row0,
               valid, k, row0 / kSegment, segs, cand_idx, cand_score))
      return -1;
  }
  return launch(select_stage2, B, kSelThreads, plan.stage2_smem, stream, cand_idx, cand_score, plan.candidates, k,
                id_offset, out_idx, out_score);
}

int cache_pack_pairs(cudaStream_t stream, const int* idx, const float* score, int n, void* pairs_out) {
  if (n <= 0) return 0;
  return launch(pack_pairs_kernel, (n + 255) / 256, 256, 0, stream, idx, score, n, static_cast<int2*>(pairs_out));
}

int cache_merge_packed(cudaStream_t stream, const void* pairs, int G, int B, int k, int* out_idx, float* out_score) {
  if (B <= 0) return 0;
  const size_t smem = static_cast<size_t>(G) * k * 8;
  if (smem > kDefaultSmem) { fprintf(stderr, "[srb200] cache_merge_packed: G * k = %d too large\n", G * k); return -1; }
  return launch(merge_packed_kernel, B, kSelThreads, smem, stream, static_cast<const int2*>(pairs), G, B, k, out_idx,
                out_score);
}

// ---- exact caches (sr_cache_create_exact): the scores of the reference's embeddingDotProduct on the fp32 rows and query
// (pkg/cache/inmemory_cache_search.go:14-20: dot = 0; dot += q[i] * c[i] in index order), bit for bit.
//
// The fp16 scan above stays the filter.  It returns k' >= k candidates per query by their fp16-operand score s16.  With
// eps >= |s16 - s_go| for every row (s_go the Go score), any row with s16 < s16_(k) - 2 eps has s_go < s16_(k) - eps <=
// s_go(t) for each of the k rows t of the fp16 top-k, so it is not in the exact top-k.  The band {s16 >= s16_(k) - 2 eps}
// therefore holds the exact top-k, and the candidate list holds the whole band when it holds every valid row (it ends in
// -1) or when its last score is strictly below s16_(k) - 2 eps.  Such a query is certified: its band is rescored in Go
// order and ordered by (score descending, index ascending).  Every other query falls back to an exhaustive exact scan.
//
// eps, for a query q and any stored row r, with Q = |q|_2, R >= |r|_2 for every row (the cache keeps the maximum of its
// rows), S = sqrt(D), and u = 2^-24 the unit roundoff of fp32:
//  1. fp16 operands.  fp16(x) = x + a with |a| <= d |x| + h, d = 2^-11 (normal range) and h = 2^-25 (half the subnormal
//     spacing), for |x| <= 65504 (larger or non-finite components are refused at the door).  Then
//     |q~ r~ - q r| <= |q| |b| + |r| |a| + |a| |b| <= (2d + d^2) |q r| + h (1 + d) (|q| + |r|) + h^2 per component, and by
//     Cauchy-Schwarz the sum is at most E1 = (2d + d^2) Q R + h (1 + d) S (Q + R) + D h^2.
//  2. The scan's fp32 sum of the exact products q~_i r~_i (11 x 11 significant bits fit in fp32, and the smallest product
//     2^-48 is a normal fp32 number).  Whatever the order -- wgmma's accumulation, the GEMV's fmaf chains and shuffle tree --
//     each partial sum is one of at most D additions, so with a rounding error per addition of at most u' = 8 u relative
//     (round-to-nearest gives u; 8 u leaves room for truncation and the tensor cores' alignment of their addends) the error
//     is at most E2 = g'_D sum |q~_i r~_i| <= g'_D ((1 + d)^2 Q R + h (1 + d) S (Q + R) + D h^2), g'_D = D u' / (1 - D u').
//  3. Go's own sum: D roundings of either rule (a product and an addition each, or one fma each) give
//     E3 = g_D sum |q_i r_i| <= g_D Q R, g_D = D u / (1 - D u).
//  4. Underflow: every rounding may also lose up to 2^-150 absolute; 2 D of them at 2^-149 each give E4 = 2 D 2^-149.
// eps = (E1 + E2 + E3 + E4) (1 + 2^-20), the last factor covering the float64 evaluation of eps and of Q.
// (oracle/cache_exact_oracle.py exact_eps restates it; tests/test_cache_exact_oracle.py checks it on adversarial rows.)
__host__ __device__ inline double exact_eps(double Q, double R, int D) {
  const double d = 1.0 / 2048, h = 1.0 / 33554432.0, u = 1.0 / 16777216.0, S = sqrt(static_cast<double>(D));
  const double g = D * u / (1 - D * u), g8 = D * 8 * u / (1 - D * 8 * u);
  const double cross = h * (1 + d) * S * (Q + R) + D * h * h;
  const double e1 = (2 * d + d * d) * Q * R + cross;
  const double e2 = g8 * ((1 + d) * (1 + d) * Q * R + cross);
  const double e3 = g * Q * R;
  const double e4 = 2.0 * D * 0x1p-149;
  return (e1 + e2 + e3 + e4) * (1 + 0x1p-20);
}

namespace {

constexpr int kExactCand = 64;   // the most candidates a query's band may hold (one thread each in exact_band_kernel)

// one Go-order term: rule 0 rounds the product, then the sum (Go amd64 v1); rule 1 is one fused multiply-add (Go arm64,
// amd64 v3).  Explicit intrinsics: nvcc would contract `acc + a * b` into an fma and turn rule 0 into rule 1.
template <int kRule>
__device__ __forceinline__ float go_term(float acc, float a, float b) {
  return kRule == 0 ? __fadd_rn(acc, __fmul_rn(a, b)) : __fmaf_rn(a, b, acc);
}

// What the bound eps covers (and sr_cache_topk checks on the host): a finite component of magnitude <= 65504, which
// rounds to a finite fp16 value.  NaN fails the comparison too.
__device__ __forceinline__ bool exact_in_range(float x) { return fabsf(x) <= 65504.f; }

// The fp16 copy of the queries that feeds the candidate scan, one CTA per query: round to nearest, as cast_rows_f16; a
// query with a component out of range is written as zeros instead, so that no NaN reaches the candidate selection
// (exact_band_kernel refuses that query).
__global__ void __launch_bounds__(256)
exact_query_f16_kernel(const float* __restrict__ queries, int D, __half* __restrict__ out) {
  const float* x = queries + static_cast<size_t>(blockIdx.x) * D;
  __half* y = out + static_cast<size_t>(blockIdx.x) * D;
  bool bad = false;
  for (int i = threadIdx.x; i < D; i += blockDim.x) bad |= !exact_in_range(x[i]);
  bad = __syncthreads_or(bad);
  for (int i = threadIdx.x; i < D; i += blockDim.x) y[i] = __float2half_rn(bad ? 0.f : x[i]);
}

// One CTA per query, one thread per candidate.  Certifies the band (see above); a certified query's band members are
// rescored in Go order from the fp32 row and fp32 query, ranked, and its k results written; any other query is appended
// to the fallback list and left to exact_scores_kernel.  A query with a component out of range is refused: its k results
// are (-1, -inf) and it never reaches the fallback.  path / band / eps: the test hook's record of the query (path 0
// certified, 1 fallback, 2 refused with band and eps 0).
template <int kRule>
__global__ void __launch_bounds__(kExactCand)
exact_band_kernel(const float* __restrict__ queries, const float* __restrict__ rows32, int D, double rmax,
                  const int* __restrict__ cand_idx, const float* __restrict__ cand_score, int kc, int k, int id_offset,
                  int* __restrict__ out_idx, float* __restrict__ out_score, int* __restrict__ fb_list,
                  int* __restrict__ fb_count, int* __restrict__ path, int* __restrict__ band, double* __restrict__ eps) {
  extern __shared__ float qs[];   // [D]
  __shared__ double red[kExactCand / 32];
  __shared__ float sv[kExactCand];
  __shared__ int si[kExactCand];
  __shared__ int order[kExactCand];
  const int q = blockIdx.x, t = threadIdx.x;
  double ss = 0;
  bool bad = false;
  for (int i = t; i < D; i += kExactCand) {
    const float x = queries[static_cast<size_t>(q) * D + i];
    qs[i] = x;
    ss += static_cast<double>(x) * x;
    bad |= !exact_in_range(x);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane_id() == 0) red[t >> 5] = ss;
  order[t] = -1;
  if (__syncthreads_or(bad)) {
    if (t == 0) { path[q] = 2; band[q] = 0; eps[q] = 0; }
    if (t < k) {
      out_idx[static_cast<size_t>(q) * k + t] = -1;
      out_score[static_cast<size_t>(q) * k + t] = -INFINITY;
    }
    return;
  }
  const double e = exact_eps(sqrt(red[0] + red[1]), rmax, D);
  const int* ci = cand_idx + static_cast<size_t>(q) * kc;
  const float* cs = cand_score + static_cast<size_t>(q) * kc;
  const bool all_rows = ci[k - 1] < 0 || ci[kc - 1] < 0;          // fewer than k' valid rows: every one is listed
  const double thr = ci[k - 1] < 0 ? -INFINITY : static_cast<double>(cs[k - 1]) - 2 * e;
  const bool certified = all_rows || static_cast<double>(cs[kc - 1]) < thr;
  const int mine = t < kc && ci[t] >= 0 && static_cast<double>(cs[t]) >= thr ? ci[t] : -1;
  const int members = __syncthreads_count(mine >= 0);
  if (t == 0) { path[q] = certified ? 0 : 1; band[q] = members; eps[q] = e; }
  if (!certified) {
    if (t == 0) fb_list[atomicAdd(fb_count, 1)] = q;
    return;
  }
  float s = -INFINITY;
  if (mine >= 0) {
    const float4* r4 = reinterpret_cast<const float4*>(rows32 + static_cast<size_t>(mine) * D);
    s = 0.f;
    for (int c = 0; c < D / 4; ++c) {
      const float4 r = __ldg(r4 + c);
      s = go_term<kRule>(s, qs[4 * c], r.x);
      s = go_term<kRule>(s, qs[4 * c + 1], r.y);
      s = go_term<kRule>(s, qs[4 * c + 2], r.z);
      s = go_term<kRule>(s, qs[4 * c + 3], r.w);
    }
  }
  sv[t] = s;
  si[t] = mine;
  __syncthreads();
  if (mine >= 0) {
    int rank = 0;
    for (int j = 0; j < kExactCand; ++j) rank += better(sv[j], si[j], s, mine) ? 1 : 0;
    if (rank < k) order[rank] = t;
  }
  __syncthreads();
  if (t < k) {
    const int w = order[t];
    out_idx[static_cast<size_t>(q) * k + t] = w >= 0 ? si[w] + id_offset : -1;
    out_score[static_cast<size_t>(q) * k + t] = w >= 0 ? sv[w] : -INFINITY;
  }
}

// Exhaustive Go-order scores of the fallback queries: scores[j, row] for the *fb_count queries listed in fb_list (rows of
// `queries`) against rows [0, n) of rows32.  A register-tiled SIMT product, 32 queries x 128 rows per tile, 4 x 4 per
// thread; every accumulator takes its D terms one at a time in index order (the K loop is never split), which is the
// Go sum.  The count stays on the device: a fixed grid strides over the tiles it implies, so with no fallback every CTA
// reads the count and exits.
constexpr int kXq = 32, kXr = 128, kXk = 8;
template <int kRule>
__global__ void __launch_bounds__(256)
exact_scores_kernel(const float* __restrict__ queries, const int* __restrict__ fb_list, const int* __restrict__ fb_count,
                    const float* __restrict__ rows32, int n, int D, int ld, float* __restrict__ scores) {
  __shared__ float qs[kXk][kXq];
  __shared__ float rs[kXk][kXr + 4];
  const int nq = *fb_count;
  const int rtiles = (n + kXr - 1) / kXr, tiles = (nq + kXq - 1) / kXq * rtiles;
  const int tq = threadIdx.x >> 5, tr = threadIdx.x & 31;    // queries q0 + tq * 4 + i, rows r0 + tr + 32 j
  const int lq = threadIdx.x >> 3, lk = threadIdx.x & 7;     // loaders: thread -> (query, k), and (row, k half)
  const int lr = threadIdx.x >> 1, lh = (threadIdx.x & 1) * 4;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int q0 = tile / rtiles * kXq, r0 = tile % rtiles * kXr;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const float* qrow = (q0 + lq < nq) ? queries + static_cast<size_t>(fb_list[q0 + lq]) * D : nullptr;
    const float* rrow = (r0 + lr < n) ? rows32 + static_cast<size_t>(r0 + lr) * D : nullptr;
    for (int k0 = 0; k0 < D; k0 += kXk) {   // ends on a barrier: the next tile's loads find qs / rs read
      qs[lk][lq] = qrow ? qrow[k0 + lk] : 0.f;
      const float4 r = rrow ? __ldg(reinterpret_cast<const float4*>(rrow + k0 + lh)) : make_float4(0.f, 0.f, 0.f, 0.f);
      rs[lh][lr] = r.x; rs[lh + 1][lr] = r.y; rs[lh + 2][lr] = r.z; rs[lh + 3][lr] = r.w;
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < kXk; ++kk) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = qs[kk][tq * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = rs[kk][tr + 32 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = go_term<kRule>(acc[i][j], a[i], b[j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int qq = q0 + tq * 4 + i;
      if (qq >= nq) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int rr = r0 + tr + 32 * j;
        if (rr < n) scores[static_cast<size_t>(qq) * ld + rr] = acc[i][j];
      }
    }
  }
}

// results of the compacted fallback queries back to their rows (a fixed grid striding over the device's count)
__global__ void exact_scatter_kernel(const int* __restrict__ fb_list, const int* __restrict__ fb_count, int k,
                                     const int* __restrict__ idx, const float* __restrict__ score, int* __restrict__ out_idx,
                                     float* __restrict__ out_score) {
  const int nq = *fb_count;
  for (int j = blockIdx.x; j < nq; j += gridDim.x) {
    const int q = fb_list[j];
    for (int r = threadIdx.x; r < k; r += blockDim.x) {
      out_idx[static_cast<size_t>(q) * k + r] = idx[static_cast<size_t>(j) * k + r];
      out_score[static_cast<size_t>(q) * k + r] = score[static_cast<size_t>(j) * k + r];
    }
  }
}

// CTAs of `kernel` that fit on the device at once (no dynamic shared memory): the fixed grid of the fallback's launches
template <typename Kernel>
int one_wave(Kernel kernel, int threads) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * sm_count();
}

// Workspace of cache_topk_exact: the candidate scan's (reused by the fallback's score chunks and selection), then the
// candidates, the fallback list and the fallback results.
struct ExactLayout {
  int kc = 0;               // candidates per query
  CachePlan scan, fallback;
  size_t cand_idx = 0, cand_score = 0, fb_list = 0, fb_idx = 0, fb_score = 0, total = 0;
};
ExactLayout exact_layout(int B, int N, int D, int k) {
  ExactLayout L;
  if (B <= 0 || k <= 0 || k > kMaxK || N < 0 || D % 8 != 0) return L;
  if (N > 0 && !plan_two_stage(L.fallback, B, N, k)) return L;
  // k' = 32 for k <= 32 and 64 above, where the two-stage plan takes it, else fewer; k' = k always fits when the
  // fallback's selection does.  Not the fused route: its 8 per list are too few to certify a band at k = 8.  Not 64 for
  // small k: stage 1 has no lane-maximum bound above k = 32 and makes 64 passes over every warp's scores, which made the
  // candidate scan of BASELINE cfg 4 at b 1024 take 128 ms against 3.7 ms for the default cache's fused route (H100 80GB
  // HBM3, 700 W).
  for (int kc : {k <= 32 ? 32 : kExactCand, 16, k}) {
    if (kc < k) continue;
    L.scan = cache_topk_plan(B, N, D, kc);
    if (L.scan.route != CACHE_REFUSED) { L.kc = kc; break; }
  }
  if (L.kc == 0) return L;
  size_t off = std::max(L.scan.workspace_bytes, N > 0 ? L.fallback.workspace_bytes : 0);
  auto take = [&](size_t bytes) { const size_t at = off; off = align_up(off + bytes, 256); return at; };
  off = align_up(off, 256);
  L.cand_idx = take(static_cast<size_t>(B) * L.kc * 4);
  L.cand_score = take(static_cast<size_t>(B) * L.kc * 4);
  L.fb_list = take(static_cast<size_t>(B + 1) * 4);   // [0] count, then the queries
  L.fb_idx = take(static_cast<size_t>(B) * k * 4);
  L.fb_score = take(static_cast<size_t>(B) * k * 4);
  L.total = off;
  return L;
}

}  // namespace

int cache_exact_candidates(int B, int N, int D, int k) { return exact_layout(B, N, D, k).kc; }
size_t cache_topk_exact_workspace_bytes(int B, int N, int D, int k) { return exact_layout(B, N, D, k).total; }
const int* cache_exact_fallback_count(const void* workspace, int B, int N, int D, int k) {
  const ExactLayout L = exact_layout(B, N, D, k);
  return L.kc ? reinterpret_cast<const int*>(static_cast<const uint8_t*>(workspace) + L.fb_list) : nullptr;
}

int cache_topk_exact(cudaStream_t stream, const float* queries32, __half* queries16, int B, const __half* cache,
                     const float* cache32, const uint8_t* valid, int N, int D, double rmax, int k, int sum_rule,
                     int id_offset, int* out_idx, float* out_score, void* workspace, size_t workspace_bytes, int* path,
                     int* band, double* eps) {
  if (B <= 0 || k <= 0) return 0;
  const ExactLayout L = exact_layout(B, N, D, k);
  if (L.kc == 0 || (sum_rule != 0 && sum_rule != 1)) {
    fprintf(stderr, "[srb200] cache_topk_exact: k=%d over %d rows unsupported (k <= %d, ceil(rows / %d) * k <= %d)\n", k,
            N, kMaxK, kSegment, static_cast<int>(kStage2SmemMax / 8));
    return -1;
  }
  if (workspace_bytes < L.total) {
    fprintf(stderr, "[srb200] cache_topk_exact: workspace too small\n");
    return -1;
  }
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  int* cand_idx = reinterpret_cast<int*>(ws + L.cand_idx);
  float* cand_score = reinterpret_cast<float*>(ws + L.cand_score);
  int* fb_count = reinterpret_cast<int*>(ws + L.fb_list);
  int* fb_list = fb_count + 1;
  if (launch(exact_query_f16_kernel, B, 256, 0, stream, queries32, D, queries16) ||
      cache_topk(stream, queries16, B, cache, valid, N, D, L.kc, 0, cand_idx, cand_score, ws, L.scan.workspace_bytes))
    return -1;
  SRB_CUDA_CHECK(cudaMemsetAsync(fb_count, 0, 4, stream));
  if (launch(sum_rule == 0 ? exact_band_kernel<0> : exact_band_kernel<1>, B, kExactCand, static_cast<size_t>(D) * 4,
             stream, queries32, cache32, D, rmax, cand_idx, cand_score, L.kc, k, id_offset, out_idx, out_score, fb_list,
             fb_count, path, band, eps))
    return -1;
  if (N == 0) return 0;   // every query of an empty store is certified
  // Exhaustive exact scan of the fallback queries only: Go-order scores in chunks, then the two-stage selection of
  // cache_topk over them, then the results back to their query rows.  The number of fallback queries stays on the device
  // (nothing waits for it on the host, so the scan can be captured into a CUDA graph): every launch below has a fixed grid
  // of about one wave whose CTAs stride over the work that number implies, and with no fallback each is one short wave
  // of early exits.
  static const int scores_grid[2] = {one_wave(exact_scores_kernel<0>, 256), one_wave(exact_scores_kernel<1>, 256)};
  static const int stage1_grid = one_wave(select_stage1_counted, kSelThreads);
  const CachePlan& P = L.fallback;
  const int chunk = P.chunk_rows;
  const TwoStageLayout W = two_stage_layout(P, B);
  float* scores = reinterpret_cast<float*>(ws);
  int* sel_idx = reinterpret_cast<int*>(ws + W.cand_idx);
  float* sel_score = reinterpret_cast<float*>(ws + W.cand_score);
  int* fb_idx = reinterpret_cast<int*>(ws + L.fb_idx);
  float* fb_score = reinterpret_cast<float*>(ws + L.fb_score);
  for (int row0 = 0; row0 < N; row0 += chunk) {
    const int n = (N - row0) < chunk ? (N - row0) : chunk;
    if (launch(sum_rule == 0 ? exact_scores_kernel<0> : exact_scores_kernel<1>, scores_grid[sum_rule], 256, 0, stream,
               queries32, fb_list, fb_count, cache32 + static_cast<size_t>(row0) * D, n, D, chunk, scores) ||
        launch(select_stage1_counted, stage1_grid, kSelThreads, 0, stream, scores, chunk, n, row0, valid, k,
               row0 / kSegment, P.segments, sel_idx, sel_score, fb_count))
      return -1;
  }
  if (launch(select_stage2_counted, sm_count(), kSelThreads, P.stage2_smem, stream, sel_idx, sel_score, P.candidates, k,
             id_offset, fb_idx, fb_score, fb_count))
    return -1;
  return launch(exact_scatter_kernel, sm_count(), 64, 0, stream, fb_list, fb_count, k, fb_idx, fb_score, out_idx,
                out_score);
}

}  // namespace srb
