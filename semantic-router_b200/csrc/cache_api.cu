// sr_cache_* : device-resident semantic cache (include/sr_b200.h).  Mirrors the in-memory backend's lookup
// (src/semantic-router/pkg/cache/inmemory_cache.go:192-234, inmemory_cache_search.go:65-89):
// entries are appended, may be invalidated (expired / evicted), and are scanned exhaustively.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/sr_b200.h"
#include "common.cuh"
#include "kernels.h"

using namespace srb;

namespace {
struct RowStore {   // one row per stored entry, row_bytes each
  uint8_t* base;
  size_t row_bytes;
  uint8_t* row(size_t r) const { return base + r * row_bytes; }
};
}  // namespace

struct sr_cache {
  int device = 0, capacity = 0, cap_pad = 0, dim = 0, id_offset = 0, size = 0;
  __half* rows = nullptr;
  // every store of row data: the fp16 rows, then an exact cache's fp32 rows; moving or compacting rows moves them in each
  std::vector<RowStore> stores;
  uint8_t* valid = nullptr;
  void* ws = nullptr;
  size_t ws_bytes = 0;
  __half* d_q = nullptr;
  float* d_q32 = nullptr;   // fp32 staging for host queries (rounded to fp16 on the device)
  int* d_idx = nullptr;
  float* d_score = nullptr;
  int q_cap = 0, res_cap = 0;
  cudaStream_t stream = nullptr;
  std::mutex mu;
  // exact caches (sr_cache_create_exact): the rows as passed to sr_cache_add, bit for bit, beside the fp16 copy the scan
  // reads; the largest L2 norm any row ever added had (removing rows leaves it an upper bound); the record of the last
  // scan per query (sr_test_cache_exact_stats), its fallback count left on the device where the scan keeps it
  bool exact = false;
  int sum_rule = 0;
  float* rows32 = nullptr;
  double rmax = 0;
  int* d_path = nullptr;
  int* d_band = nullptr;
  double* d_eps = nullptr;
  int last_b = 0, last_kc = 0;
  const int* last_fallback = nullptr;
};

namespace {
int cfail(const char* msg) {
  fprintf(stderr, "[srb200] %s\n", msg);
  return -1;
}
// What the exact scan's bound covers (cache_scan.cu): finite components that round to a finite fp16 value.  Returns the
// largest L2 norm of the n rows of dim values, or -1 when a component falls outside.
double checked_max_norm(const float* x, size_t n, int dim) {
  double best = 0;
  for (size_t r = 0; r < n; ++r) {
    double ss = 0;
    for (int i = 0; i < dim; ++i) {
      const float v = x[r * dim + i];
      if (!(std::fabs(v) <= 65504.f)) return -1;   // NaN fails the comparison too
      ss += static_cast<double>(v) * v;
    }
    best = std::max(best, std::sqrt(ss));
  }
  return best;
}
// Frees p and allocates it anew at `bytes`; false, with p null, when that fails
template <typename T>
bool regrow(T*& p, size_t bytes) {
  if (p) cudaFree(p);
  p = nullptr;
  if (cudaMalloc(reinterpret_cast<void**>(&p), bytes) == cudaSuccess) return true;
  p = nullptr;
  return false;
}
// Grows the per-cache scratch.  Caller holds c->mu.  Buffers may still be referenced by work queued on the cache's
// stream or on a caller's stream (sr_cache_topk_dev), so everything on the device drains before anything is freed.
int ensure(sr_cache* c, int b, int k) {
  const int n = c->size > 0 ? c->size : 1;
  const size_t need = c->exact ? cache_topk_exact_workspace_bytes(b, n, c->dim, k) : cache_topk_workspace_bytes(b, n, c->dim, k);
  if (b > c->q_cap || b * k > c->res_cap || need > c->ws_bytes) cudaDeviceSynchronize();
  const size_t nb = static_cast<size_t>(b);
  if (b > c->q_cap) {
    c->q_cap = 0;
    if (!regrow(c->d_q, nb * c->dim * 2) || !regrow(c->d_q32, nb * c->dim * 4) ||
        (c->exact && (!regrow(c->d_path, nb * 4) || !regrow(c->d_band, nb * 4) || !regrow(c->d_eps, nb * 8))))
      return -1;
    c->q_cap = b;
  }
  if (b * k > c->res_cap) {
    c->res_cap = 0;
    if (!regrow(c->d_idx, nb * k * 4) || !regrow(c->d_score, nb * k * 4)) return -1;
    c->res_cap = b * k;
  }
  if (need > c->ws_bytes) {
    c->ws_bytes = 0;
    if (!regrow(c->ws, need)) return -1;
    c->ws_bytes = need;
  }
  return 0;
}
// d_queries_f32: the queries before their fp16 rounding, which an exact cache scores with (null: refused there); an exact
// cache rounds them to fp16 into its own query buffer itself and does not read d_queries_f16
int topk_dev_locked(sr_cache* c, const void* d_queries_f16, const float* d_queries_f32, int b, int k, void* cuda_stream) {
  if (c->exact && !d_queries_f32)
    return cfail("sr_cache_topk: an exact cache needs the fp32 queries (sr_cache_topk, sr_cache_topk_f32_dev)");
  cudaSetDevice(c->device);
  if (ensure(c, b, k)) return cfail("sr_cache_topk: allocation failed");
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->stream;
  if (!c->exact)
    return cache_topk(s, static_cast<const __half*>(d_queries_f16), b, c->rows, c->valid, c->size, c->dim, k, c->id_offset,
                      c->d_idx, c->d_score, c->ws, c->ws_bytes);
  if (cache_topk_exact(s, d_queries_f32, c->d_q, b, c->rows, c->rows32, c->valid, c->size, c->dim, c->rmax, k, c->sum_rule,
                       c->id_offset, c->d_idx, c->d_score, c->ws, c->ws_bytes, c->d_path, c->d_band, c->d_eps))
    return -1;
  c->last_b = b;
  c->last_kc = cache_exact_candidates(b, c->size, c->dim, k);
  c->last_fallback = cache_exact_fallback_count(c->ws, b, c->size, c->dim, k);
  return 0;
}
// fp32 queries on the device [b, dim]: a default cache rounds them to fp16 into its own query buffer (as sr_cache_topk
// always has) and scans that; an exact cache scores them as they are
int topk_f32_locked(sr_cache* c, const float* d_queries_f32, int b, int k, void* cuda_stream) {
  cudaSetDevice(c->device);
  if (ensure(c, b, k)) return cfail("sr_cache_topk: allocation failed");
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->stream;
  if (!c->exact && srb::cast_rows_f16(s, d_queries_f32, static_cast<size_t>(b) * c->dim, c->d_q)) return -1;
  return topk_dev_locked(c, c->d_q, d_queries_f32, b, k, cuda_stream);
}
}  // namespace

namespace srb {
// api.cu (sr_cache_lookup_ids) holds the cache's mutex from the scan until its D2H copies have landed
std::mutex& cache_mutex(sr_cache* c) { return c->mu; }
int cache_topk_dev_locked(sr_cache* c, const void* d_queries_f16, const float* d_queries_f32, int b, int k,
                          void* cuda_stream) {
  return topk_dev_locked(c, d_queries_f16, d_queries_f32, b, k, cuda_stream);
}
int cache_exact_stats(sr_cache* c, int b, int32_t* path, int32_t* band, double* eps, int* candidates, int* fallback) {
  std::lock_guard<std::mutex> lk(c->mu);
  if (!c->exact || c->last_b <= 0 || b != c->last_b) return -1;
  cudaSetDevice(c->device);
  if (cudaMemcpy(path, c->d_path, static_cast<size_t>(b) * 4, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(band, c->d_band, static_cast<size_t>(b) * 4, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(eps, c->d_eps, static_cast<size_t>(b) * 8, cudaMemcpyDeviceToHost) != cudaSuccess)
    return -1;
  if (candidates) *candidates = c->last_kc;
  if (fallback) {
    *fallback = 0;
    if (c->last_fallback && cudaMemcpy(fallback, c->last_fallback, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  }
  return 0;
}
}  // namespace srb

extern "C" {

static int cache_create(int device, int capacity, int dim, int id_offset, bool exact, int sum_rule, sr_cache** out) {
  if (!out || capacity <= 0 || dim <= 0 || dim % 8 != 0) return cfail("sr_cache_create: bad arguments (dim % 8 == 0)");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return cfail("sr_cache_create: no such CUDA device");
  cudaSetDevice(device);
  sr_cache* c = new sr_cache();
  c->device = device; c->capacity = capacity; c->dim = dim; c->id_offset = id_offset;
  c->exact = exact; c->sum_rule = sum_rule;
  c->cap_pad = (capacity + 255) / 256 * 256;  // GEMM N tiles may read (never report) the padding rows
  if (cudaMalloc(reinterpret_cast<void**>(&c->rows), static_cast<size_t>(c->cap_pad) * dim * 2) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&c->valid), c->cap_pad) != cudaSuccess ||
      (exact && cudaMalloc(reinterpret_cast<void**>(&c->rows32), static_cast<size_t>(capacity) * dim * 4) != cudaSuccess) ||
      cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
    sr_cache_free(c);
    return cfail("sr_cache_create: allocation failed");
  }
  cudaMemset(c->rows, 0, static_cast<size_t>(c->cap_pad) * dim * 2);
  cudaMemset(c->valid, 0, c->cap_pad);
  c->stores.push_back({reinterpret_cast<uint8_t*>(c->rows), static_cast<size_t>(dim) * 2});
  if (exact) c->stores.push_back({reinterpret_cast<uint8_t*>(c->rows32), static_cast<size_t>(dim) * 4});
  *out = c;
  return 0;
}

int sr_cache_create(int device, int capacity, int dim, int id_offset, sr_cache** out) {
  return cache_create(device, capacity, dim, id_offset, false, 0, out);
}

int sr_cache_create_exact(int device, int capacity, int dim, int id_offset, int sum_rule, sr_cache** out) {
  if (sum_rule != 0 && sum_rule != 1) return cfail("sr_cache_create_exact: sum_rule must be 0 (unfused) or 1 (fused)");
  return cache_create(device, capacity, dim, id_offset, true, sum_rule, out);
}

void sr_cache_free(sr_cache* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
  void* ptrs[] = {c->rows, c->valid, c->ws, c->d_q, c->d_q32, c->d_idx, c->d_score, c->rows32, c->d_path, c->d_band, c->d_eps};
  for (void* p : ptrs) if (p) cudaFree(p);
  delete c;
}

int sr_cache_add(sr_cache* c, const float* rows, int n) {
  if (!c || !rows || n <= 0) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->size + n > c->capacity) return cfail("sr_cache_add: capacity exceeded");
  const double norm = c->exact ? checked_max_norm(rows, static_cast<size_t>(n), c->dim) : 0;
  if (norm < 0) return cfail("sr_cache_add: an exact cache takes finite components of magnitude <= 65504 only");
  cudaSetDevice(c->device);
  // fp32 up in pieces of <= 64 MiB, rounded to fp16 (rn) on the device straight into the store.  An exact cache keeps the
  // fp32 rows as they are, so its pieces go up into rows32 and the fp16 copy is rounded from there; a default cache stages
  // them.
  const size_t piece_rows = std::max<size_t>(1, (64u << 20) / (static_cast<size_t>(c->dim) * 4));
  float* stage = nullptr;
  if (!c->exact &&
      cudaMalloc(reinterpret_cast<void**>(&stage), std::min<size_t>(piece_rows, n) * c->dim * 4) != cudaSuccess)
    return cfail("sr_cache_add: allocation failed");
  bool ok = true;
  for (size_t r0 = 0; ok && r0 < static_cast<size_t>(n); r0 += piece_rows) {
    const size_t nr = std::min<size_t>(piece_rows, n - r0), ne = nr * c->dim, at = (c->size + r0) * c->dim;
    float* up = c->exact ? c->rows32 + at : stage;
    ok = cudaMemcpyAsync(up, rows + r0 * c->dim, ne * 4, cudaMemcpyHostToDevice, c->stream) == cudaSuccess &&
         srb::cast_rows_f16(c->stream, up, ne, c->rows + at) == 0;
  }
  ok = ok && cudaMemsetAsync(c->valid + c->size, 1, n, c->stream) == cudaSuccess;
  ok = cudaStreamSynchronize(c->stream) == cudaSuccess && ok;
  if (stage) cudaFree(stage);
  if (!ok) return cfail("sr_cache_add: H2D failed");
  c->rmax = std::max(c->rmax, norm);
  const int first = c->size;
  c->size += n;
  return first;
}

int sr_cache_invalidate(sr_cache* c, int local_row) { return sr_cache_set_valid(c, local_row, 0); }

// ---- lifecycle mirror of the reference's entries slice (pkg/cache/inmemory_cache_lifecycle.go): the Go backend keeps
// entries[i] <-> device row i, so eviction (swap with the last entry, :296-303), TTL cleanup (stable compaction, :120-137)
// and pending entries (ResponseBody == nil: present but not searchable, inmemory_cache_search.go:71-73) have device forms.
int sr_cache_set_valid(sr_cache* c, int local_row, int valid) {
  if (!c) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (local_row < 0 || local_row >= c->size) return -1;
  cudaSetDevice(c->device);
  const uint8_t v = valid ? 1 : 0;
  return cudaMemcpy(c->valid + local_row, &v, 1, cudaMemcpyHostToDevice) == cudaSuccess ? 0 : -1;
}

int sr_cache_move(sr_cache* c, int dst_row, int src_row) {
  if (!c) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (dst_row < 0 || src_row < 0 || dst_row >= c->size || src_row >= c->size) return -1;
  if (dst_row == src_row) return 0;
  cudaSetDevice(c->device);
  bool ok = cudaMemcpyAsync(c->valid + dst_row, c->valid + src_row, 1, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess;
  for (const RowStore& s : c->stores)
    ok = ok && cudaMemcpyAsync(s.row(dst_row), s.row(src_row), s.row_bytes, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess;
  return (cudaStreamSynchronize(c->stream) == cudaSuccess && ok) ? 0 : -1;
}

int sr_cache_truncate(sr_cache* c, int new_size) {
  if (!c) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (new_size < 0 || new_size > c->size) return -1;
  cudaSetDevice(c->device);
  if (new_size < c->size && cudaMemset(c->valid + new_size, 0, c->size - new_size) != cudaSuccess) return -1;
  c->size = new_size;
  return 0;
}

// Stable compaction: rows with keep[i] != 0 move down in order (what cleanupExpiredEntriesInternal does to the slice).
// Runs of kept rows travel through a bounded scratch buffer, so a run never overlaps its own destination.
int sr_cache_compact(sr_cache* c, const uint8_t* keep, int n) {
  if (!c || !keep) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (n != c->size) return cfail("sr_cache_compact: keep mask must cover every row");
  cudaSetDevice(c->device);
  int first_drop = 0;
  while (first_drop < n && keep[first_drop]) ++first_drop;
  if (first_drop == n) return n;                       // nothing to remove
  std::vector<uint8_t> valid(static_cast<size_t>(n));
  if (cudaMemcpy(valid.data(), c->valid, n, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  size_t unit = 0;   // every store's runs go through the same scratch, sized for the widest store's rows
  for (const RowStore& s : c->stores) unit = std::max(unit, s.row_bytes);
  const int scratch_rows = static_cast<int>(std::min<size_t>(static_cast<size_t>(n), std::max<size_t>(1, (64u << 20) / unit)));
  void* scratch = nullptr;
  if (cudaMalloc(&scratch, static_cast<size_t>(scratch_rows) * unit) != cudaSuccess)
    return cfail("sr_cache_compact: allocation failed");
  bool ok = true;
  int w = first_drop;
  for (int r = first_drop; ok && r < n;) {
    if (!keep[r]) { ++r; continue; }
    int e = r;
    while (e < n && keep[e] && e - r < scratch_rows) ++e;   // run [r, e) of kept rows -> [w, w + e - r)
    for (const RowStore& s : c->stores) {
      const size_t bytes = static_cast<size_t>(e - r) * s.row_bytes;
      ok = ok && cudaMemcpyAsync(scratch, s.row(r), bytes, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess &&
           cudaMemcpyAsync(s.row(w), scratch, bytes, cudaMemcpyDeviceToDevice, c->stream) == cudaSuccess;
    }
    for (int i = r; i < e; ++i) valid[w + (i - r)] = valid[i];
    w += e - r;
    r = e;
  }
  for (int i = w; i < n; ++i) valid[i] = 0;
  ok = ok && cudaMemcpyAsync(c->valid, valid.data(), n, cudaMemcpyHostToDevice, c->stream) == cudaSuccess;
  ok = cudaStreamSynchronize(c->stream) == cudaSuccess && ok;
  cudaFree(scratch);
  if (!ok) return cfail("sr_cache_compact: copy failed");
  c->size = w;
  return w;
}

int sr_cache_size(const sr_cache* c) {
  if (!c) return -1;
  std::lock_guard<std::mutex> lk(const_cast<sr_cache*>(c)->mu);
  return c->size;
}
int sr_cache_dim(const sr_cache* c) { return c ? c->dim : -1; }

int sr_cache_topk_dev(sr_cache* c, const void* d_queries_f16, int b, int k, void* cuda_stream) {
  if (!c || b <= 0 || k <= 0) return -1;
  // the lock covers growing the scratch and queueing the scan; the result buffers belong to the cache, so callers of
  // this asynchronous entry serialise their use of one cache themselves (sr_b200.h)
  std::lock_guard<std::mutex> lk(c->mu);
  return topk_dev_locked(c, d_queries_f16, nullptr, b, k, cuda_stream);
}

int sr_cache_topk(sr_cache* c, const float* queries, int b, int k, int32_t* out_idx, float* out_score) {
  if (!c || !queries || b <= 0 || k <= 0 || !out_idx || !out_score) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->exact && checked_max_norm(queries, static_cast<size_t>(b), c->dim) < 0)
    return cfail("sr_cache_topk: an exact cache takes finite query components of magnitude <= 65504 only");
  cudaSetDevice(c->device);
  if (ensure(c, b, k)) return cfail("sr_cache_topk: allocation failed");
  // fp32 up, rounded to fp16 (rn) on the device: a host conversion loop over b*dim values costs more than the scan at
  // large b
  const size_t nq = static_cast<size_t>(b) * c->dim;
  if (cudaMemcpyAsync(c->d_q32, queries, nq * 4, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) return -1;
  if (topk_f32_locked(c, c->d_q32, b, k, nullptr)) return -1;
  cudaMemcpyAsync(out_idx, c->d_idx, static_cast<size_t>(b) * k * 4, cudaMemcpyDeviceToHost, c->stream);
  cudaMemcpyAsync(out_score, c->d_score, static_cast<size_t>(b) * k * 4, cudaMemcpyDeviceToHost, c->stream);
  const cudaError_t e = cudaStreamSynchronize(c->stream);
  if (e != cudaSuccess) { fprintf(stderr, "[srb200] sr_cache_topk: %s\n", cudaGetErrorString(e)); return -1; }
  return 0;
}

int sr_cache_topk_packed_dev(sr_cache* c, const void* d_queries_f16, int b, int k, void* d_pairs_out, void* cuda_stream) {
  if (!c || b <= 0 || k <= 0 || !d_pairs_out) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (topk_dev_locked(c, d_queries_f16, nullptr, b, k, cuda_stream)) return -1;
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->stream;
  return cache_pack_pairs(s, c->d_idx, c->d_score, b * k, d_pairs_out);
}

int sr_cache_topk_f32_dev(sr_cache* c, const float* d_queries_f32, int b, int k, void* cuda_stream) {
  if (!c || !d_queries_f32 || b <= 0 || k <= 0) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  return topk_f32_locked(c, d_queries_f32, b, k, cuda_stream);
}

int sr_cache_topk_packed_f32_dev(sr_cache* c, const float* d_queries_f32, int b, int k, void* d_pairs_out, void* cuda_stream) {
  if (!c || !d_queries_f32 || b <= 0 || k <= 0 || !d_pairs_out) return -1;
  std::lock_guard<std::mutex> lk(c->mu);
  if (topk_f32_locked(c, d_queries_f32, b, k, cuda_stream)) return -1;
  cudaStream_t s = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->stream;
  return cache_pack_pairs(s, c->d_idx, c->d_score, b * k, d_pairs_out);
}

int sr_cache_merge_packed_dev(int device, const void* d_pairs_parts, int g, int b, int k, int32_t* d_out_idx, float* d_out_score,
                              void* cuda_stream) {
  if (!d_pairs_parts || g <= 0 || b <= 0 || k <= 0 || !d_out_idx || !d_out_score) return -1;
  cudaSetDevice(device);
  return cache_merge_packed(static_cast<cudaStream_t>(cuda_stream), d_pairs_parts, g, b, k, d_out_idx, d_out_score);
}

const int32_t* sr_cache_dev_idx(const sr_cache* c) { return c ? c->d_idx : nullptr; }
const float* sr_cache_dev_score(const sr_cache* c) { return c ? c->d_score : nullptr; }

// host-side k-way merge (descending score, lower global id wins ties)
int sr_cache_merge_topk(const int32_t* idx_parts, const float* score_parts, int g, int b, int k, int32_t* out_idx,
                        float* out_score) {
  if (!idx_parts || !score_parts || g <= 0 || b <= 0 || k <= 0) return -1;
  std::vector<int> cur(g);
  for (int q = 0; q < b; ++q) {
    std::fill(cur.begin(), cur.end(), 0);
    for (int r = 0; r < k; ++r) {
      int best_g = -1, best_i = -1;
      float best_v = 0.f;
      for (int s = 0; s < g; ++s) {
        if (cur[s] >= k) continue;
        const size_t o = (static_cast<size_t>(s) * b + q) * k + cur[s];
        const int i = idx_parts[o];
        if (i < 0) continue;
        const float v = score_parts[o];
        if (best_g < 0 || v > best_v || (v == best_v && i < best_i)) { best_g = s; best_i = i; best_v = v; }
      }
      out_idx[static_cast<size_t>(q) * k + r] = best_i;
      out_score[static_cast<size_t>(q) * k + r] = best_g >= 0 ? best_v : -INFINITY;
      if (best_g >= 0) ++cur[best_g];
    }
  }
  return 0;
}

}  // extern "C"
