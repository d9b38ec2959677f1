/* C restatement of the reference's Go linear cache scan (TEST INFRASTRUCTURE / CPU BASELINE ONLY).
 *
 * Follows src/semantic-router/pkg/cache/inmemory_cache_search.go:
 *   embeddingDotProduct       :14-20  -- sequential scalar f32 FMA-free dot product
 *   scanLinearForSimilarity   :65-89  -- bestIndex=-1; update when bestIndex==-1 || dot > best
 * No expiry/nil handling here (all rows valid) -- that is covered by cache_oracle.scan_linear.
 * Parity: restated, not executed against the Go code (no Go toolchain) -- "parity unpinned".
 */
#include <stddef.h>
#ifdef _OPENMP
#include <omp.h>
#endif

static float dot_scalar(const float *q, const float *c, int d) {
    float dot = 0.0f;
    for (int i = 0; i < d; ++i) dot += q[i] * c[i];
    return dot;
}

void oracle_scan_linear(const float *queries, const float *entries, int b, int n, int d,
                        int *best_idx, float *best_score, int threads) {
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#pragma omp parallel for schedule(static) if (threads != 1)
#endif
    for (int qi = 0; qi < b; ++qi) {
        const float *q = queries + (size_t)qi * d;
        int bi = -1;
        float bs = 0.0f;
        for (int i = 0; i < n; ++i) {
            float s = dot_scalar(q, entries + (size_t)i * d, d);
            if (bi == -1 || s > bs) { bs = s; bi = i; }
        }
        best_idx[qi] = bi;
        best_score[qi] = bs;
    }
}
