/* C restatement of the reference's Go embeddingDotProduct under both ways Go compiles it (TEST INFRASTRUCTURE ONLY).
 *
 * src/semantic-router/pkg/cache/inmemory_cache_search.go:14-20: dot := float32(0); for i: dot += q[i] * c[i].
 *   rule 0: the product rounded to fp32, then added (amd64 at GOAMD64=v1) -- the loop of cache_scan.c's dot_scalar;
 *   rule 1: one fused multiply-add per term (arm64, ppc64le, s390x, amd64 at GOAMD64=v3 and higher).
 * fmaf is the correctly rounded C99 fused multiply-add; fp-contract=off keeps the compiler from fusing rule 0.
 * Parity: restated, not executed against the Go code (no Go toolchain).
 */
#include <math.h>
#include <stddef.h>
#ifdef _OPENMP
#include <omp.h>
#endif

__attribute__((optimize("fp-contract=off")))
static float dot_rule(const float *q, const float *c, int d, int rule) {
    float dot = 0.0f;
    if (rule == 0) {
        for (int i = 0; i < d; ++i) { float p = q[i] * c[i]; dot = dot + p; }
    } else {
        for (int i = 0; i < d; ++i) dot = fmaf(q[i], c[i], dot);
    }
    return dot;
}

/* scores [b, n]: every query against every entry under `rule` */
void oracle_scores_go(const float *queries, const float *entries, int b, int n, int d, int rule, float *scores,
                      int threads) {
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#pragma omp parallel for collapse(2) schedule(static) if (threads != 1)
#endif
    for (int qi = 0; qi < b; ++qi)
        for (int i = 0; i < n; ++i)
            scores[(size_t)qi * n + i] = dot_rule(queries + (size_t)qi * d, entries + (size_t)i * d, d, rule);
}
