//go:build !windows && cgo && b200 && (amd64.v3 || arm64 || ppc64le || s390x)

package cache

// goSumRule tells sr_cache_create_exact how this binary evaluates embeddingDotProduct's `dot += q[i] * c[i]`: on these
// targets the Go compiler fuses it into one multiply-add per term (amd64.v3 holds for GOAMD64=v3 and higher).
const goSumRule = 1
