//go:build !windows && cgo && b200 && !(amd64.v3 || arm64 || ppc64le || s390x)

package cache

// goSumRule tells sr_cache_create_exact how this binary evaluates embeddingDotProduct's `dot += q[i] * c[i]`: amd64 below
// GOAMD64=v3 has no fused multiply-add, so each product is rounded to float32 before it is added.
const goSumRule = 0
