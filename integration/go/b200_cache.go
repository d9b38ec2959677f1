//go:build !windows && cgo && b200

// Package cache: device-resident backend for the semantic cache (backend_type: "b200").
//
// Drop this file into src/semantic-router/pkg/cache/ of the reference and build with `-tags b200`.  It implements the
// reference's CacheBackend interface (cache_interface.go) on top of the B200 library's cache entry points
// (include/sr_b200.h: sr_cache_*): the embeddings of the entries live in HBM, one row per element of the entries slice in
// slice order, in an exact store (sr_cache_create_exact: the fp32 rows beside an fp16 copy, scores bitwise those of
// embeddingDotProduct as this binary's Go compiler evaluates it, goSumRule), and FindSimilar asks the GPU for the best
// row instead of running
// scanLinearForSimilarity (inmemory_cache_search.go:65-89) over a Go slice under a read lock.  Everything that is not
// arithmetic is the reference's own bookkeeping and reuses its types: CacheEntry, the FIFO / LRU / LFU policies and the
// ExpirationHeap of eviction_policy.go.  Each slice mutation has its device form:
//
//	append (AddEntry / AddPendingRequest)      sr_cache_add (+ sr_cache_set_valid(row, 0) for a pending entry)
//	UpdateWithResponse                          sr_cache_set_valid(row, 1)
//	isExpired at lookup time                    sr_cache_set_valid(row, 0) for the ids whose deadline has passed
//	evictOne: swap with the last, shrink        sr_cache_move(victim, last) + sr_cache_truncate(last)
//	cleanupExpiredEntriesInternal: compaction   sr_cache_compact(keep mask)
//
// The same logic, line for line, runs in this repository's tests as semantic-router_b200/cache_backend.py against
// oracle/cache_lifecycle_oracle.py (tests/test_cache_lifecycle_gpu.py) -- the Go toolchain is not part of the build image.
package cache

/*
#cgo LDFLAGS: -L${SRCDIR}/../../../../candle-binding/target/release -lcandle_semantic_router
#include <stdint.h>
#include <stdlib.h>
typedef struct sr_cache sr_cache;
int sr_cache_create_exact(int device, int capacity, int dim, int id_offset, int sum_rule, sr_cache** out);
void sr_cache_free(sr_cache* c);
int sr_cache_add(sr_cache* c, const float* rows, int n);
int sr_cache_set_valid(sr_cache* c, int local_row, int valid);
int sr_cache_move(sr_cache* c, int dst_row, int src_row);
int sr_cache_truncate(sr_cache* c, int new_size);
int sr_cache_compact(sr_cache* c, const uint8_t* keep, int n);
int sr_cache_topk(sr_cache* c, const float* queries, int b, int k, int32_t* out_idx, float* out_score);
*/
import "C"

import (
	"fmt"
	"sync"
	"sync/atomic"
	"time"
	"unsafe"
)

// B200CacheType selects this backend in cache_factory.go: `case B200CacheType: return NewB200Cache(options), nil`.
const B200CacheType CacheBackendType = "b200"

type B200Cache struct {
	SimilarityTracker
	mu                  sync.Mutex
	store               *C.sr_cache
	dim                 int
	entries             []CacheEntry // Embedding is nil: row i of the device store holds it
	entryMap            map[string]int
	similarityThreshold float32
	maxEntries          int
	ttlSeconds          int
	enabled             bool
	hitCount            int64
	missCount           int64
	policyType          EvictionPolicyType
	lru                 *LRUPolicy
	lfu                 *LFUPolicy
	fifo                *FIFOPolicy
	expirationHeap      *ExpirationHeap
	switchedOff         []string // ids whose deadline passed at a lookup: invalid on the device, removed at the next cleanup
	embed               func(string) ([]float32, error)
	lastCleanupTime     *time.Time
}

// NewB200Cache mirrors NewInMemoryCache (inmemory_cache.go:124-178).  `embed` is the cache's embedding call
// (generateEmbedding, :192-233); its vectors must be unit length like the reference's.
func NewB200Cache(options InMemoryCacheOptions, device int, dim int, embed func(string) ([]float32, error)) (*B200Cache, error) {
	capacity := options.MaxEntries
	if capacity <= 0 {
		capacity = 1 << 20
	}
	c := &B200Cache{
		dim: dim, entryMap: map[string]int{}, similarityThreshold: options.SimilarityThreshold,
		maxEntries: options.MaxEntries, ttlSeconds: options.TTLSeconds, enabled: options.Enabled,
		policyType: options.EvictionPolicy, expirationHeap: NewExpirationHeap(), embed: embed,
	}
	switch options.EvictionPolicy {
	case LRUEvictionPolicyType:
		c.lru = NewLRUPolicy()
	case LFUEvictionPolicyType:
		c.lfu = NewLFUPolicy()
	default:
		c.fifo = NewFIFOPolicy()
	}
	if rc := C.sr_cache_create_exact(C.int(device), C.int(capacity), C.int(dim), 0, C.int(goSumRule), &c.store); rc != 0 {
		return nil, fmt.Errorf("sr_cache_create_exact failed (no sm_90 GPU?)")
	}
	return c, nil
}

func (c *B200Cache) IsEnabled() bool        { return c.enabled }
func (c *B200Cache) CheckConnection() error { return nil }

func (c *B200Cache) onInsert(i int, id string) {
	switch {
	case c.lru != nil:
		c.lru.OnInsert(i, id)
	case c.lfu != nil:
		c.lfu.OnInsert(i, id)
	default:
		c.fifo.OnInsert(i, id)
	}
}
func (c *B200Cache) onAccess(i int, id string) {
	if c.lru != nil {
		c.lru.OnAccess(i, id)
	} else if c.lfu != nil {
		c.lfu.OnAccess(i, id)
	}
}
func (c *B200Cache) onRemove(i int, id string) {
	delete(c.entryMap, id)
	c.expirationHeap.Remove(id)
	switch {
	case c.lru != nil:
		c.lru.OnRemove(i, id)
	case c.lfu != nil:
		c.lfu.OnRemove(i, id)
	default:
		c.fifo.OnRemove(i, id)
	}
}
func (c *B200Cache) onMove(id string, from, to int) {
	c.entryMap[id] = to
	c.expirationHeap.UpdateIndex(id, to)
	switch {
	case c.lru != nil:
		c.lru.UpdateIndex(id, from, to)
	case c.lfu != nil:
		c.lfu.UpdateIndex(id, from, to)
	default:
		c.fifo.UpdateIndex(id, from, to)
	}
}
func (c *B200Cache) evictVictim() int {
	switch {
	case c.lru != nil:
		return c.lru.Evict()
	case c.lfu != nil:
		return c.lfu.Evict()
	default:
		return c.fifo.Evict()
	}
}

// cleanupExpired == cleanupExpiredEntriesInternal (inmemory_cache_lifecycle.go:99-168); caller holds c.mu.
func (c *B200Cache) cleanupExpired() {
	if c.ttlSeconds <= 0 {
		return
	}
	gone := append(c.switchedOff, c.expirationHeap.PopExpired(time.Now())...)
	c.switchedOff = nil
	if len(gone) == 0 {
		return
	}
	expired := make(map[string]bool, len(gone))
	for _, id := range gone {
		expired[id] = true
	}
	keep := make([]C.uint8_t, len(c.entries))
	w := 0
	for r := range c.entries {
		e := c.entries[r]
		if !expired[e.RequestID] {
			keep[r] = 1
			if w != r {
				c.entries[w] = e
				c.onMove(e.RequestID, r, w)
			}
			w++
		} else {
			c.onRemove(r, e.RequestID)
		}
	}
	C.sr_cache_compact(c.store, &keep[0], C.int(len(keep)))
	c.entries = c.entries[:w]
	now := time.Now()
	c.lastCleanupTime = &now
}

// evictOne == evictOne (inmemory_cache_lifecycle.go:257-310); caller holds c.mu.
func (c *B200Cache) evictOne() {
	if len(c.entries) == 0 {
		return
	}
	v := c.evictVictim()
	if v < 0 || v >= len(c.entries) {
		return
	}
	c.onRemove(v, c.entries[v].RequestID)
	last := len(c.entries) - 1
	if v != last {
		moved := c.entries[last]
		c.entries[v] = moved
		C.sr_cache_move(c.store, C.int(v), C.int(last))
		c.onMove(moved.RequestID, last, v)
	}
	C.sr_cache_truncate(c.store, C.int(last))
	c.entries = c.entries[:last]
}

func (c *B200Cache) appendEntry(requestID, model, query string, requestBody, responseBody []byte, ttlSeconds int) error {
	if !c.enabled || ttlSeconds == 0 {
		return nil
	}
	effectiveTTL := ttlSeconds
	if ttlSeconds == -1 {
		effectiveTTL = c.ttlSeconds
	}
	embedding, err := c.embed(query)
	if err != nil {
		return fmt.Errorf("failed to generate embedding: %w", err)
	}
	if len(embedding) != c.dim {
		return fmt.Errorf("embedding has %d dimensions, the store %d", len(embedding), c.dim)
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	c.cleanupExpired()
	if c.maxEntries > 0 && len(c.entries) >= c.maxEntries {
		c.evictOne()
	}
	now := time.Now()
	row := int(C.sr_cache_add(c.store, (*C.float)(unsafe.Pointer(&embedding[0])), 1))
	if row != len(c.entries) {
		return fmt.Errorf("device store out of step with the entries slice (row %d, entries %d)", row, len(c.entries))
	}
	if responseBody == nil {
		C.sr_cache_set_valid(c.store, C.int(row), 0) // pending: in the slice, skipped by the scan (inmemory_cache_search.go:71-73)
	}
	e := CacheEntry{RequestID: requestID, RequestBody: requestBody, ResponseBody: responseBody, Model: model, Query: query,
		Timestamp: now, LastAccessAt: now, TTLSeconds: ttlSeconds}
	if effectiveTTL > 0 {
		e.ExpiresAt = now.Add(time.Duration(effectiveTTL) * time.Second)
	}
	c.entries = append(c.entries, e)
	c.entryMap[requestID] = row
	c.onInsert(row, requestID)
	if effectiveTTL > 0 {
		c.expirationHeap.Add(requestID, row, e.ExpiresAt)
	}
	return nil
}

func (c *B200Cache) AddPendingRequest(requestID, model, query string, requestBody []byte, ttlSeconds int) error {
	return c.appendEntry(requestID, model, query, requestBody, nil, ttlSeconds)
}

func (c *B200Cache) AddEntry(requestID, model, query string, requestBody, responseBody []byte, ttlSeconds int) error {
	if responseBody == nil {
		responseBody = []byte{}
	}
	return c.appendEntry(requestID, model, query, requestBody, responseBody, ttlSeconds)
}

// UpdateWithResponse == inmemory_cache.go:324-381.
func (c *B200Cache) UpdateWithResponse(requestID string, responseBody []byte, ttlSeconds int) error {
	if !c.enabled {
		return nil
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	c.cleanupExpired()
	target := -1
	if i, ok := c.entryMap[requestID]; ok && i >= 0 && i < len(c.entries) && c.entries[i].RequestID == requestID && c.entries[i].ResponseBody == nil {
		target = i
	} else {
		for i := range c.entries {
			if c.entries[i].RequestID == requestID && c.entries[i].ResponseBody == nil {
				target = i
				c.entryMap[requestID] = i
				break
			}
		}
	}
	if target == -1 {
		return fmt.Errorf("no pending request found for request ID: %s", requestID)
	}
	now := time.Now()
	if responseBody == nil {
		responseBody = []byte{}
	}
	c.entries[target].ResponseBody = responseBody
	c.entries[target].Timestamp = now
	c.entries[target].LastAccessAt = now
	C.sr_cache_set_valid(c.store, C.int(target), 1)
	if ttlSeconds != -1 {
		c.entries[target].TTLSeconds = ttlSeconds
		if ttlSeconds > 0 {
			c.entries[target].ExpiresAt = now.Add(time.Duration(ttlSeconds) * time.Second)
			c.expirationHeap.UpdateExpiration(requestID, c.entries[target].ExpiresAt)
		}
	}
	return nil
}

func (c *B200Cache) FindSimilar(model string, query string) ([]byte, bool, error) {
	return c.FindSimilarWithThreshold(model, query, c.similarityThreshold)
}

// FindSimilarWithThreshold == inmemory_cache_search.go:100-207 with the scan on the GPU.
func (c *B200Cache) FindSimilarWithThreshold(model string, query string, threshold float32) ([]byte, bool, error) {
	if !c.enabled {
		return nil, false, nil
	}
	q, err := c.embed(query)
	if err != nil {
		return nil, false, fmt.Errorf("failed to generate embedding: %w", err)
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	now := time.Now()
	// what isExpired() would skip at `now` is switched off on the device; the entries stay in the slice until cleanup
	for {
		id, idx, at, ok := c.expirationHeap.PeekNext()
		if !ok || !now.After(at) {
			break
		}
		c.expirationHeap.Remove(id)
		c.switchedOff = append(c.switchedOff, id)
		if idx >= 0 && idx < len(c.entries) && c.entries[idx].RequestID == id && c.entries[idx].ResponseBody != nil {
			C.sr_cache_set_valid(c.store, C.int(idx), 0)
		}
	}
	if len(c.entries) == 0 {
		atomic.AddInt64(&c.missCount, 1)
		return nil, false, nil
	}
	var idx C.int32_t
	var score C.float
	if rc := C.sr_cache_topk(c.store, (*C.float)(unsafe.Pointer(&q[0])), 1, 1, &idx, &score); rc != 0 {
		return nil, false, fmt.Errorf("sr_cache_topk failed")
	}
	best := int(idx)
	if best < 0 || best >= len(c.entries) {
		atomic.AddInt64(&c.missCount, 1)
		return nil, false, nil
	}
	sim := float32(score)
	c.StoreSimilarity(sim)
	if sim >= threshold {
		atomic.AddInt64(&c.hitCount, 1)
		e := &c.entries[best] // updateAccessInfo (inmemory_cache_lifecycle.go:185-236): sliding TTL
		now = time.Now()
		e.LastAccessAt = now
		e.HitCount++
		c.onAccess(best, e.RequestID)
		effectiveTTL := c.ttlSeconds
		if e.TTLSeconds > 0 {
			effectiveTTL = e.TTLSeconds
		}
		if effectiveTTL > 0 {
			e.ExpiresAt = now.Add(time.Duration(effectiveTTL) * time.Second)
			c.expirationHeap.UpdateExpiration(e.RequestID, e.ExpiresAt)
		}
		return e.ResponseBody, true, nil
	}
	atomic.AddInt64(&c.missCount, 1)
	return nil, false, nil
}

func (c *B200Cache) GetStats() CacheStats {
	c.mu.Lock()
	defer c.mu.Unlock()
	hits, misses := atomic.LoadInt64(&c.hitCount), atomic.LoadInt64(&c.missCount)
	ratio := 0.0
	if hits+misses > 0 {
		ratio = float64(hits) / float64(hits+misses)
	}
	return CacheStats{TotalEntries: len(c.entries), HitCount: hits, MissCount: misses, HitRatio: ratio, LastCleanupTime: c.lastCleanupTime}
}

func (c *B200Cache) Close() error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if c.store != nil {
		C.sr_cache_free(c.store)
		c.store = nil
	}
	c.entries = nil
	return nil
}
