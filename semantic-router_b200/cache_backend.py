"""Device-resident semantic-cache backend: host-side mirror of integration/go/b200_cache.go (SURVEY.md section 8 f2).

The reference keeps every entry's embedding in a Go slice and scans it with a scalar loop under a read lock
(src/semantic-router/pkg/cache/inmemory_cache_search.go:65-89).  This backend keeps the embeddings in HBM (one fp16 row per
entry, row i == entries[i]) and asks the CUDA library for the best row (`sr_cache_topk`, k = 1: descending score, lowest row
first on ties == "first maximum wins"), while everything that is NOT arithmetic stays host bookkeeping with the reference's
semantics: pending entries (present, not searchable), per-entry and global TTL with the sliding window on a hit, lazy expiry
at lookup time, O(k) cleanup, FIFO / LRU / LFU eviction with "swap with the last entry".  Every slice mutation has its device
form (include/sr_b200.h: sr_cache_add / set_valid / move / truncate / compact).

The Go toolchain is absent in this image, so this Python class is what the tests drive (tests/test_cache_lifecycle_gpu.py
replays random operation sequences against oracle/cache_lifecycle_oracle.py); the Go file carries the same logic behind
the reference's CacheBackend interface (pkg/cache/cache_interface.go).  Method names follow the Go interface.
"""
from __future__ import annotations

import heapq
import itertools
import time
from collections import OrderedDict
from typing import Callable, Dict, List, Optional

import numpy as np

from .binding import Cache


class _Evictor:
    """eviction_policy.go: FIFO (:113-190), LRU (:198-290), LFU (:330-480) -- the victim each Evict() returns."""

    def __init__(self, kind: str):
        if kind not in ("fifo", "lru", "lfu"):
            raise ValueError("eviction policy must be fifo, lru or lfu")
        self.kind = kind
        self.queue: "OrderedDict[str, None]" = OrderedDict()
        self.count: Dict[str, int] = {}
        self.by_count: Dict[int, "OrderedDict[str, None]"] = {}
        self.floor = 0

    def inserted(self, rid: str):
        self.removed(rid)
        if self.kind == "lfu":
            self.count[rid] = 1
            self.by_count.setdefault(1, OrderedDict())[rid] = None
            self.floor = 1
        else:
            self.queue[rid] = None

    def accessed(self, rid: str):
        if self.kind == "lru":
            if rid in self.queue:
                self.queue.move_to_end(rid)
        elif self.kind == "lfu" and rid in self.count:
            c = self.count[rid]
            bucket = self.by_count.get(c)
            if bucket is not None:
                bucket.pop(rid, None)
                if c == self.floor and not bucket:
                    self.floor += 1
            self.count[rid] = c + 1
            self.by_count.setdefault(c + 1, OrderedDict())[rid] = None

    def removed(self, rid: str):
        if self.kind == "lfu":
            c = self.count.pop(rid, None)
            if c is not None:
                self.by_count.get(c, OrderedDict()).pop(rid, None)
        else:
            self.queue.pop(rid, None)

    def victim(self) -> Optional[str]:
        if self.kind != "lfu":
            if not self.queue:
                return None
            rid, _ = self.queue.popitem(last=False)
            return rid
        bucket = self.by_count.get(self.floor)
        if not bucket:
            for c in range(self.floor, self.floor + 1001):
                if self.by_count.get(c):
                    self.floor, bucket = c, self.by_count[c]
                    break
            else:
                return None
        rid, _ = bucket.popitem(last=False)
        self.count.pop(rid, None)
        return rid


class B200SemanticCache:
    """CacheBackend over a device-resident store.  `embed`: text -> unit vector (float32 [dim]); in the router that is the
    library's own embedding call (GetEmbedding2DMatryoshka at layer 6 / dim 256 by default, inmemory_cache.go:192-233)."""

    def __init__(self, dim: int, similarity_threshold: float, max_entries: int, ttl_seconds: int, eviction_policy: str = "fifo",
                 embed: Optional[Callable[[str], np.ndarray]] = None, device: int = 0, clock: Callable[[], float] = time.time,
                 capacity: Optional[int] = None, exact: bool = False, sum_rule: int = 0):
        self.dim = dim
        self.threshold = np.float32(similarity_threshold)
        self.max_entries = max_entries
        self.ttl_seconds = ttl_seconds
        self.embed = embed
        self.clock = clock
        cap = capacity or (max_entries if max_entries > 0 else 1 << 16)
        # exact: hit decisions on the reference's own fp32 scores (sr_cache_create_exact) under the Go build's sum rule
        self.store = Cache(cap, dim, device=device, exact=exact, sum_rule=sum_rule)
        self.evictor = _Evictor(eviction_policy)
        # entries[i] <-> device row i
        self.request_id: List[str] = []
        self.response: List[Optional[bytes]] = []
        self.ttl: List[int] = []
        self.expires_at: List[Optional[float]] = []
        self.last_access: List[float] = []
        self.hit_count: List[int] = []
        self.index_of: Dict[str, int] = {}
        self._heap: List = []
        self._deadline: Dict[str, float] = {}
        self._tick = itertools.count()
        self._switched_off: List[str] = []     # ids whose deadline passed at a lookup: off on the device, removed at the next cleanup
        self._lazily_expired: set = set()      # same for entries that only fall under the global TTL (no own deadline)
        self._no_deadline = 0                  # how many entries carry no deadline of their own
        self.hits = self.misses = 0

    # ---- expiration heap (eviction_policy.go:536-598)
    def _deadline_set(self, rid, at):
        self._deadline[rid] = at
        heapq.heappush(self._heap, (at, next(self._tick), rid))

    def _due(self, now) -> List[str]:
        """PopExpired (:577-588): every id whose deadline is <= now, including the ones a lookup already switched off."""
        out, self._switched_off = self._switched_off, []
        while self._heap and self._heap[0][0] <= now:
            at, _, rid = heapq.heappop(self._heap)
            if self._deadline.get(rid) == at:
                del self._deadline[rid]
                out.append(rid)
        return [rid for rid in out if rid in self.index_of]

    def _forget(self, rid):
        self.index_of.pop(rid, None)
        self._deadline.pop(rid, None)
        self.evictor.removed(rid)
        self._lazily_expired.discard(rid)

    # ---- slice mutations with their device forms
    def _cleanup_expired(self):                       # cleanupExpiredEntriesInternal (inmemory_cache_lifecycle.go:99-168)
        if self.ttl_seconds <= 0:
            return
        gone = set(self._due(self.clock()))
        if not gone:
            return
        keep = np.array([rid not in gone for rid in self.request_id], dtype=np.uint8)
        for rid in gone:
            self._forget(rid)
        self.store.compact(keep)                      # stable: survivors keep their order, like the slice compaction
        for name in ("request_id", "response", "ttl", "expires_at", "last_access", "hit_count"):
            col = getattr(self, name)
            setattr(self, name, [v for v, k in zip(col, keep) if k])
        self.index_of = {rid: i for i, rid in enumerate(self.request_id)}

    def _evict_one(self):                             # evictOne (:257-310)
        if not self.request_id:
            return
        rid = self.evictor.victim()
        if rid is None or rid not in self.index_of:
            return
        i = self.index_of[rid]
        self._forget(rid)
        last = len(self.request_id) - 1
        if i != last:                                 # swap with the last entry and shrink
            self.store.move(i, last)
            for name in ("request_id", "response", "ttl", "expires_at", "last_access", "hit_count"):
                col = getattr(self, name)
                col[i] = col[last]
            self.index_of[self.request_id[i]] = i
        self.store.truncate(last)
        for name in ("request_id", "response", "ttl", "expires_at", "last_access", "hit_count"):
            getattr(self, name).pop()

    def _append(self, rid, response, embedding, ttl_seconds):
        effective = self.ttl_seconds if ttl_seconds == -1 else ttl_seconds
        self._cleanup_expired()
        if self.max_entries > 0 and len(self.request_id) >= self.max_entries:
            self._evict_one()
        now = self.clock()
        row = self.store.add(np.asarray(embedding, dtype=np.float32)[None])
        assert row == len(self.request_id)
        if response is None:
            self.store.set_valid(row, False)          # pending: in the slice, skipped by the scan (search.go:71-73)
        self.request_id.append(rid)
        self.response.append(response)
        self.ttl.append(ttl_seconds)
        self.expires_at.append(now + effective if effective > 0 else None)
        self._no_deadline += 0 if effective > 0 else 1
        self.last_access.append(now)
        self.hit_count.append(0)
        self.index_of[rid] = row
        self.evictor.inserted(rid)
        if effective > 0:
            self._deadline_set(rid, now + effective)

    # ---- CacheBackend (pkg/cache/cache_interface.go)
    def AddPendingRequest(self, request_id: str, model: str, query: str, request_body: bytes, ttl_seconds: int = -1,
                          embedding: Optional[np.ndarray] = None):
        if ttl_seconds == 0:
            return
        self._append(request_id, None, self.embed(query) if embedding is None else embedding, ttl_seconds)

    def AddEntry(self, request_id: str, model: str, query: str, request_body: bytes, response_body: bytes, ttl_seconds: int = -1,
                 embedding: Optional[np.ndarray] = None):
        if ttl_seconds == 0:
            return
        self._append(request_id, response_body, self.embed(query) if embedding is None else embedding, ttl_seconds)

    def UpdateWithResponse(self, request_id: str, response_body: bytes, ttl_seconds: int = -1):
        self._cleanup_expired()
        i = self.index_of.get(request_id, -1)
        if not (0 <= i < len(self.request_id) and self.response[i] is None):
            i = next((k for k, (r, b) in enumerate(zip(self.request_id, self.response)) if r == request_id and b is None), -1)
        if i < 0:
            raise KeyError(f"no pending request found for request ID: {request_id}")
        now = self.clock()
        self.response[i] = response_body
        self.last_access[i] = now
        self.store.set_valid(i, True)
        if ttl_seconds != -1:
            self.ttl[i] = ttl_seconds
            if ttl_seconds > 0:
                self.expires_at[i] = now + ttl_seconds
                if request_id in self._deadline:
                    self._deadline_set(request_id, now + ttl_seconds)

    def _is_expired(self, i, now) -> bool:            # isExpired (:170-182)
        if self.expires_at[i] is not None:
            return now > self.expires_at[i]
        return self.ttl_seconds > 0 and now - self.last_access[i] >= self.ttl_seconds

    def _sync_expiry(self, now):
        """The scan must skip what isExpired() skips at `now` (inmemory_cache_search.go:74-77) although the entry stays in the
        slice until the next cleanup.  Deadlines are in a heap, so the rows to switch off are popped in order (strictly
        before now: isExpired is `now.After(ExpiresAt)`), remembered for that cleanup, and cost nothing when nothing is due."""
        while self._heap and self._heap[0][0] < now:
            at, _, rid = heapq.heappop(self._heap)
            if self._deadline.get(rid) != at:
                continue                              # a stale heap item: the deadline was moved by a hit / an update
            del self._deadline[rid]
            self._switched_off.append(rid)
            i = self.index_of.get(rid, -1)
            if i >= 0 and self.response[i] is not None:
                self.store.set_valid(i, False)
        if self._no_deadline and self.ttl_seconds > 0:   # entries without a per-entry deadline: global TTL on last access
            for i, at in enumerate(self.expires_at):
                if at is None and self.response[i] is not None and self.request_id[i] not in self._lazily_expired \
                        and self._is_expired(i, now):
                    self.store.set_valid(i, False)
                    self._lazily_expired.add(self.request_id[i])

    def FindSimilar(self, model: str, query: str, embedding: Optional[np.ndarray] = None):
        return self.FindSimilarWithThreshold(model, query, float(self.threshold), embedding=embedding)

    def FindSimilarWithThreshold(self, model: str, query: str, threshold: float, embedding: Optional[np.ndarray] = None):
        """-> (response | None, hit).  Also exposes .last_best = (index, similarity) like SimilarityTracker does."""
        q = np.asarray(self.embed(query) if embedding is None else embedding, dtype=np.float32)
        now = self.clock()
        self._sync_expiry(now)
        if len(self.request_id) == 0:
            self.misses += 1
            self.last_best = (-1, 0.0)
            return None, False
        idx, score = self.store.topk(q[None], 1)
        best, sim = int(idx[0, 0]), np.float32(score[0, 0])
        if best < 0:
            self.misses += 1
            self.last_best = (-1, 0.0)
            return None, False
        self.last_best = (best, float(sim))
        if sim >= np.float32(threshold):
            self.hits += 1
            rid = self.request_id[best]                # updateAccessInfo (:185-236): sliding TTL
            now = self.clock()
            self.last_access[best] = now
            self.hit_count[best] += 1
            self.evictor.accessed(rid)
            effective = self.ttl[best] if self.ttl[best] > 0 else self.ttl_seconds
            if effective > 0:
                self.expires_at[best] = now + effective
                if rid in self._deadline:
                    self._deadline_set(rid, now + effective)
            return self.response[best], True
        self.misses += 1
        return None, False

    def GetStats(self):
        total = self.hits + self.misses
        return {"TotalEntries": len(self.request_id), "HitCount": self.hits, "MissCount": self.misses,
                "HitRatio": (self.hits / total) if total else 0.0}

    def Close(self):
        self.store.close()
