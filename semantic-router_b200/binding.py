"""ctypes binding over include/sr_b200.h (side-door ABI) -- the Python mirror of the wrappers in
candle-binding/semantic-router.go (`ClassifyModernBertTextWithProbabilities` :3036, `GetEmbedding2DMatryoshka`
:1548, `CalculateSimilarityBatch` :1769 ...), at the token-id level.  Fails loudly when the CUDA library
is missing: there is no fallback implementation."""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence

import numpy as np

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libcandle_semantic_router.so")
# the same objects + the sr_test_* unit-op hooks (include/sr_b200_testhooks.h); the product library does not export them
HOOKS_LIB_PATH = os.environ.get("SR_B200_HOOKS_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib",
                                                                       "libcandle_semantic_router_testhooks.so")
_lib = None


class SrError(RuntimeError):
    pass


class ModelInfo(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("arch", "hidden", "layers", "heads", "intermediate", "vocab", "max_pos",
                                       "num_heads_loaded", "device")]


def load_library(path: Optional[str] = None):
    global _lib
    if _lib is not None:
        return _lib
    path = path or os.environ.get("SR_B200_LIB", LIB_PATH)
    if not os.path.exists(path):
        raise SrError(f"CUDA extension not built: {path} missing (run `python __graft_entry__.py`); "
                      "there is no CPU fallback")
    L = C.CDLL(path)
    vp, ip, fp = C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float)
    L.sr_last_error.restype = C.c_char_p
    L.sr_model_load.argtypes = [C.c_char_p, C.c_int, C.POINTER(vp)]
    L.sr_model_add_head.argtypes = [vp, C.c_char_p, C.c_int]
    L.sr_model_free.argtypes = [vp]
    L.sr_model_free.restype = None
    L.sr_model_info.argtypes = [vp, C.POINTER(ModelInfo)]
    L.sr_head_num_classes.argtypes = [vp, C.c_int]
    L.sr_classify_ids.argtypes = [vp, C.c_int, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp]
    L.sr_classify_tokens_ids.argtypes = [vp, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp]
    L.sr_embed_ids.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, vp]
    L.sr_embed_ids_padded.argtypes = [vp, vp, vp, vp, C.c_int, vp]
    L.sr_classify_multi_ids.argtypes = [vp, vp, C.c_int, vp, vp, C.c_int, vp, vp]
    L.sr_model_load_lora_shared.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.sr_lora_shared_mode.argtypes = [vp]
    L.sr_lora_shared_tasks.argtypes = [vp]
    L.sr_checkpoint_has_adapters.argtypes = [C.c_char_p]
    L.sr_classify_lora_shared_ids.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp]
    L.sr_model_set_stream.argtypes = [vp, vp]
    L.sr_model_set_precise.argtypes = [vp, C.c_int]
    L.sr_reserve.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.sr_forward_dev.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
    L.sr_head_seq_dev.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int]
    L.sr_head_tokens_dev.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.sr_head_embed_dev.argtypes = [vp, vp, C.c_int, C.c_int]
    L.sr_sync.argtypes = [vp]
    for f in ("sr_dev_probs", "sr_dev_logits", "sr_dev_cls", "sr_dev_conf", "sr_dev_emb", "sr_dev_hidden"):
        getattr(L, f).argtypes = [vp]
        getattr(L, f).restype = vp
    L.sr_cache_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]
    L.sr_cache_free.argtypes = [vp]
    L.sr_cache_free.restype = None
    L.sr_cache_add.argtypes = [vp, vp, C.c_int]
    L.sr_cache_invalidate.argtypes = [vp, C.c_int]
    L.sr_cache_size.argtypes = [vp]
    L.sr_cache_set_valid.argtypes = [vp, C.c_int, C.c_int]
    L.sr_cache_move.argtypes = [vp, C.c_int, C.c_int]
    L.sr_cache_truncate.argtypes = [vp, C.c_int]
    L.sr_cache_compact.argtypes = [vp, vp, C.c_int]
    L.sr_cache_topk.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp]
    L.sr_cache_dim.argtypes = [vp]
    L.sr_cache_lookup_ids.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp]
    L.sr_cache_topk_dev.argtypes = [vp, vp, C.c_int, C.c_int, vp]
    L.sr_cache_dev_idx.argtypes = [vp]
    L.sr_cache_dev_idx.restype = vp
    L.sr_cache_dev_score.argtypes = [vp]
    L.sr_cache_dev_score.restype = vp
    L.sr_cache_merge_topk.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp]
    L.sr_cache_topk_packed_dev.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp]
    L.sr_cache_merge_packed_dev.argtypes = [C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    _attach_hooks(L)
    _lib = L
    return L


_hooks = None


def hooks():
    """libcandle_semantic_router_testhooks.so: the product objects plus the sr_test_* entry points (tests / tools only)."""
    global _hooks
    if _hooks is None:
        if not os.path.exists(HOOKS_LIB_PATH):
            raise SrError(f"test-hook library not built: {HOOKS_LIB_PATH} (run `python __graft_entry__.py`)")
        H = C.CDLL(HOOKS_LIB_PATH)
        vp = C.c_void_p
        H.sr_test_gemm.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_int]
        H.sr_test_attention.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
        H.sr_test_attention_tc.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        H.sr_test_attention_win.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        H.sr_test_layernorm.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_float, vp, vp]
        H.sr_test_gemm_fold.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_int,
                                        vp, vp, vp, C.c_float, C.c_int, vp, vp, vp]
        H.sr_test_gemm_resid_hl.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, vp]
        H.sr_test_hl_to_f32.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp]
        _hooks = H
    return _hooks


def _attach_hooks(L):
    """Tests and tools written against `lib().sr_test_*` keep working: the names resolve to the hook library's entry
    points (the very same kernels, linked from the same objects).  Nothing is attached when that library is absent."""
    if not os.path.exists(HOOKS_LIB_PATH):
        return
    H = hooks()
    for name in ("sr_test_gemm", "sr_test_gemm_fold", "sr_test_attention", "sr_test_attention_tc", "sr_test_attention_win",
                 "sr_test_layernorm", "sr_test_bio_decode", "sr_test_hallucination_spans"):
        setattr(L, name, getattr(H, name))


def lib():
    return load_library()


def device_count() -> int:
    return int(lib().sr_device_count())


def _err(what: str) -> SrError:
    return SrError(f"{what}: {lib().sr_last_error().decode(errors='replace')}")


def pack(seqs: Sequence[np.ndarray]):
    """List of id arrays -> (ids int32 [T], cu_seqlens int32 [B+1])."""
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    cu = np.zeros(len(seqs) + 1, dtype=np.int32)
    cu[1:] = np.cumsum(lens)
    ids = np.ascontiguousarray(np.concatenate([np.asarray(s, dtype=np.int32) for s in seqs]))
    return ids, cu


def _p(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data


class Model:
    """One encoder (+ heads) resident on one GPU.  Mirrors the reference's per-task OnceLock slots
    (candle-binding/src/ffi/init.rs:19-60) as explicit objects."""

    def __init__(self, model_dir: str, device: int = 0):
        self._h = C.c_void_p()
        if lib().sr_model_load(model_dir.encode(), device, C.byref(self._h)) != 0:
            raise _err("sr_model_load")
        info = ModelInfo()
        lib().sr_model_info(self._h, C.byref(info))
        self.info = info
        self.hidden = info.hidden

    def close(self):
        if self._h:
            lib().sr_model_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def set_precise(self, on: bool = True):
        """fp32-equivalent encoder arithmetic (split-fp16 GEMM operands, fp32 in between): include/sr_b200.h."""
        if lib().sr_model_set_precise(self._h, 1 if on else 0) != 0:
            raise _err("sr_model_set_precise")

    def add_head(self, model_dir: str, token_level: int = -1) -> int:
        r = lib().sr_model_add_head(self._h, model_dir.encode(), token_level)
        if r < 0:
            raise _err("sr_model_add_head")
        return r

    def num_classes(self, head: int = 0) -> int:
        return int(lib().sr_head_num_classes(self._h, head))

    # ---- host-buffer entries (the e2e path: H2D + compute + D2H inside the call)
    def classify_ids(self, seqs: Sequence[np.ndarray], head: int = 0, pooler_mode: int = 0) -> Dict[str, np.ndarray]:
        ids, cu = pack(seqs)
        return self.classify_packed(ids, cu, head, pooler_mode)

    def classify_packed(self, ids: np.ndarray, cu: np.ndarray, head: int = 0, pooler_mode: int = 0,
                        want_logits: bool = True):
        B, Cn = len(cu) - 1, self.num_classes(head)
        probs = np.empty((B, Cn), dtype=np.float32)
        logits = np.empty((B, Cn), dtype=np.float32) if want_logits else None
        cls = np.empty(B, dtype=np.int32)
        conf = np.empty(B, dtype=np.float32)
        if lib().sr_classify_ids(self._h, head, _p(ids), _p(cu), B, pooler_mode, _p(probs), _p(logits), _p(cls),
                                 _p(conf)) != 0:
            raise _err("sr_classify_ids")
        return {"probs": probs, "logits": logits, "cls": cls, "conf": conf}

    def classify_tokens_ids(self, seqs: Sequence[np.ndarray], head: int = 0):
        ids, cu = pack(seqs)
        T, Cn = len(ids), self.num_classes(head)
        probs = np.empty((T, Cn), dtype=np.float32)
        logits = np.empty((T, Cn), dtype=np.float32)
        pred = np.empty(T, dtype=np.int32)
        conf = np.empty(T, dtype=np.float32)
        if lib().sr_classify_tokens_ids(self._h, head, _p(ids), _p(cu), len(cu) - 1, _p(probs), _p(logits), _p(pred),
                                        _p(conf)) != 0:
            raise _err("sr_classify_tokens_ids")
        return {"probs": probs, "logits": logits, "pred": pred, "conf": conf, "cu": cu}

    def embed_ids(self, seqs: Sequence[np.ndarray], target_layer: int = 0, target_dim: int = 0) -> np.ndarray:
        ids, cu = pack(seqs)
        dim = self.hidden if target_dim <= 0 else target_dim
        emb = np.empty((len(cu) - 1, dim), dtype=np.float32)
        if lib().sr_embed_ids(self._h, _p(ids), _p(cu), len(cu) - 1, target_layer, target_dim, _p(emb)) != 0:
            raise _err("sr_embed_ids")
        return emb

    def embed_ids_padded(self, seqs: Sequence[np.ndarray], real_lens: Sequence[int]) -> np.ndarray:
        """BertSimilarity under a fixed-padding tokenizer: pads are queries, masked as keys, summed by the pooling."""
        ids, cu = pack(seqs)
        rl = np.ascontiguousarray(real_lens, dtype=np.int32)
        info = ModelInfo()
        lib().sr_model_info(self._h, C.byref(info))
        emb = np.empty((len(seqs), info.hidden), dtype=np.float32)
        if lib().sr_embed_ids_padded(self._h, _p(ids), _p(cu), _p(rl), len(seqs), _p(emb)) != 0:
            raise _err("sr_embed_ids_padded")
        return emb

    def classify_multi_ids(self, seqs: Sequence[np.ndarray], heads: Sequence[int], token_level: Sequence[bool]):
        ids, cu = pack(seqs)
        B, T = len(cu) - 1, len(ids)
        hs = np.asarray(heads, dtype=np.int32)
        probs, cls = [], []
        for h, tok in zip(heads, token_level):
            rows = T if tok else B
            probs.append(np.empty((rows, self.num_classes(h)), dtype=np.float32))
            cls.append(np.empty(rows, dtype=np.int32))
        pp = (C.c_void_p * len(heads))(*[p.ctypes.data for p in probs])
        cp = (C.c_void_p * len(heads))(*[c.ctypes.data for c in cls])
        if lib().sr_classify_multi_ids(self._h, _p(hs), len(heads), _p(ids), _p(cu), B, pp, cp) != 0:
            raise _err("sr_classify_multi_ids")
        return probs, cls


class LoraSharedModel(Model):
    """ONE base encoder + the unmerged LoRA adapters and heads of several task checkpoints over it (sr_b200.h:
    sr_model_load_lora_shared); a batch runs once, every task's rows with its own rank-r terms."""

    LOWRANK, GROUPED = 0, 1

    def __init__(self, task_dirs: Sequence[str], token_level: Sequence[int], device: int = 0, mode: int = 0):
        self._h = C.c_void_p()
        dirs = (C.c_char_p * len(task_dirs))(*[d.encode() for d in task_dirs])
        tl = np.asarray(token_level, dtype=np.int32)
        if lib().sr_model_load_lora_shared(dirs, _p(tl), len(task_dirs), mode, device, C.byref(self._h)) != 0:
            raise _err("sr_model_load_lora_shared")
        info = ModelInfo()
        lib().sr_model_info(self._h, C.byref(info))
        self.info = info
        self.hidden = info.hidden
        self.token_level = [bool(t) for t in token_level]
        self.tasks = lib().sr_lora_shared_tasks(self._h)

    def classify_shared_ids(self, seqs: Sequence[np.ndarray], pooler_mode: int = 0):
        ids, cu = pack(seqs)
        B, T = len(cu) - 1, len(ids)
        probs, cls, conf = [], [], []
        for t, tok in enumerate(self.token_level):
            rows = T if tok else B
            probs.append(np.empty((rows, self.num_classes(t)), dtype=np.float32))
            cls.append(np.empty(rows, dtype=np.int32))
            conf.append(np.empty(rows, dtype=np.float32))
        arr = lambda xs: (C.c_void_p * len(xs))(*[x.ctypes.data for x in xs])
        if lib().sr_classify_lora_shared_ids(self._h, _p(ids), _p(cu), B, pooler_mode, arr(probs), arr(cls), arr(conf)) != 0:
            raise _err("sr_classify_lora_shared_ids")
        return probs, cls, conf


class Cache:
    """Device-resident semantic cache shard (mirror of pkg/cache/inmemory_cache.go's lookup side)."""

    def __init__(self, capacity: int, dim: int, device: int = 0, id_offset: int = 0):
        self._h = C.c_void_p()
        if lib().sr_cache_create(device, capacity, dim, id_offset, C.byref(self._h)) != 0:
            raise SrError("sr_cache_create failed")
        self.dim = dim

    def close(self):
        if self._h:
            lib().sr_cache_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def add(self, rows: np.ndarray) -> int:
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        r = lib().sr_cache_add(self._h, _p(rows), rows.shape[0])
        if r < 0:
            raise SrError("sr_cache_add failed")
        return r

    def invalidate(self, row: int):
        if lib().sr_cache_invalidate(self._h, row) != 0:
            raise SrError("sr_cache_invalidate failed")

    def __len__(self):
        return int(lib().sr_cache_size(self._h))

    # ---- lifecycle mirror of the reference's entries slice (sr_b200.h)
    def set_valid(self, row: int, valid: bool):
        if lib().sr_cache_set_valid(self._h, row, 1 if valid else 0) != 0:
            raise SrError("sr_cache_set_valid failed")

    def move(self, dst: int, src: int):
        if lib().sr_cache_move(self._h, dst, src) != 0:
            raise SrError("sr_cache_move failed")

    def truncate(self, n: int):
        if lib().sr_cache_truncate(self._h, n) != 0:
            raise SrError("sr_cache_truncate failed")

    def compact(self, keep: np.ndarray) -> int:
        k = np.ascontiguousarray(keep, dtype=np.uint8)
        r = lib().sr_cache_compact(self._h, _p(k), k.shape[0])
        if r < 0:
            raise SrError("sr_cache_compact failed")
        return r

    def topk(self, queries: np.ndarray, k: int):
        q = np.ascontiguousarray(queries, dtype=np.float32)
        idx = np.empty((q.shape[0], k), dtype=np.int32)
        sc = np.empty((q.shape[0], k), dtype=np.float32)
        if lib().sr_cache_topk(self._h, _p(q), q.shape[0], k, _p(idx), _p(sc)) != 0:
            raise SrError("sr_cache_topk failed")
        return idx, sc


    def lookup_ids(self, model: "Model", seqs: Sequence[np.ndarray], k: int, target_layer: int = 0):
        """Embed + scan in one call (the embedding stays on the device): pkg/cache/inmemory_cache_search.go:27-176."""
        ids, cu = pack(seqs)
        b = len(cu) - 1
        idx = np.empty((b, k), dtype=np.int32)
        sc = np.empty((b, k), dtype=np.float32)
        if lib().sr_cache_lookup_ids(model.handle, self._h, _p(ids), _p(cu), b, target_layer, k, _p(idx), _p(sc)) != 0:
            raise _err("sr_cache_lookup_ids")
        return idx, sc


def merge_topk(idx_parts: List[np.ndarray], score_parts: List[np.ndarray]):
    g = len(idx_parts)
    b, k = idx_parts[0].shape
    ip = np.ascontiguousarray(np.stack(idx_parts), dtype=np.int32)
    sp = np.ascontiguousarray(np.stack(score_parts), dtype=np.float32)
    oi = np.empty((b, k), dtype=np.int32)
    os_ = np.empty((b, k), dtype=np.float32)
    if lib().sr_cache_merge_topk(_p(ip), _p(sp), g, b, k, _p(oi), _p(os_)) != 0:
        raise SrError("sr_cache_merge_topk failed")
    return oi, os_
