"""Static KV cache with the reference's interface (Engine/Llama_KV.py:4-103) on sequoia_b200 kernels."""
from __future__ import annotations

from typing import List, Optional

import torch

from . import ops

MAX_BATCH = 8            # SQ_MAX_BATCH (include/sequoia_b200.h)


class KV_Cache:
    """(L, B, H_kv, M, D) K and V; scatter by storage ids, accepted-path gather / compaction.  B = batch_size sequences
    (sequoia_b200.batch); the host-index methods (initialize_kv, gather_kv*) serve B = 1 only.

    Mirrors Engine/Llama_KV.py: same constructor, attributes (k_cache, v_cache, kv_offset, num_layers,
    max_length) and methods.  `k_cache` / `v_cache` may be handed in preallocated (the engine binds its TMA
    descriptors to them)."""

    def __init__(self, config, batch_size: int = 1, max_length: int = 256, device="cuda:0", dtype=torch.float16,
                 k_cache: Optional[torch.Tensor] = None, v_cache: Optional[torch.Tensor] = None):
        if dtype != torch.float16:
            raise NotImplementedError("sequoia_b200 kernels are fp16 (the reference default dtype)")
        if not 1 <= batch_size <= MAX_BATCH:
            raise ValueError(f"batch_size must be in 1..{MAX_BATCH}, got {batch_size}")
        self.batch_size = batch_size
        self.config = config
        self.max_length = max_length
        self.device = device
        self.dtype = dtype
        if k_cache is None:
            shape = (config.num_hidden_layers, batch_size, config.num_key_value_heads, max_length,
                     config.hidden_size // config.num_attention_heads)
            k_cache = torch.zeros(shape, device=device, dtype=dtype)
            v_cache = torch.zeros(shape, device=device, dtype=dtype)
        self.k_cache, self.v_cache = k_cache, v_cache
        self.num_layers = k_cache.shape[0]
        self.kv_offset = 0

    # Llama_KV.py:38-46
    def initialize_kv(self, k_cache: torch.Tensor, v_cache: torch.Tensor, kv_len: int):
        self._single("initialize_kv")
        self.k_cache[..., :kv_len, :].copy_(k_cache[..., :kv_len, :])
        self.v_cache[..., :kv_len, :].copy_(v_cache[..., :kv_len, :])
        self.kv_offset = kv_len

    def _single(self, what: str):
        if self.batch_size != 1:
            raise RuntimeError(f"KV_Cache.{what} addresses one sequence; this cache holds {self.batch_size} "
                               "(a batch compacts through ops.kv_gather_batch)")

    def _gather(self, indices: List[int], offset: int, zero_tail: bool = True):
        self._single("gather_kv")
        n = len(indices)
        idx = torch.tensor(list(indices), dtype=torch.int32).to(self.k_cache.device, non_blocking=False) if n else None
        if n:
            assert min(indices) >= 0 and max(indices) < self.max_length
        if n * self.k_cache.shape[-1] * 2 > 200 * 1024:      # too many rows to stage on chip: scratch path (any length)
            ops.kv_gather_big(self.k_cache, self.v_cache, idx, n, offset, zero_tail=zero_tail)
        else:
            ops.kv_gather(self.k_cache, self.v_cache, idx, n, offset, zero_tail=zero_tail)
        self.kv_offset = offset + n

    # Llama_KV.py:50-58
    def gather_kv(self, indices: List[int]):
        self._gather(indices, 0)

    # Llama_KV.py:60-68 (bit-exact incl. the zeroed tail).  Tree objects use the device-driven variant below.
    def gather_kv_incremental(self, indices: List[int], offset: int):
        self._gather(indices, offset)

    def gather_from_state(self, accept_idx: torch.Tensor, state: torch.Tensor, max_n: int, zero_tail: bool = False):
        """Graph-static compaction: n = state[N_NEW], offset = state[P_OLD], indices = accept_idx (device int32).
        The caller updates kv_offset once it has read the accept length back.  Unlike Llama_KV.py:65-66 the tail rows
        (>= offset + n) are left stale here: every consumer of this path uses the packed tree mask, under which rows
        >= kv_len are never visible (the reference-API gather_kv* methods above do zero the tail, bit-exact)."""
        self._single("gather_from_state")
        ops.kv_gather(self.k_cache, self.v_cache, accept_idx, 0, 0, state=state, max_n=max_n, zero_tail=zero_tail)

    # Llama_KV.py:72-89 (kept for API completeness; the engine's forward appends K/V inside its RoPE kernel)
    def update_kv_cache(self, new_k_cache: torch.Tensor, new_v_cache: torch.Tensor, layer_idx: int,
                        storage_ids: torch.LongTensor, debug: bool = False):
        self._single("update_kv_cache")
        input_length = len(storage_ids)
        if debug:
            assert input_length == new_k_cache.shape[-2]
            assert input_length == new_v_cache.shape[-2]
        self.k_cache[layer_idx].index_copy_(dim=-2, index=storage_ids, source=new_k_cache)
        self.v_cache[layer_idx].index_copy_(dim=-2, index=storage_ids, source=new_v_cache)
        if layer_idx == self.num_layers - 1:
            self.kv_offset += input_length
        return self.k_cache[layer_idx], self.v_cache[layer_idx]

    # Llama_KV.py:91-94
    def clear(self):
        self.k_cache.zero_()
        self.v_cache.zero_()
        self.kv_offset = 0

    # Llama_KV.py:96-100
    def get_usable_length(self, layer_idx: int, input_length: int):
        if layer_idx == self.num_layers - 1:
            return self.kv_offset
        return self.kv_offset + input_length

    # Llama_KV.py:102-103
    def set_kv_len(self, kv_len: int):
        self.kv_offset = kv_len
