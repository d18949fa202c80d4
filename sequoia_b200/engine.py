"""Inference engines with the reference's class API (Engine/Engine.py) on sequoia_b200 kernels.

InferenceEngine / GraphInferenceEngine  = draft  ("FI": attends the whole static cache under a dense (w, M) mask)
InferenceEngineTG / GraphInferenceEngineTG = target ("TG": attends kv_len = kv_offset + w slots, mask (w, kv_len)).

Same constructors, attributes (.engine.max_length, .engine.kv_cache, .dtype, .device ...) and methods as the
reference, so Tree/SpecTree.py-style callers and tests/testbed.py drop in.  Tree objects of this package bypass the
dense-mask API and call ``engine.engine.runner.forward`` with the packed tree mask + device state (see tree.py).
"""
from __future__ import annotations

import gc
from typing import List, Optional

import torch

from .kv import MAX_BATCH, KV_Cache
from .model import LlamaRunner

F16 = torch.float16


def _prep_mask(attention_mask: torch.Tensor, n: int):
    if attention_mask.dtype != F16:
        raise TypeError(f"attention mask must be float16 (got {attention_mask.dtype}); Tree hard-codes fp16 masks "
                        "(Tree/Tree.py:4)")
    m = attention_mask
    while m.dim() > 2:
        m = m[0]
    if m.stride(-1) != 1:
        m = m.contiguous()
    assert m.shape[0] == n
    return m


def _check_batch(batch_size: int, tp_group):
    if not 1 <= batch_size <= MAX_BATCH:
        raise ValueError(f"batch_size must be in 1..{MAX_BATCH}, got {batch_size}")
    if batch_size > 1 and tp_group is not None:
        raise NotImplementedError("a batch of several sequences runs on one GPU: tensor parallelism needs batch_size=1")


class InferenceEngine:
    """Engine/Engine.py:8-60 (draft).  batch_size > 1: caches and activations for that many sequences
    (sequoia_b200.batch.BatchTree); the dense-mask methods then refuse, they address one sequence."""

    _TG = False

    def __init__(self, max_length: int, model_name_or_path, dtype=torch.float16, device="cuda:0", tp_group=None,
                 batch_size: int = 1):
        _check_batch(batch_size, tp_group)
        if dtype != torch.float16:
            raise NotImplementedError("sequoia_b200 engines are fp16 (reference default)")
        self.device = device
        self.dtype = dtype
        self.max_length = max_length
        self.batch_size = batch_size
        self.runner = LlamaRunner(model_name_or_path, max_length, device=device, tp_group=tp_group, batch_size=batch_size)
        self.model = self.runner                      # reference attribute name
        self.model_config = self.runner.cfg
        self.kv_cache = KV_Cache(config=self.model_config, batch_size=batch_size, max_length=max_length, device=device,
                                 dtype=dtype, k_cache=self.runner.k_cache, v_cache=self.runner.v_cache)

    def _single(self, what: str):
        if self.batch_size != 1:
            raise RuntimeError(f"{what} takes one sequence's dense mask; this engine holds a batch of {self.batch_size} "
                               "(drive it through sequoia_b200.batch.BatchTree)")

    @torch.inference_mode()
    def model_run(self, input_ids: torch.LongTensor, storage_ids: torch.LongTensor,
                  attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.LongTensor] = None,
                  debug: bool = False):
        self._single("model_run")
        n = input_ids.shape[1]
        if debug:
            assert storage_ids.shape[0] == n
            assert attention_mask.shape[-2] == n
            assert position_ids.shape[1] == n
        ids = input_ids.reshape(-1).contiguous()
        pos = position_ids.reshape(-1).contiguous()
        sto = storage_ids.contiguous()
        mask = _prep_mask(attention_mask, n)
        if self._TG:
            kv_len = self.kv_cache.kv_offset + n
            if tuple(attention_mask.shape) != (1, 1, n, kv_len):       # Engine/Llama_modules.py:238-242
                raise ValueError(f"Attention mask should be of size {(1, 1, n, kv_len)}, but is {tuple(attention_mask.size())}")
        else:
            kv_len = self.max_length
            if mask.shape[-1] != self.max_length:
                raise ValueError(f"Attention mask should have {self.max_length} columns, but is {tuple(attention_mask.size())}")
        out = self.runner.forward(n, ids, pos, sto, kv_end=kv_len, dense_mask=mask, mask_ld=mask.stride(0))
        self.kv_cache.kv_offset += n                                    # Llama_KV.py:87-88
        return out.clone().view(1, n, -1)

    def clear_kv(self):
        self.kv_cache.clear()

    def initialize_kv(self, k_cache: torch.Tensor, v_cache: torch.Tensor, kv_len: int):
        self.kv_cache.initialize_kv(k_cache, v_cache, kv_len)

    def gather_kv(self, indices: List[int]):
        self._single("gather_kv")
        self.kv_cache.gather_kv(indices)

    def get_kv_cache(self, in_place=False):
        if not in_place:
            return self.kv_cache.k_cache.clone(), self.kv_cache.v_cache.clone()
        return self.kv_cache.k_cache, self.kv_cache.v_cache


class InferenceEngineTG(InferenceEngine):
    """Engine/Engine.py:62-125 (target).  `offloading` is accepted and ignored: the weights stay resident in device memory."""

    _TG = True

    def __init__(self, max_length: int, model_name_or_path, dtype=torch.float16, device="cuda:0", offloading=False,
                 tp_group=None, batch_size: int = 1):
        super().__init__(max_length, model_name_or_path, dtype=dtype, device=device, tp_group=tp_group,
                         batch_size=batch_size)
        self.offloading = offloading

    def set_kv_len(self, kv_len: int):
        self.kv_cache.set_kv_len(kv_len)


def capture_graph(engine: InferenceEngine, decoding_seqlen: int = 1, mempool=None, n_warmups: int = 3):
    """Engine/Engine.py:127-166: static inputs, warm-up on a side stream, capture model_run, replay closure."""
    device = engine.device
    dtype = engine.dtype
    static_input_ids = torch.full((1, decoding_seqlen), 0, dtype=torch.long, device=device)
    static_position_ids = torch.full((1, decoding_seqlen), 0, dtype=torch.long, device=device)
    static_storage_ids = torch.arange(decoding_seqlen, dtype=torch.long, device=device)
    static_attn_mask = torch.full((decoding_seqlen, engine.max_length), 0, dtype=dtype, device=device)[None, None, :, :]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(n_warmups):
            static_logits = engine.model_run(input_ids=static_input_ids, storage_ids=static_storage_ids,
                                             position_ids=static_position_ids, attention_mask=static_attn_mask)
        s.synchronize()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, pool=mempool):
        static_logits = engine.model_run(input_ids=static_input_ids, storage_ids=static_storage_ids,
                                         position_ids=static_position_ids, attention_mask=static_attn_mask)

    def run(input_ids, storage_ids, position_ids, attn_mask):
        static_input_ids.copy_(input_ids)
        static_storage_ids.copy_(storage_ids)
        static_position_ids.copy_(position_ids)
        static_attn_mask.copy_(attn_mask)
        graph.replay()
        return static_logits.clone()

    return run


class GraphInferenceEngine:
    """Engine/Engine.py:168-244."""

    def __init__(self, max_length: int, model_name_or_path, dtype=torch.float16, device="cuda:0", tp_group=None,
                 batch_size: int = 1):
        _check_batch(batch_size, tp_group)
        self.device = device
        self.dtype = dtype
        self.max_length = max_length
        self.engine = InferenceEngine(max_length=max_length, model_name_or_path=model_name_or_path, dtype=dtype,
                                      device=device, tp_group=tp_group, batch_size=batch_size)
        self.callables = {}
        self.mempool = None

    @torch.inference_mode()
    def initialize_cuda_graph(self, decoding_seqlens: List[int], n_warmups=3):
        self.engine._single("initialize_cuda_graph")
        gc.collect()
        self.mempool = torch.cuda.graphs.graph_pool_handle()
        for decoding_seqlen in decoding_seqlens:
            if decoding_seqlen not in self.callables and decoding_seqlen != 0:
                self.callables[decoding_seqlen] = capture_graph(engine=self.engine, decoding_seqlen=decoding_seqlen,
                                                                mempool=self.mempool, n_warmups=n_warmups)
        self.engine.clear_kv()

    @torch.inference_mode()
    def graph_inference(self, input_ids: torch.LongTensor, storage_ids: torch.LongTensor,
                        position_ids: Optional[torch.LongTensor] = None, attn_mask: Optional[torch.Tensor] = None,
                        debug: bool = False):
        dec_length = input_ids.shape[1]
        if debug:
            assert input_ids.shape[0] == 1
            assert storage_ids.shape[0] == dec_length
            assert position_ids.shape[0] == 1 and position_ids.shape[1] == dec_length
            assert attn_mask.shape[2] == dec_length and attn_mask.shape[3] == self.engine.max_length
            assert attn_mask.shape[0] == 1 and attn_mask.shape[1] == 1
        if dec_length in self.callables:
            return self.callables[dec_length](input_ids, storage_ids, position_ids, attn_mask)
        return self.inference(input_ids, storage_ids, position_ids, attn_mask)

    def clear_kv(self):
        self.engine.clear_kv()

    def initialize_kv(self, k_cache: torch.Tensor, v_cache: torch.Tensor, kv_len: int):
        self.engine.initialize_kv(k_cache, v_cache, kv_len)

    def get_kv_cache(self, in_place=False):
        return self.engine.get_kv_cache(in_place=in_place)

    def gather_kv(self, indices: List[int]):
        self.engine.gather_kv(indices)

    @torch.inference_mode()
    def inference(self, input_ids: torch.LongTensor, storage_ids: torch.LongTensor,
                  position_ids: Optional[torch.LongTensor] = None, attn_mask: Optional[torch.Tensor] = None):
        return self.engine.model_run(input_ids=input_ids, storage_ids=storage_ids, attention_mask=attn_mask,
                                     position_ids=position_ids)


class GraphInferenceEngineTG:
    """Engine/Engine.py:247-289."""

    def __init__(self, max_length: int, model_name_or_path, dtype=torch.float16, device="cuda:0", offloading=False,
                 tp_group=None, batch_size: int = 1):
        _check_batch(batch_size, tp_group)
        self.device = device
        self.dtype = dtype
        self.max_length = max_length
        self.engine = InferenceEngineTG(max_length=max_length, model_name_or_path=model_name_or_path, dtype=dtype,
                                        device=device, offloading=offloading, tp_group=tp_group, batch_size=batch_size)

    def clear_kv(self):
        drv = getattr(self, "_tp_driver", None)
        if drv is not None:
            drv.send_ctrl(3)                             # OP_CLEAR: follower ranks clear their shards too
        self.engine.clear_kv()

    def initialize_kv(self, k_cache: torch.Tensor, v_cache: torch.Tensor, kv_len: int):
        self.engine.initialize_kv(k_cache, v_cache, kv_len)

    def get_kv_cache(self, in_place=False):
        return self.engine.get_kv_cache(in_place=in_place)

    def gather_kv(self, indices: List[int]):
        self.engine.gather_kv(indices)

    def set_kv_len(self, kv_len: int):
        self.engine.set_kv_len(kv_len)

    @torch.no_grad()
    def inference(self, input_ids: torch.LongTensor, storage_ids: torch.LongTensor,
                  position_ids: Optional[torch.LongTensor] = None, attn_mask: Optional[torch.Tensor] = None):
        return self.engine.model_run(input_ids=input_ids, storage_ids=storage_ids, attention_mask=attn_mask,
                                     position_ids=position_ids)


class OffloadEngine(GraphInferenceEngineTG):
    """Engine/offload_engine.py:416-451 surface.  The reference streams a 70B target from host memory because it
    does not fit an L40.  Here the weights stay resident (a 70B target fits 80 GB GPUs only TP-sharded, e.g. over 8
    ranks), so this is the TG engine."""

    def __init__(self, max_length: int, model_name_or_path, dtype=torch.float16, device="cuda:0", stay_layers=None,
                 tp_group=None):
        super().__init__(max_length, model_name_or_path, dtype=dtype, device=device, offloading=True, tp_group=tp_group)
