"""Drop-in attention backend for `chitu.attn_backend` (reference: chitu/attn_backend.py).

`B200AttnBackend` implements the four methods the models call (SURVEY.md §8b):
prepare_metadata_for_decode, attn_varlen_func (prefill: the absorbed-MLA form runs the sm_90a
prefill kernel; GQA prefill stays on flash_attn / torch SDPA), attn_with_kvcache (GQA attention over the KV cache
with in-place append: the decode kernel for seqlen_q == 1, the sm_90a multi-token kernel for seqlen_q > 1 — chunked
prefill, prefill on a cached prefix, speculative verification; over the paged cache with a block_table, in the io dtype
or in fp8 e4m3 (half the KV bytes), and over the non-paged [B, S, Hkv, D] cache of KVCacheManager without one) and
mla_attn_with_kvcache (absorbed-MLA attention over the paged latent cache, in bf16 or fp8 e4m3: the decode kernel with
fused append for one query token per request, the sm_90a multi-token kernel for seqlen_q > 1 — multi-token-prediction
verification, chunked prefill on a cached prefix).
"""
from __future__ import annotations

import math
from typing import Optional, Union

import torch

from . import _lib, workspace
from ._lib import check, current_stream, dtype_code, ptr, require_cuda

__all__ = ["AttnBackend", "B200AttnBackend"]

_MLA_QK, _MLA_V = 576, 512          # absorbed MLA: kv_lora_rank + qk_rope_head_dim, kv_lora_rank


class AttnBackend:
    """Interface (chitu/attn_backend.py:24-164)."""

    def prepare_metadata_for_decode(self, *args, **kwargs):
        pass

    def attn_varlen_func(self, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                         dropout_p=0.0, causal=False, window_size=(-1, -1), softcap=0.0, softmax_scale=None):
        raise NotImplementedError()

    def attn_with_kvcache(self, q, k_cache, v_cache, k=None, v=None, cache_seqlens=None, cache_leftpad=None,
                          block_table=None, causal=False, window_size=(-1, -1), softcap=0.0, softmax_scale=None):
        raise NotImplementedError()


class B200AttnBackend(AttnBackend):
    """sm_90a decode attention.  Constructor arguments replace the reference's reads of
    `get_global_args()` (attn_backend.py:508-511, 691-695) so the class is usable stand-alone;
    `from_global_args(args)` mirrors the reference construction."""

    def __init__(self, kv_lora_rank: int = 512, qk_rope_head_dim: int = 64, qk_nope_head_dim: int = 128,
                 max_seq_len: Optional[int] = None, max_reqs: Optional[int] = None, n_local_heads: int = 128):
        self.kv_lora_rank = kv_lora_rank
        self.qk_rope_head_dim = qk_rope_head_dim
        self.qk_nope_head_dim = qk_nope_head_dim
        self.max_seq_len = max_seq_len
        self.max_reqs = max_reqs          # infer.max_reqs: the largest decode batch a graph is captured for
        self.n_local_heads = n_local_heads
        self.block_size = None
        self._plan_view = None

    @classmethod
    def from_global_args(cls, args):
        m = args.models
        tp = max(int(getattr(args.infer, "tp_size", 1) or 1), 1)
        return cls(getattr(m, "kv_lora_rank", 512), getattr(m, "qk_rope_head_dim", 64),
                   getattr(m, "qk_nope_head_dim", 128), getattr(args.infer, "max_seq_len", None),
                   getattr(args.infer, "max_reqs", None), max(getattr(m, "n_heads", 128) // tp, 1))

    # -- a1: attn_backend.py:29-30 / 697-705.  Runs outside the CUDA graph (models/model.py:540).
    def prepare_metadata_for_decode(self, cache_seqlens_excl_this_decode, cache_seqlens_incl_this_decode,
                                    block_table, block_size, softmax_scale=None):
        self.block_size = block_size
        B = cache_seqlens_excl_this_decode.shape[0]
        # Persistent split-KV workspace: reserve exactly what `_ws()` will ask for at the LARGEST decode batch
        # (graphs are captured per batch size in arrival order, models/model.py:537-622; a buffer a captured
        # kernel was given is never freed — see workspace.py — so this only avoids a second allocation).
        Bmax = max(B, self.max_reqs or 0, 1)
        workspace.reserve("attn", workspace.attn_bytes(Bmax, self.n_local_heads, max(self.kv_lora_rank, 128)),
                          block_table.device)
        # a1 proper: the length-aware split-KV plan of this step, computed ON THE DEVICE from the step's lengths (the
        # reference's FlashInfer variant does O(B) .item() syncs here, attn_backend.py:620-637; FlashMLA runs
        # get_mla_metadata).  The MLA decode kernel finds it at the end of the attention workspace.
        if block_size == 64 and B > 0 and torch.is_tensor(cache_seqlens_incl_this_decode):
            H = self.n_local_heads
            buf, n = self._ws(B, H, max(self.kv_lora_rank, 128), block_table.device)
            hint = self.max_seq_len if self.max_seq_len else block_table.shape[1] * block_size
            check(_lib.load().chitu_b200_attn_plan(ptr(cache_seqlens_incl_this_decode), B, H, block_size, int(hint), ptr(buf), n,
                                                   current_stream()), "attn_plan")
            self._plan_view = buf[n - _lib.ATTN_PLAN_BYTES:].view(torch.int32)

    def last_plan(self):
        """int32 view of the device-side split plan written by the last prepare_metadata_for_decode (tests / debugging)."""
        return self._plan_view

    def _ws(self, B, H, DV, device):
        buf = workspace.get("attn", workspace.attn_bytes(B, H, DV), device)
        return buf, buf.numel()

    # -- prefill (SURVEY §8f n4).  attn_backend.py:193-206 (FlashAttnBackend), flash_attn_varlen_func semantics.
    def attn_varlen_func(self, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                         dropout_p=0.0, causal=False, window_size=(-1, -1), softcap=0.0, softmax_scale=None):
        """Varlen prefill attention.  The absorbed-MLA form DeepSeek's prefill calls (model_deepseek_v3.py:588-602):
        bf16 q [Tq, H, 576], k [Tk, 1, 576], v [Tk, 1, 512], no dropout / window / softcap, runs the sm_90a kernel
        (chitu_b200_mla_prefill): no host synchronisation, capturable in a CUDA graph, deterministic; returns
        [Tq, H, 512].  softmax_scale=None means 1/sqrt(576).  Every other shape (GQA prefill) takes flash_attn, or
        torch SDPA per sequence when flash_attn is not installed."""
        if (q.dtype == k.dtype == v.dtype == torch.bfloat16 and q.dim() == 3 and q.shape[-1] == _MLA_QK
                and k.dim() == 3 and tuple(k.shape[1:]) == (1, _MLA_QK) and v.dim() == 3
                and tuple(v.shape[1:]) == (1, _MLA_V) and dropout_p == 0.0 and tuple(window_size) == (-1, -1)
                and softcap == 0.0):
            return self._mla_prefill(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, causal, softmax_scale)
        return self._attn_varlen_library(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p,
                                         causal, window_size, softcap, softmax_scale)

    @staticmethod
    def _mla_prefill(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, causal, softmax_scale):
        require_cuda(q, k, v, cu_seqlens_q, cu_seqlens_k)
        assert q.is_contiguous() and k.stride(-1) == 1 and v.stride(-1) == 1
        assert cu_seqlens_q.dtype == torch.int32 and cu_seqlens_k.dtype == torch.int32
        assert cu_seqlens_q.is_contiguous() and cu_seqlens_k.is_contiguous()
        assert cu_seqlens_q.numel() == cu_seqlens_k.numel() >= 1
        Tq, H, _ = q.shape
        out = torch.empty((Tq, H, _MLA_V), dtype=q.dtype, device=q.device)
        scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(_MLA_QK)
        check(_lib.load().chitu_b200_mla_prefill(
            ptr(q), ptr(k), k.stride(0), ptr(v), v.stride(0), ptr(cu_seqlens_q), ptr(cu_seqlens_k),
            cu_seqlens_q.numel() - 1, H, Tq, k.shape[0], int(max_seqlen_q), int(bool(causal)), float(scale), ptr(out),
            current_stream()), "mla_prefill")
        return out

    # Exactly what the reference's FlashAttnBackend does (attn_backend.py:193-206): flash_attn_varlen_func when the
    # library is importable; otherwise torch's fused SDPA per sequence (no [H, Tq, Tk] fp32 score tensor, no host loop
    # over heads).  Both are library calls on a path this repository does not optimise (GQA prefill).
    @staticmethod
    def _attn_varlen_library(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                             dropout_p=0.0, causal=False, window_size=(-1, -1), softcap=0.0, softmax_scale=None):
        assert dropout_p == 0.0
        if q.dtype in (torch.float16, torch.bfloat16) and q.shape[-1] <= 256 and k.shape[-1] == v.shape[-1]:
            try:
                import flash_attn
                extra = {"softcap": softcap} if softcap != 0.0 else {}
                return flash_attn.flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                                                         dropout_p=0.0, causal=causal, window_size=window_size,
                                                         softmax_scale=softmax_scale, **extra)
            except ImportError:
                pass
        assert window_size == (-1, -1) and softcap == 0.0
        out = torch.empty((q.shape[0], q.shape[1], v.shape[-1]), dtype=q.dtype, device=q.device)
        scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(q.shape[-1])
        cq, ck = cu_seqlens_q.tolist(), cu_seqlens_k.tolist()            # one sync per prefill batch
        for i in range(len(cq) - 1):
            qi = q[cq[i]:cq[i + 1]].transpose(0, 1).unsqueeze(0)         # [1, Hq, Tq, D]
            ki = k[ck[i]:ck[i + 1]].transpose(0, 1).unsqueeze(0)
            vi = v[ck[i]:ck[i + 1]].transpose(0, 1).unsqueeze(0)
            tq, tk = qi.shape[2], ki.shape[2]
            mask = None
            if causal and tq != tk:                                      # bottom-right aligned causal mask (flash_attn semantics)
                mask = torch.ones(tq, tk, dtype=torch.bool, device=q.device).tril(diagonal=tk - tq)
            oi = torch.nn.functional.scaled_dot_product_attention(qi, ki, vi, attn_mask=mask, is_causal=causal and tq == tk,
                                                                  scale=scale, enable_gqa=qi.shape[1] != ki.shape[1])
            out[cq[i]:cq[i + 1]] = oi[0].transpose(0, 1)
        return out

    # -- a5: attn_backend.py:92-164 (FlashAttn impl :208-243)
    def attn_with_kvcache(self, q, k_cache, v_cache, k=None, v=None,
                          cache_seqlens: Optional[Union[int, torch.Tensor]] = None,
                          cache_leftpad: Optional[torch.Tensor] = None,
                          block_table: Optional[torch.Tensor] = None, causal=False, window_size=(-1, -1),
                          softcap=0.0, softmax_scale=None):
        """GQA attention over the KV cache with the in-place append of k / v (flash_attn_with_kvcache semantics).
        q [B, sq, Hq, D]; with block_table the caches are paged [num_blocks, page, Hkv, D], without it [Bc, S, Hkv, D].
        A paged cache in torch.float8_e4m3fn (both caches) runs the e4m3 kernels; otherwise the caches are in q's dtype."""
        fp8 = (k_cache.dtype == torch.float8_e4m3fn, v_cache.dtype == torch.float8_e4m3fn)
        if fp8[0] != fp8[1]:
            raise RuntimeError("attn_with_kvcache: k_cache and v_cache must have the same dtype")
        if block_table is None:
            if fp8[0]:
                raise RuntimeError("attn_with_kvcache: the fp8 KV cache is built for the paged cache only")
            return self._contiguous(q, k_cache, v_cache, k, v, cache_seqlens, cache_leftpad, causal, window_size,
                                    softcap, softmax_scale)
        assert cache_leftpad is None and window_size == (-1, -1) and softcap == 0.0
        require_cuda(q, k_cache, v_cache, block_table)
        return self._paged(q, k_cache, v_cache, k, v, cache_seqlens, block_table, causal, softmax_scale, fp8[0])

    @staticmethod
    def _seqlens(q, cache_seqlens):
        """cache_seqlens as a tensor on q's device: an int stands for every request."""
        if not torch.is_tensor(cache_seqlens):
            cache_seqlens = torch.full((q.shape[0],), int(cache_seqlens), dtype=torch.int32, device=q.device)
        return cache_seqlens

    def _kv_args(self, q, k, v, Hkv, cache_seqlens, softmax_scale, cache_keys):
        """What both cache layouts check and pass: cache_seqlens (a tensor, see _seqlens) int32 and contiguous, the
        new k / v rows [B, sq, Hkv, D] in q's dtype as their strides (k_sb, k_st, v_sb, v_st) (zeros without them),
        the softmax scale (default 1/sqrt(D)) and the length hint (max_seq_len, else the keys the cache holds)."""
        B, sq, _, D = q.shape
        assert cache_seqlens.dtype == torch.int32 and cache_seqlens.is_contiguous()
        strides = (0, 0, 0, 0)
        if k is not None:
            assert v is not None and k.shape == (B, sq, Hkv, D) and v.shape == (B, sq, Hkv, D)
            assert k.dtype == v.dtype == q.dtype
            # heads must be dense; the batch and token strides are free (views into a fused qkv GEMM output)
            assert k.stride(-1) == 1 and k.stride(-2) == D and v.stride(-1) == 1 and v.stride(-2) == D
            strides = (k.stride(0), k.stride(1), v.stride(0), v.stride(1))
        scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
        hint = self.max_seq_len if self.max_seq_len else cache_keys
        return strides, float(scale), int(hint)

    def _paged(self, q, k_cache, v_cache, k, v, cache_seqlens, block_table, causal, softmax_scale, fp8):
        """Paged caches [num_blocks, page, Hkv, D]: the sq new k / v rows are appended at cache_seqlens[b] + i (true
        page indexing), then query i attends to the first cache_seqlens[b] + sq keys (without k / v:
        cache_seqlens[b]), bottom-right causal when `causal`.  sq == 1 runs the decode kernel
        (chitu_b200_gqa_paged_decode), sq > 1 the multi-token kernel (chitu_b200_gqa_paged_prefill: chunked prefill,
        prefill on a cached prefix, speculative verification).
        `fp8`: e4m3 caches, sq >= 1 (chitu_b200_gqa_paged_attn_fp8kv): the same semantics, with each new k / v element
        stored as x.float().clamp(-448, 448).to(float8_e4m3fn) and each cache element decoded exactly to q's dtype
        (bf16 | fp16) before the unchanged arithmetic.  The appended rows are attended in their stored form.  No scale.
        Built for D == 128, Hq / Hkv in {1, 2, 4, 8} and a power-of-two page that is a multiple of 64; no host
        synchronisation, capturable in a CUDA graph, deterministic."""
        B, sq, Hq, D = q.shape
        num_blocks, page, Hkv, Dk = k_cache.shape
        assert Dk == D and v_cache.shape == k_cache.shape
        if fp8:
            assert q.dtype in (torch.bfloat16, torch.float16)
        else:
            assert k_cache.dtype == v_cache.dtype == q.dtype
        assert q.is_contiguous() and k_cache.is_contiguous() and v_cache.is_contiguous()
        assert block_table.dtype == torch.int32 and block_table.stride(-1) == 1
        cache_seqlens = self._seqlens(q, cache_seqlens)
        strides, scale, hint = self._kv_args(q, k, v, Hkv, cache_seqlens, softmax_scale, block_table.shape[1] * page)
        out = torch.empty_like(q)
        ws, wsn = self._ws(B, Hq, D, q.device)
        lib, bt = _lib.load(), (ptr(block_table), block_table.stride(0))
        if fp8:
            check(lib.chitu_b200_gqa_paged_attn_fp8kv(
                ptr(q), sq * Hq * D, ptr(k_cache), ptr(v_cache), ptr(k), ptr(v), *strides, None, None,
                ptr(cache_seqlens), *bt, B, sq, Hq, Hkv, D, page, num_blocks, hint, int(bool(causal)), scale, ptr(out),
                ptr(ws), wsn, dtype_code(q.dtype), current_stream()), "gqa_paged_attn_fp8kv")
        elif sq == 1:
            check(lib.chitu_b200_gqa_paged_decode(
                ptr(q), ptr(k_cache), ptr(v_cache), ptr(k), ptr(v), strides[0], strides[2], ptr(cache_seqlens), *bt, B,
                Hq, Hkv, D, page, hint, scale, ptr(out), ptr(ws), wsn, dtype_code(q.dtype), current_stream()),
                "gqa_paged_decode")
        else:
            check(lib.chitu_b200_gqa_paged_prefill(
                ptr(q), ptr(k_cache), ptr(v_cache), ptr(k), ptr(v), *strides, ptr(cache_seqlens), *bt, B, sq, Hq, Hkv,
                D, page, num_blocks, hint, int(bool(causal)), scale, ptr(out), ptr(ws), wsn, dtype_code(q.dtype),
                current_stream()), "gqa_paged_prefill")
        return out

    def _contiguous(self, q, k_cache, v_cache, k, v, cache_seqlens, cache_leftpad, causal, window_size, softcap,
                    softmax_scale):
        """No block table (chitu_b200_gqa_contiguous_attn): k_cache / v_cache [Bc, S, Hkv, D] with Bc >= B, request b
        on cache row b; the sq new k / v rows are appended at cache_seqlens[b] + i, then query i attends to the first
        cache_seqlens[b] + sq keys (without k / v: cache_seqlens[b]), bottom-right causal when `causal`.  A new row at a
        position >= S is not written and no key >= S is read.  sq == 1 and sq > 1 alike; no host synchronisation,
        capturable in a CUDA graph, deterministic."""
        if cache_leftpad is not None or tuple(window_size) != (-1, -1) or softcap != 0.0:
            raise RuntimeError("gqa_contiguous_attn: cache_leftpad, window_size and softcap are not built")
        cache_seqlens = self._seqlens(q, cache_seqlens)
        require_cuda(q, k_cache, v_cache, k, v, cache_seqlens)
        B, sq, Hq, D = q.shape
        Bc, S, Hkv, Dk = k_cache.shape
        cst = k_cache.stride()
        assert v_cache.shape == k_cache.shape and v_cache.stride() == cst and cst[1:] == (Hkv * D, D, 1)
        assert Dk == D and Bc >= B and k_cache.dtype == v_cache.dtype == q.dtype and q.is_contiguous()
        strides, scale, hint = self._kv_args(q, k, v, Hkv, cache_seqlens, softmax_scale, S)
        out = torch.empty_like(q)
        ws, wsn = self._ws(B, Hq, D, q.device)
        check(_lib.load().chitu_b200_gqa_contiguous_attn(
            ptr(q), ptr(k_cache), ptr(v_cache), cst[0], S, ptr(k), ptr(v), *strides, ptr(cache_seqlens), B, sq,
            Hq, Hkv, D, hint, int(bool(causal)), scale, ptr(out), ptr(ws), wsn, dtype_code(q.dtype),
            current_stream()), "gqa_contiguous_attn")
        return out

    # -- a2: attn_backend.py:707-774 (Triton), :536-572 (FlashMLA), :660-684 (FlashInfer)
    def mla_attn_with_kvcache(self, q_nope, q_pe, kv_cache, kv,
                              cache_seqlens_excl_this_decode: Union[int, torch.Tensor],
                              cache_seqlens_incl_this_decode: Union[int, torch.Tensor],
                              block_table: torch.Tensor, causal=True, window_size=(-1, -1), softcap=0.0,
                              softmax_scale=None):
        """Absorbed-MLA attention over the paged latent cache.  q_nope [B, H, C] (or [B, 1, H, C]): one decode token
        per request with the fused append of `kv` (chitu_b200_mla_decode), returned as [B, 1, H, C].
        q_nope [B, sq, H, C] with sq > 1: multi-token-prediction verification or chunked prefill, see
        `_mla_paged_prefill`.  A kv_cache in torch.float8_e4m3fn takes both call shapes through `_mla_fp8kv`."""
        require_cuda(q_nope, q_pe, kv_cache, block_table)
        if kv_cache.dtype == torch.float8_e4m3fn:
            return self._mla_fp8kv(q_nope, q_pe, kv_cache, kv, cache_seqlens_excl_this_decode, block_table, causal,
                                   window_size, softcap, softmax_scale)
        if q_nope.dim() == 4:
            B, sq, H, C = q_nope.shape
            if sq > 1:
                return self._mla_paged_prefill(q_nope, q_pe, kv_cache, kv, cache_seqlens_excl_this_decode, block_table,
                                               causal, window_size, softcap, softmax_scale)
            q_nope, q_pe = q_nope.view(B, H, C), q_pe.view(B, H, q_pe.shape[-1])
        assert kv_cache.ndim == 3  # (num_blocks, block_size, dim)
        B, H, C = q_nope.shape
        R = q_pe.shape[-1]
        page = kv_cache.size(1)
        assert kv_cache.size(2) == C + R
        assert q_nope.is_contiguous() and q_pe.is_contiguous() and kv_cache.is_contiguous()
        assert q_nope.dtype == torch.bfloat16 and kv_cache.dtype == torch.bfloat16
        assert block_table.dtype == torch.int32 and block_table.stride(-1) == 1
        seq_excl = cache_seqlens_excl_this_decode
        assert seq_excl.dtype == torch.int32 and seq_excl.is_contiguous()
        new_kv = None
        if kv is not None:
            new_kv = kv.reshape(B, C + R)
            assert new_kv.is_contiguous()
        if softmax_scale is None:
            softmax_scale = 1.0 / ((self.qk_rope_head_dim + self.qk_nope_head_dim) ** 0.5)
        o = torch.empty(B, H, C, dtype=q_nope.dtype, device=q_nope.device)
        ws, wsn = self._ws(B, H, C, q_nope.device)
        hint = self.max_seq_len if self.max_seq_len else block_table.shape[1] * page
        check(_lib.load().chitu_b200_mla_decode(
            ptr(q_nope), ptr(q_pe), ptr(kv_cache), ptr(new_kv), ptr(seq_excl), ptr(block_table),
            block_table.stride(0), B, H, C, R, page, kv_cache.size(0), int(hint), float(softmax_scale), ptr(o), ptr(ws), wsn,
            current_stream()), "mla_decode")
        return o.view(B, 1, H, -1)

    def _mla_paged_prefill(self, q_nope, q_pe, kv_cache, kv, seq_excl, block_table, causal, window_size, softcap,
                           softmax_scale):
        """sq > 1 query tokens per request (chitu_b200_mla_paged_prefill): the B * sq rows of `kv` ([B, sq, C + R] in
        any contiguous shape, or None) are appended at seq_excl[b] + i, then query i attends to the first
        seq_excl[b] + sq keys (without kv: seq_excl[b]), bottom-right causal when `causal`.  The decode arithmetic and
        default scale; returns [B, sq, H, C] bf16.  No host synchronisation, capturable in a CUDA graph, deterministic."""
        if tuple(window_size) != (-1, -1) or softcap != 0.0:
            raise RuntimeError("mla_paged_prefill: window_size and softcap are not built")
        B, sq, H, C = q_nope.shape
        R = q_pe.shape[-1]
        assert kv_cache.ndim == 3 and kv_cache.size(2) == C + R and q_pe.shape == (B, sq, H, R)
        assert q_nope.is_contiguous() and q_pe.is_contiguous() and kv_cache.is_contiguous()
        assert q_nope.dtype == q_pe.dtype == kv_cache.dtype == torch.bfloat16
        assert block_table.dtype == torch.int32 and block_table.stride(-1) == 1
        assert seq_excl.dtype == torch.int32 and seq_excl.is_contiguous()
        if kv is not None:
            assert kv.dtype == torch.bfloat16 and kv.is_contiguous() and kv.numel() == B * sq * (C + R)
        if softmax_scale is None:
            softmax_scale = 1.0 / ((self.qk_rope_head_dim + self.qk_nope_head_dim) ** 0.5)
        page = kv_cache.size(1)
        o = torch.empty(B, sq, H, C, dtype=q_nope.dtype, device=q_nope.device)
        ws, wsn = self._ws(B, H, C, q_nope.device)
        hint = self.max_seq_len if self.max_seq_len else block_table.shape[1] * page
        check(_lib.load().chitu_b200_mla_paged_prefill(
            ptr(q_nope), ptr(q_pe), ptr(kv_cache), ptr(kv), ptr(seq_excl), ptr(block_table), block_table.stride(0), B, sq,
            H, C, R, page, kv_cache.size(0), int(hint), int(bool(causal)), float(softmax_scale), ptr(o), ptr(ws), wsn,
            current_stream()), "mla_paged_prefill")
        return o

    def _mla_fp8kv(self, q_nope, q_pe, kv_cache, kv, seq_excl, block_table, causal, window_size, softcap,
                   softmax_scale):
        """The e4m3 latent cache [num_blocks, 64, C + R] (chitu_b200_mla_attn_fp8kv), both call shapes: q_nope
        [B, H, C] or [B, sq, H, C], bf16 q / kv / output.  The semantics of the bf16 cache, with each new kv element
        stored as x.float().clamp(-448, 448).to(float8_e4m3fn) and each cache element decoded exactly to bf16 before
        the unchanged arithmetic; the appended rows are attended in their stored form.  sq == 1 is the decode with the
        fused append and the device split plan of prepare_metadata_for_decode; returns [B, sq, H, C].  No host
        synchronisation, capturable in a CUDA graph, deterministic."""
        if tuple(window_size) != (-1, -1) or softcap != 0.0:
            raise RuntimeError("mla_attn_fp8kv: window_size and softcap are not built")
        if q_nope.dtype != torch.bfloat16 or q_pe.dtype != torch.bfloat16 or (kv is not None and kv.dtype != torch.bfloat16):
            raise RuntimeError("mla_attn_fp8kv: q_nope, q_pe and kv must be bfloat16 (only the cache is fp8)")
        require_cuda(seq_excl, kv)
        if q_nope.dim() == 3:
            q_nope, q_pe = q_nope.unsqueeze(1), q_pe.unsqueeze(1)
        B, sq, H, C = q_nope.shape
        R = q_pe.shape[-1]
        assert kv_cache.ndim == 3 and kv_cache.size(2) == C + R and q_pe.shape == (B, sq, H, R)
        assert q_nope.is_contiguous() and q_pe.is_contiguous() and kv_cache.is_contiguous()
        assert block_table.dtype == torch.int32 and block_table.stride(-1) == 1
        assert seq_excl.dtype == torch.int32 and seq_excl.is_contiguous()
        if kv is not None:
            assert kv.is_contiguous() and kv.numel() == B * sq * (C + R)
        if softmax_scale is None:
            softmax_scale = 1.0 / ((self.qk_rope_head_dim + self.qk_nope_head_dim) ** 0.5)
        page = kv_cache.size(1)
        o = torch.empty(B, sq, H, C, dtype=q_nope.dtype, device=q_nope.device)
        ws, wsn = self._ws(B, H, C, q_nope.device)
        hint = self.max_seq_len if self.max_seq_len else block_table.shape[1] * page
        check(_lib.load().chitu_b200_mla_attn_fp8kv(
            ptr(q_nope), ptr(q_pe), ptr(kv_cache), ptr(kv), ptr(seq_excl), ptr(block_table), block_table.stride(0), B, sq,
            H, C, R, page, kv_cache.size(0), int(hint), int(bool(causal)), float(softmax_scale), ptr(o), ptr(ws), wsn,
            current_stream()), "mla_attn_fp8kv")
        return o
