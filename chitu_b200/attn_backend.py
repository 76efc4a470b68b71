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

__all__ = ["AttnBackend", "B200AttnBackend", "gqa_paged_attention", "mla_paged_attention"]

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
        _, page, Hkv, Dk = k_cache.shape
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
        ws, _ = self._ws(B, Hq, D, q.device)
        gqa_paged_attention(q, sq * Hq * D, k_cache, v_cache, k, v, strides, None, cache_seqlens, block_table, B, sq, Hq,
                            hint, causal, scale, out, ws)
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
        """Absorbed-MLA attention over the paged latent cache kv_cache [num_blocks, 64, C + R], bf16 q / kv / output.
        q_nope [B, H, C] (or [B, 1, H, C]): one decode token per request with the fused append of `kv` and the device
        split plan of prepare_metadata_for_decode, returned as [B, 1, H, C].  q_nope [B, sq, H, C] with sq > 1:
        multi-token-prediction verification or chunked prefill; the B * sq rows of `kv` ([B, sq, C + R] in any
        contiguous shape, or None) are appended at seq_excl[b] + i, then query i attends to the first seq_excl[b] + sq
        keys (without kv: seq_excl[b]), bottom-right causal when `causal`; returns [B, sq, H, C].  softmax_scale=None
        means 1 / sqrt(qk_rope_head_dim + qk_nope_head_dim); window_size and softcap are not built.
        A kv_cache in torch.float8_e4m3fn takes both call shapes with the same semantics, each new kv element stored as
        x.float().clamp(-448, 448).to(float8_e4m3fn) and each cache element decoded exactly to bf16 before the unchanged
        arithmetic; the appended rows are attended in their stored form.  No host synchronisation, capturable in a CUDA
        graph, deterministic."""
        seq_excl = cache_seqlens_excl_this_decode
        require_cuda(q_nope, q_pe, kv_cache, block_table, seq_excl, kv)
        if tuple(window_size) != (-1, -1) or softcap != 0.0:
            raise RuntimeError("mla_attn_with_kvcache: window_size and softcap are not built")
        if any(t is not None and t.dtype != torch.bfloat16 for t in (q_nope, q_pe, kv)):
            raise RuntimeError("mla_attn_with_kvcache: q_nope, q_pe and kv must be bfloat16 (the cache may be fp8)")
        if q_nope.dim() == 3:
            q_nope, q_pe = q_nope.unsqueeze(1), q_pe.unsqueeze(1)
        B, sq, H, C = q_nope.shape
        R = q_pe.shape[-1]
        assert kv_cache.dtype in (torch.bfloat16, torch.float8_e4m3fn)
        assert kv_cache.ndim == 3 and kv_cache.size(2) == C + R and q_pe.shape == (B, sq, H, R)
        assert q_nope.is_contiguous() and q_pe.is_contiguous() and kv_cache.is_contiguous()
        assert block_table.dtype == torch.int32 and block_table.stride(-1) == 1
        assert seq_excl.dtype == torch.int32 and seq_excl.is_contiguous()
        if kv is not None:
            assert kv.is_contiguous() and kv.numel() == B * sq * (C + R)
        if softmax_scale is None:
            softmax_scale = 1.0 / ((self.qk_rope_head_dim + self.qk_nope_head_dim) ** 0.5)
        o = torch.empty(B, sq, H, C, dtype=q_nope.dtype, device=q_nope.device)
        ws, _ = self._ws(B, H, C, q_nope.device)
        hint = self.max_seq_len if self.max_seq_len else block_table.shape[1] * kv_cache.size(1)
        mla_paged_attention(q_nope, q_pe, kv_cache, kv, seq_excl, block_table, hint, causal, softmax_scale, o, ws)
        return o


def gqa_paged_attention(q, q_sb, k_cache, v_cache, k_new, v_new, kv_strides, rope, cache_seqlens, block_table, B, sq,
                        Hq, max_seqlen_hint, causal, softmax_scale, out, workspace):
    """GQA attention over the paged caches k_cache / v_cache [num_blocks, page, Hkv, D] as one C call, the entry picked
    from the cache dtype, sq and the query layout:
      - an e4m3 cache: chitu_b200_gqa_paged_attn_fp8kv, any sq;
      - sq > 1: chitu_b200_gqa_paged_prefill;
      - sq == 1 with `rope` or a strided q (q_sb != Hq * D): chitu_b200_gqa_paged_decode_rope;
      - otherwise chitu_b200_gqa_paged_decode.
    q: B * sq query rows, batch stride q_sb elements; k_new / v_new: the new rows or None, with strides
    kv_strides = (k_sb, k_st, v_sb, v_st) in elements (the decode entries read only the batch strides); rope: the fp32
    (cos, sin) [B, D / 2] of the rotary fused at sq == 1, or None; workspace: the split-KV workspace (uint8).  The entries
    and their arguments are described in include/chitu_b200.h; the caller checks the tensors."""
    lib = _lib.load()
    num_blocks, page, Hkv, D = k_cache.shape
    cos, sin = rope if rope is not None else (None, None)
    k_sb, _, v_sb, _ = kv_strides
    caches = (ptr(k_cache), ptr(v_cache), ptr(k_new), ptr(v_new))
    pages = (ptr(cache_seqlens), ptr(block_table), block_table.stride(0), B)
    hint, causal, scale = int(max_seqlen_hint), int(bool(causal)), float(softmax_scale)
    tail = (ptr(out), ptr(workspace), workspace.numel(), dtype_code(q.dtype), current_stream())
    if k_cache.dtype == torch.float8_e4m3fn:
        check(lib.chitu_b200_gqa_paged_attn_fp8kv(ptr(q), q_sb, *caches, *kv_strides, ptr(cos), ptr(sin), *pages, sq, Hq,
                                                  Hkv, D, page, num_blocks, hint, causal, scale, *tail),
              "gqa_paged_attn_fp8kv")
    elif sq > 1:
        assert rope is None and q_sb == sq * Hq * D
        check(lib.chitu_b200_gqa_paged_prefill(ptr(q), *caches, *kv_strides, *pages, sq, Hq, Hkv, D, page, num_blocks,
                                               hint, causal, scale, *tail), "gqa_paged_prefill")
    elif rope is not None or q_sb != Hq * D:
        check(lib.chitu_b200_gqa_paged_decode_rope(ptr(q), q_sb, *caches, k_sb, v_sb, ptr(cos), ptr(sin), *pages, Hq,
                                                   Hkv, D, page, hint, scale, *tail), "gqa_paged_decode_rope")
    else:
        check(lib.chitu_b200_gqa_paged_decode(ptr(q), *caches, k_sb, v_sb, *pages, Hq, Hkv, D, page, hint, scale,
                                              *tail), "gqa_paged_decode")


def mla_paged_attention(q_nope, q_pe, kv_cache, new_kv, seqlens_excl, block_table, max_seqlen_hint, causal,
                        softmax_scale, out, workspace):
    """Absorbed-MLA attention over the paged latent cache kv_cache [num_blocks, page, C + R] as one C call, the entry
    picked from the cache dtype and sq:
      - an e4m3 cache: chitu_b200_mla_attn_fp8kv, any sq;
      - sq == 1: chitu_b200_mla_decode (the one query row sees every key: it takes no `causal`);
      - sq > 1: chitu_b200_mla_paged_prefill.
    q_nope [B, H, C] (sq = 1) or [B, sq, H, C], q_pe the same with R; new_kv: the B * sq new rows or None; out None
    (sq == 1): the split merge is left to chitu_b200_mla_absorb_o_merge_quant.  The entries and their arguments are
    described in include/chitu_b200.h; the caller checks the tensors."""
    lib = _lib.load()
    B, H, C, R = q_nope.shape[0], q_nope.shape[-2], q_nope.shape[-1], q_pe.shape[-1]
    sq = q_nope.shape[1] if q_nope.dim() == 4 else 1
    num_blocks, page, _ = kv_cache.shape
    head = (ptr(q_nope), ptr(q_pe), ptr(kv_cache), ptr(new_kv), ptr(seqlens_excl), ptr(block_table),
            block_table.stride(0), B)
    hint, scale = int(max_seqlen_hint), float(softmax_scale)
    tail = (ptr(out), ptr(workspace), workspace.numel(), current_stream())
    if kv_cache.dtype == torch.float8_e4m3fn:
        fn, name = lib.chitu_b200_mla_attn_fp8kv, "mla_attn_fp8kv"
    elif sq == 1:
        check(lib.chitu_b200_mla_decode(*head, H, C, R, page, num_blocks, hint, scale, *tail), "mla_decode")
        return
    else:
        fn, name = lib.chitu_b200_mla_paged_prefill, "mla_paged_prefill"
    check(fn(*head, sq, H, C, R, page, num_blocks, hint, int(bool(causal)), scale, *tail), name)
