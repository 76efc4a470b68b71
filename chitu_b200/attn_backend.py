"""Drop-in attention backend for `chitu.attn_backend` (reference: chitu/attn_backend.py).

`B200AttnBackend` implements the four methods the models call (SURVEY.md §8b):
prepare_metadata_for_decode, attn_varlen_func (prefill: out of the decode hot path, delegated to
the reference-style fp32 formulation on the GPU), attn_with_kvcache (GQA paged decode with
in-place append) and mla_attn_with_kvcache (absorbed-MLA paged decode with fused append).
"""
from __future__ import annotations

import math
from typing import Optional, Union

import torch

from . import _lib, workspace
from ._lib import check, current_stream, dtype_code, ptr, require_cuda

__all__ = ["AttnBackend", "B200AttnBackend"]

_MAX_SPLITS = 128


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
        workspace.reserve("attn", self._ws_bytes(Bmax, self.n_local_heads, max(self.kv_lora_rank, 128)),
                          block_table.device)
        # a1 proper: the length-aware split-KV plan of this step, computed ON THE DEVICE from the step's lengths (the
        # reference's FlashInfer variant does O(B) .item() syncs here, attn_backend.py:620-637; FlashMLA runs
        # get_mla_metadata).  The MLA decode kernel finds it in the last 256 bytes of the attention workspace.
        if block_size == 64 and B > 0 and torch.is_tensor(cache_seqlens_incl_this_decode):
            H = self.n_local_heads
            buf, n = self._ws(B, H, max(self.kv_lora_rank, 128), block_table.device)
            hint = self.max_seq_len if self.max_seq_len else block_table.shape[1] * block_size
            check(_lib.load().chitu_b200_attn_plan(ptr(cache_seqlens_incl_this_decode), B, H, block_size, int(hint), ptr(buf), n,
                                                   current_stream()), "attn_plan")
            self._plan_view = buf[n - 256:].view(torch.int32)

    def last_plan(self):
        """int32 view of the device-side split plan written by the last prepare_metadata_for_decode (tests / debugging)."""
        return self._plan_view

    @staticmethod
    def _ws_bytes(B, H, DV):
        lib = _lib.load()
        # largest split count whose partials fit a bounded workspace (<= 256 MiB)
        splits = _MAX_SPLITS
        while splits > 1 and lib.chitu_b200_attn_workspace_bytes(B, H, DV, splits) > (256 << 20):
            splits //= 2
        return lib.chitu_b200_attn_workspace_bytes(B, H, DV, splits)

    def _ws(self, B, H, DV, device):
        buf = workspace.get("attn", self._ws_bytes(B, H, DV), device)
        return buf, buf.numel()

    # -- prefill (NOT on the decode hot path; SURVEY §8f n4, §8b "inherit prefill from Ref/flash_attn").
    # Exactly what the reference's FlashAttnBackend does (attn_backend.py:193-206): flash_attn_varlen_func when the
    # library is importable; otherwise torch's fused SDPA per sequence (no [H, Tq, Tk] fp32 score tensor, no host loop
    # over heads).  Both are library calls on a path this repository does not optimise.
    def attn_varlen_func(self, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
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
        if block_table is None:
            raise NotImplementedError("B200AttnBackend implements the paged (block_table) decode path")
        assert cache_leftpad is None and window_size == (-1, -1) and softcap == 0.0
        require_cuda(q, k_cache, v_cache, block_table)
        B, sq, Hq, D = q.shape
        assert sq == 1, "decode only (seqlen_q == 1)"
        num_blocks, page, Hkv, Dk = k_cache.shape
        assert Dk == D and v_cache.shape == k_cache.shape
        assert q.is_contiguous() and k_cache.is_contiguous() and v_cache.is_contiguous()
        assert block_table.dtype == torch.int32 and block_table.stride(-1) == 1
        if not torch.is_tensor(cache_seqlens):
            cache_seqlens = torch.full((B,), int(cache_seqlens), dtype=torch.int32, device=q.device)
        assert cache_seqlens.dtype == torch.int32 and cache_seqlens.is_contiguous()
        ksb = vsb = 0
        if k is not None:
            assert v is not None and k.shape == (B, 1, Hkv, D) and v.shape == (B, 1, Hkv, D)
            # heads must be dense; the batch stride is free (views into a fused qkv GEMM output)
            assert k.stride(-1) == 1 and k.stride(-2) == D and v.stride(-1) == 1 and v.stride(-2) == D
            ksb, vsb = k.stride(0), v.stride(0)
        scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
        out = torch.empty_like(q)
        ws, wsn = self._ws(B, Hq, D, q.device)
        hint = self.max_seq_len if self.max_seq_len else block_table.shape[1] * page
        check(_lib.load().chitu_b200_gqa_paged_decode(
            ptr(q), ptr(k_cache), ptr(v_cache), ptr(k), ptr(v), ksb, vsb, ptr(cache_seqlens), ptr(block_table),
            block_table.stride(0), B, Hq, Hkv, D, page, int(hint), float(scale), ptr(out), ptr(ws), wsn,
            dtype_code(q.dtype), current_stream()), "gqa_paged_decode")
        return out

    # -- a2: attn_backend.py:707-774 (Triton), :536-572 (FlashMLA), :660-684 (FlashInfer)
    def mla_attn_with_kvcache(self, q_nope, q_pe, kv_cache, kv,
                              cache_seqlens_excl_this_decode: Union[int, torch.Tensor],
                              cache_seqlens_incl_this_decode: Union[int, torch.Tensor],
                              block_table: torch.Tensor, causal=True, window_size=(-1, -1), softcap=0.0,
                              softmax_scale=None):
        require_cuda(q_nope, q_pe, kv_cache, block_table)
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
