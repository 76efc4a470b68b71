"""Drop-in for `chitu/ops.py`: same function names, argument meaning and error behaviour
(asserts on non-contiguous inputs), bodies replaced by libchitu_b200 (sm_90a CUDA).

Reference: thu-pacman/chitu, chitu/ops.py (file:line cited per function).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from . import _lib, workspace
from ._lib import check, current_stream, dtype_code, ptr, require_cuda

__all__ = [
    "append_to_paged_kv_cache",
    "scatter_kv_to_cache",
    "apply_rotary_pos_emb",
    "apply_rotary_pos_emb_triton",
    "act_quant_deepseek_v3",
    "weight_dequant_deepseek_v3",
    "weight_dequant_soft_fp8_deepseek_v3",
    "fp8_gemm_deepseek_v3",
    "soft_fp8_gemm_deepseek_v3",
    "rms_norm",
    "silu_and_mul",
    "linear",
    "sample_top_k_top_p",
    "accept_draft_tokens_greedy",
    "accept_draft_tokens_sampled",
]

# impl selector for the linears: 0 auto, 1 SIMT, 2 wgmma (tests flip this)
LINEAR_IMPL = 0


def _linear_ws(M: int, N: int, device):
    n = _lib.load().chitu_b200_linear_workspace_bytes(M, N)
    if n <= 0:
        return None, 0
    buf = workspace.get("linear", n, device)
    return buf, buf.numel()


def append_to_paged_kv_cache(kv_cache, page_table, this_kv, old_seq_lens):
    """chitu/ops.py:50-91.  kv_cache[page_table[i][len_i // 64]][len_i % 64] = this_kv[i]
    (the literal 64 is the reference's, triton_kernels.py:38,42).
    A float8_e4m3fn cache of 64-token pages takes bf16 / fp16 rows and stores each element as
    x.float().clamp(-448, 448).to(float8_e4m3fn) (plain .to() would turn values beyond +-464 into NaN), the rule of
    the e4m3 attention paths' own appends.  One row per request per call: to write a prompt's k / v or latent rows into
    a cache of any page size (e4m3 included), call `scatter_kv_to_cache`."""
    assert kv_cache.is_contiguous()
    assert page_table.is_contiguous()
    assert this_kv.is_contiguous()
    assert old_seq_lens.is_contiguous()
    require_cuda(kv_cache, page_table, this_kv, old_seq_lens)
    page_size = kv_cache.shape[1]
    batch_size, num_pages_per_sample = page_table.shape
    assert this_kv.shape[0] == batch_size
    assert old_seq_lens.shape[0] == batch_size
    tot = this_kv.numel() // batch_size
    assert kv_cache.numel() // (kv_cache.shape[0] * kv_cache.shape[1]) == tot
    assert page_table.dtype == torch.int32 and old_seq_lens.dtype == torch.int32
    if kv_cache.dtype == torch.float8_e4m3fn and this_kv.dtype != kv_cache.dtype:
        assert this_kv.dtype in (torch.bfloat16, torch.float16) and page_size == 64
        check(_lib.load().chitu_b200_append_paged_kv_e4m3(
            ptr(kv_cache), ptr(page_table), ptr(this_kv), ptr(old_seq_lens), batch_size, num_pages_per_sample, tot,
            dtype_code(this_kv.dtype), current_stream()), "append_paged_kv_e4m3")
        return
    assert this_kv.dtype == kv_cache.dtype
    check(
        _lib.load().chitu_b200_append_paged_kv(
            ptr(kv_cache), ptr(page_table), ptr(this_kv), ptr(old_seq_lens), batch_size,
            num_pages_per_sample, page_size, 64, tot * kv_cache.element_size(), current_stream(),
        ),
        "append_paged_kv",
    )


def scatter_kv_to_cache(k_cache, v_cache, k, v, cu_seqlens, block_table=None, cache_seqlens=None):
    """Writes the prompts' k / v rows into the KV cache after the prefill attention, every request of the batch in one
    launch (the page scatter of PagedKVCacheManager.finalize_cache_bylayer_prefill, cache_manager.py:93-142, without
    its per-request loop).  Row t of request b, k[cu_seqlens[b] + t] for t < cu_seqlens[b + 1] - cu_seqlens[b], goes
    to position p = cache_seqlens[b] + t (p = t without cache_seqlens).

    GQA: k / v [total, Hkv, D] with dense heads and any row stride (views of a fused qkv output); caches
    [num_blocks, page, Hkv, D] with a block table (page block_table[b, p // page], slot p % page, any page size), or
    [Bc, S, Hkv, D] without one (row p of cache entry b; rows with p >= S are not written).  MLA: kv_cache
    [num_blocks, 64, 576] and kv [total, 576] as k_cache / k, with v_cache = v = None.  cu_seqlens int32 [B + 1] and
    cache_seqlens int32 [B] on the device.  A float8_e4m3fn paged cache takes bf16 / fp16 rows and stores each element
    as x.float().clamp(-448, 448).to(float8_e4m3fn); otherwise the caches have the rows' dtype and get their bits.
    In place, no host synchronisation (capturable in a CUDA graph), returns None."""
    def refuse(why):
        raise RuntimeError(f"scatter_kv_to_cache: {why}")

    tensors = [t for t in (k_cache, v_cache, k, v, cu_seqlens, block_table, cache_seqlens) if t is not None]
    require_cuda(*tensors)
    if any(t.device != k_cache.device for t in tensors):
        refuse("every tensor must be on the cache's device")
    if (v_cache is None) != (v is None):
        refuse("v_cache and v are given together (GQA) or both None (MLA)")
    if k.dtype not in (torch.bfloat16, torch.float16) or k_cache.dtype not in (k.dtype, torch.float8_e4m3fn):
        refuse(f"{k.dtype} rows into a {k_cache.dtype} cache are not built")
    if block_table is None and k_cache.dtype == torch.float8_e4m3fn:
        refuse("the fp8 KV cache is built for the paged cache only")
    row_shape = tuple(k_cache.shape[2:])
    if k_cache.dim() < 3 or tuple(k.shape[1:]) != row_shape:
        refuse(f"rows {tuple(k.shape)} do not match the cache {tuple(k_cache.shape)}")
    if not (_dense_rows(k, 1) and _dense_rows(k_cache, 2)):
        refuse("the elements of a row must be dense in k and in the cache")
    if v is not None and (v_cache.shape != k_cache.shape or v_cache.dtype != k_cache.dtype or v.dtype != k.dtype
                          or v.shape != k.shape or not _dense_rows(v, 1) or v_cache.stride() != k_cache.stride()):
        refuse("v / v_cache must match k / k_cache in shape, dtype and layout")
    if k.shape[0] >= 2 ** 31:
        refuse("more than 2^31 - 1 rows")
    if cu_seqlens.dtype != torch.int32 or cu_seqlens.dim() != 1 or cu_seqlens.numel() < 1 \
            or not cu_seqlens.is_contiguous():
        refuse("cu_seqlens must be a contiguous int32 [B + 1] tensor")
    B = cu_seqlens.numel() - 1
    if cache_seqlens is not None and (cache_seqlens.dtype != torch.int32 or tuple(cache_seqlens.shape) != (B,)
                                      or not cache_seqlens.is_contiguous()):
        refuse("cache_seqlens must be a contiguous int32 [B] tensor")
    if block_table is not None:
        if block_table.dtype != torch.int32 or block_table.dim() != 2 or block_table.stride(-1) != 1 \
                or block_table.shape[0] < B or not k_cache.is_contiguous():
            refuse("block_table must be int32 [>= B, pages] with unit column stride, over contiguous caches")
        paged, cache_sb, cache_rows = (ptr(block_table), block_table.stride(0), k_cache.shape[1]), 0, 0
    else:
        if k_cache.shape[0] < B:
            refuse(f"a non-paged cache holds {k_cache.shape[0]} requests, fewer than {B}")
        if not _dense_rows(k_cache, 1):
            refuse("a non-paged cache [Bc, S, ...] must be dense from its second dim on")
        paged, cache_sb, cache_rows = (None, 0, 0), k_cache.stride(0), k_cache.shape[1]
    check(_lib.load().chitu_b200_scatter_kv(
        ptr(k_cache), ptr(v_cache), ptr(k), k.stride(0), ptr(v), 0 if v is None else v.stride(0), ptr(cu_seqlens),
        ptr(cache_seqlens), *paged, cache_sb, cache_rows, B, k.shape[0], math.prod(row_shape), dtype_code(k.dtype),
        dtype_code(k_cache.dtype), current_stream()), "scatter_kv")


def _dense_rows(t, lead):
    """The dims of `t` from `lead` on are laid out as a contiguous block (dims of size 1 may have any stride)."""
    want = 1
    for size, stride in reversed(list(zip(t.shape[lead:], t.stride()[lead:]))):
        if size != 1 and stride != want:
            return False
        want *= size
    return True


def apply_rotary_pos_emb_triton(q, k, cos, sin, rotary_type="hf-llama", block_size=128):
    """chitu/ops.py:123-240 (name kept for drop-in; nothing here is Triton)."""
    lib = _lib.load()
    require_cuda(q, k, cos, sin)
    if rotary_type == "hf-llama":
        assert q.is_contiguous() and k.is_contiguous() and cos.is_contiguous() and sin.is_contiguous()
        qb, qh, qd = q.shape
        kb, kh, kd = k.shape
        cos_c, sin_c = cos.to(q.dtype), sin.to(q.dtype)
        q_out, k_out = torch.empty_like(q), torch.empty_like(k)
        check(lib.chitu_b200_rotary_half(ptr(q), ptr(q_out), ptr(cos_c), ptr(sin_c), qb, qh, qd,
                                         dtype_code(q.dtype), current_stream()), "rotary_half")
        check(lib.chitu_b200_rotary_half(ptr(k), ptr(k_out), ptr(cos_c), ptr(sin_c), kb, kh, kd,
                                         dtype_code(k.dtype), current_stream()), "rotary_half")
        return q_out, k_out
    elif rotary_type == "llama":
        q_shape, k_shape = q.shape, k.shape
        if q.dim() == 4:
            q = q.view(-1, q.shape[-2], q.shape[-1])
        elif q.dim() == 2:
            q = q.view(-1, 1, q.shape[-1])
        else:
            assert q.dim() == 3
        if k.dim() == 4:
            k = k.view(-1, k.shape[-2], k.shape[-1])
        elif k.dim() == 2:
            k = k.view(-1, 1, k.shape[-1])
        else:
            assert k.dim() == 3
        assert q.shape[-1] == k.shape[-1]
        assert q.shape[0] == k.shape[0]
        assert q.shape[-1] // 2 == cos.shape[-1]
        assert q.shape[-1] // 2 == sin.shape[-1]
        assert q.stride(-1) == 1 and k.stride(-1) == 1
        bs, hq, rot = q.shape
        _, hk, _ = k.shape
        cos_c = cos.contiguous().float()
        sin_c = sin.contiguous().float()
        out_q = torch.empty((bs, hq, rot), dtype=q.dtype, device=q.device)
        out_k = torch.empty((bs, hk, rot), dtype=k.dtype, device=k.device)
        check(lib.chitu_b200_rotary_interleaved(ptr(q), ptr(k), ptr(out_q), ptr(out_k), ptr(cos_c), ptr(sin_c),
                                                bs, hq, hk, rot, q.stride(0), q.stride(1), k.stride(0),
                                                k.stride(1), dtype_code(q.dtype), current_stream()),
              "rotary_interleaved")
        return out_q.view(q_shape), out_k.view(k_shape)
    else:
        raise ValueError(f"Unknown rotary type: {rotary_type}")


def apply_rotary_pos_emb(q, k, cos, sin, rotary_type="hf-llama"):
    """chitu/ops.py:311-326."""
    if rotary_type in ("hf-llama", "llama"):
        return apply_rotary_pos_emb_triton(q, k, cos, sin, rotary_type=rotary_type)
    raise ValueError(f"Unknown rotary type: {rotary_type}")


def act_quant_deepseek_v3(x: torch.Tensor, block_size: int = 128) -> Tuple[torch.Tensor, torch.Tensor]:
    """chitu/ops.py:329-353."""
    assert x.is_contiguous(), "Input tensor must be contiguous"
    assert x.size(-1) % block_size == 0, (
        f"Last dimension size must be divisible by block_size (block_size={block_size})")
    require_cuda(x)
    y = torch.empty_like(x, dtype=torch.float8_e4m3fn)
    s = x.new_empty(*x.size()[:-1], x.size(-1) // block_size, dtype=torch.float32)
    K = x.size(-1)
    rows = x.numel() // K
    check(_lib.load().chitu_b200_act_quant_fp8(ptr(x), ptr(y), ptr(s), rows, K, block_size, 0, 0.0,
                                               dtype_code(x.dtype), current_stream()), "act_quant_fp8")
    return y, s


def _weight_dequant(x, s, block_size, soft):
    assert x.is_contiguous() and s.is_contiguous(), "Input tensors must be contiguous"
    assert s.dim() == x.dim(), "Scale tensors must have the same number of dimensions with the weight tensor"
    require_cuda(x, s)
    if x.dim() == 2:
        M, N = x.size()
        B = 1
    elif x.dim() == 3:
        B, M, N = x.size()
    else:
        assert False, "Weight tensor must have 2 or 3 dimensions"
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    check(_lib.load().chitu_b200_weight_dequant_fp8(ptr(x), ptr(s), ptr(y), B, M, N, block_size, int(soft),
                                                    current_stream()), "weight_dequant_fp8")
    return y


def weight_dequant_deepseek_v3(x: torch.Tensor, s: torch.Tensor, block_size: int = 128) -> torch.Tensor:
    """chitu/ops.py:356-392 (output dtype bf16 == the reference's default dtype for DeepSeek)."""
    return _weight_dequant(x, s, block_size, False)


def weight_dequant_soft_fp8_deepseek_v3(x: torch.Tensor, s: torch.Tensor, block_size: int = 128) -> torch.Tensor:
    """chitu/ops.py:395-449."""
    return _weight_dequant(x, s, block_size, True)


def fp8_gemm_deepseek_v3(a: torch.Tensor, a_s: torch.Tensor, b: torch.Tensor, b_s: torch.Tensor):
    """chitu/ops.py:452-483."""
    assert a.is_contiguous() and b.is_contiguous(), "Input tensors must be contiguous"
    assert a_s.is_contiguous() and b_s.is_contiguous(), "Scaling factor tensors must be contiguous"
    require_cuda(a, a_s, b, b_s)
    K = a.size(-1)
    M = a.numel() // K
    N = b.size(0)
    c = a.new_empty(*a.size()[:-1], N, dtype=torch.bfloat16)
    ws, wsn = _linear_ws(M, N, a.device)
    check(_lib.load().chitu_b200_fp8_gemm(ptr(a), ptr(a_s), ptr(b), ptr(b_s), ptr(c), M, N, K, None, ptr(ws), wsn,
                                          LINEAR_IMPL, current_stream()), "fp8_gemm")
    return c


def soft_fp8_gemm_deepseek_v3(a: torch.Tensor, b: torch.Tensor, b_s: torch.Tensor):
    """chitu/ops.py:486-511."""
    assert a.is_contiguous() and b.is_contiguous(), "Input tensors must be contiguous"
    assert b_s.is_contiguous(), "Scaling factor tensor must be contiguous"
    require_cuda(a, b, b_s)
    K = a.size(-1)
    M = a.numel() // K
    N = b.size(0)
    c = a.new_empty(*a.size()[:-1], N, dtype=a.dtype)
    # wgmma path (bf16, K % 128 == 0): fp8 weight tiles are converted to bf16 in shared memory between TMA and MMA
    ws, wsn = _linear_ws(M, N, a.device)
    check(_lib.load().chitu_b200_soft_fp8_gemm(ptr(a), ptr(b), ptr(b_s), ptr(c), M, N, K, dtype_code(a.dtype),
                                               ptr(ws), wsn, LINEAR_IMPL, current_stream()),
          "soft_fp8_gemm")
    return c


# ---- operators the reference takes from torch (F.linear / F.rms_norm / F.silu) ------------------

def linear(x: torch.Tensor, weight: torch.Tensor, bias=None, residual=None) -> torch.Tensor:
    """F.linear for bf16/fp16 weights (`linear_op` of tensor_parallel.py:51,115; the
    element_size()>1 branch of linear_deepseek_v3, model_deepseek_v3.py:84-85)."""
    assert x.is_contiguous() and weight.is_contiguous()
    require_cuda(x, weight)
    K = x.size(-1)
    M = x.numel() // K
    N = weight.size(0)
    assert weight.size(1) == K and weight.dtype == x.dtype
    y = x.new_empty(*x.size()[:-1], N)
    ws, wsn = _linear_ws(M, N, x.device)
    if residual is not None:
        assert residual.is_contiguous() and residual.numel() == M * N
    check(_lib.load().chitu_b200_linear_bf16(ptr(x), ptr(weight), ptr(bias), ptr(residual), ptr(y), M, N, K,
                                             dtype_code(x.dtype), ptr(ws), wsn, LINEAR_IMPL, current_stream()),
          "linear_bf16")
    return y


SOFT_FP8 = False   # the reference reads infer.soft_fp8 from its global args (model_deepseek_v3.py:86); integrators set this


def linear_deepseek_v3(x: torch.Tensor, weight: torch.Tensor, weight_scale: Optional[torch.Tensor] = None,
                       bias: Optional[torch.Tensor] = None, soft_fp8: Optional[bool] = None) -> torch.Tensor:
    """The `linear_op` hook of the DeepSeek parallel linears (model_deepseek_v3.py:53-106): weights wider than one byte go
    to `linear`; one-byte weights are either W8A16 (`soft_fp8`: bf16 activations, weight tile rounded to bf16 in the
    kernel) or W8A8 (act_quant 1x128 + block-scaled fp8 GEMM).  After `plugin.install()` the reference's own dispatcher
    reaches the same three operators by name; this mirror is for callers that use chitu_b200 directly."""
    if weight.element_size() > 1:
        return linear(x, weight, bias)
    assert weight_scale is not None
    lead, K = x.shape[:-1], x.shape[-1]
    x2 = x.reshape(-1, K)
    if SOFT_FP8 if soft_fp8 is None else soft_fp8:
        y = soft_fp8_gemm_deepseek_v3(x2, weight, weight_scale)
    else:
        xq, xs = act_quant_deepseek_v3(x2, 128)
        y = fp8_gemm_deepseek_v3(xq, xs, weight, weight_scale)
    if bias is not None:
        y += bias
    return y.view(*lead, y.shape[-1])


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """RMSNorm.forward (chitu/models/model.py:50-78)."""
    assert x.is_contiguous() and weight.is_contiguous()
    require_cuda(x, weight)
    dim = x.size(-1)
    w = weight if weight.dtype == x.dtype else weight.to(x.dtype)
    y = torch.empty_like(x)
    check(_lib.load().chitu_b200_rmsnorm(ptr(x), ptr(w), ptr(y), x.numel() // dim, dim, eps, dtype_code(x.dtype),
                                         current_stream()), "rmsnorm")
    return y


def silu_and_mul(x: torch.Tensor) -> torch.Tensor:
    """SiluAndMul.forward (chitu/fused_moe.py:24-39)."""
    assert x.is_contiguous()
    require_cuda(x)
    d = x.shape[-1] // 2
    out = x.new_empty(*x.shape[:-1], d)
    check(_lib.load().chitu_b200_silu_and_mul(ptr(x), ptr(out), x.numel() // (2 * d), d, dtype_code(x.dtype),
                                              current_stream()), "silu_and_mul")
    return out


# ---- fused variants used by the decode engine (SURVEY §8f n1: prologue fusion) ---------------------

def rms_norm_quant(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, want_y: bool = True):
    """RMSNorm followed by act_quant_deepseek_v3 in one launch -> (y bf16 | None, q fp8, s fp32)."""
    assert x.is_contiguous() and x.dtype == torch.bfloat16 and x.dim() == 2
    require_cuda(x, weight)
    rows, dim = x.shape
    y = torch.empty_like(x) if want_y else None
    q = torch.empty_like(x, dtype=torch.float8_e4m3fn)
    s = x.new_empty(rows, dim // 128, dtype=torch.float32)
    check(_lib.load().chitu_b200_rmsnorm_quant_fp8(ptr(x), ptr(weight), ptr(y), ptr(q), ptr(s), rows, dim, dim, dim,
                                                   float(eps), current_stream()), "rmsnorm_quant_fp8")
    return y, q, s


def silu_mul_quant(x: torch.Tensor):
    """SiluAndMul followed by act_quant_deepseek_v3 in one launch: x [rows, 2F] -> (q fp8 [rows,F], s)."""
    assert x.is_contiguous() and x.dtype == torch.bfloat16 and x.dim() == 2
    require_cuda(x)
    rows, F2 = x.shape
    F = F2 // 2
    q = torch.empty(rows, F, dtype=torch.float8_e4m3fn, device=x.device)
    s = torch.empty(rows, F // 128, dtype=torch.float32, device=x.device)
    check(_lib.load().chitu_b200_silu_mul_quant_fp8(ptr(x), ptr(q), ptr(s), rows, F, current_stream()), "silu_mul_quant")
    return q, s


def embedding(ids: torch.Tensor, table: torch.Tensor, vocab_start: int = 0) -> torch.Tensor:
    """Local lookup of `VocabParallelEmbedding.forward` (chitu/tensor_parallel.py:199-208): `table` holds the rows
    [vocab_start, vocab_start + table.size(0)) of the vocabulary; ids outside that range give zero rows (the
    reference masks them before its all-reduce)."""
    assert table.is_contiguous() and ids.dtype == torch.int64
    require_cuda(ids, table)
    ids = ids.contiguous()
    T, dim = ids.numel(), table.size(1)
    out = torch.empty(*ids.shape, dim, dtype=table.dtype, device=table.device)
    check(_lib.load().chitu_b200_embedding(ptr(ids), ptr(table), ptr(out), T, dim, int(vocab_start), table.size(0),
                                           dtype_code(table.dtype), current_stream()), "embedding")
    return out



def sample_top_k_top_p(logits: torch.Tensor, temperatures: torch.Tensor, top_ks: torch.Tensor, top_ps: torch.Tensor,
                       uniforms: torch.Tensor = None, return_stats: bool = False):
    """NormalExecutor.update_response's sampling branch (executor.py:104-110) + top_k_top_p_min_p_sampling_from_probs_torch
    (utils.py:62-81) in one kernel per step: logits [B, V] -> token ids int64 [B].  `uniforms` (fp32 [B] in [0,1)) default
    to torch.rand on the logits' device."""
    assert logits.dim() == 2 and logits.stride(-1) == 1
    require_cuda(logits, temperatures, top_ks, top_ps)
    B, V = logits.shape
    if uniforms is None:
        uniforms = torch.rand(B, device=logits.device, dtype=torch.float32)
    tok = torch.empty(B, dtype=torch.int64, device=logits.device)
    kept = torch.empty(B, dtype=torch.int32, device=logits.device) if return_stats else None
    mass = torch.empty(B, dtype=torch.float32, device=logits.device) if return_stats else None
    check(_lib.load().chitu_b200_sample_top_k_top_p(ptr(logits), logits.stride(0), B, V, dtype_code(logits.dtype),
                                                    ptr(temperatures.float().contiguous()), ptr(top_ks.to(torch.int32).contiguous()),
                                                    ptr(top_ps.float().contiguous()), ptr(uniforms.float().contiguous()), ptr(tok),
                                                    ptr(kept), ptr(mass), current_stream()), "sample_top_k_top_p")
    return (tok, kept, mass) if return_stats else tok


def accept_draft_tokens_greedy(target: torch.Tensor, drafts: torch.Tensor, n_draft: torch.Tensor,
                               seq_lens: torch.Tensor):
    """Greedy acceptance of speculative drafts after a verify step over k + 1 positions per request, in one launch.
    target int64 [B, k + 1] (the argmax at each verified position), drafts int64 [B, k], n_draft int32 [B] (each
    request's draft length, 0..k) and seq_lens int32 [B], all contiguous on one CUDA device.  Request b accepts the
    a_b leading drafts that equal the target (i < n_draft[b]) and emits target[b, :a_b + 1]; seq_lens[b] grows by
    a_b + 1 in place.  Returns (out_tokens int64 [B, k + 1] with -1 after the emitted tokens, accepted int32 [B],
    next_tokens int64 [B] = target[b, a_b]).  No host synchronisation (capturable)."""
    def refuse(why):
        raise ValueError(f"accept_draft_tokens_greedy: {why}")

    ts = (target, drafts, n_draft, seq_lens)
    if not all(isinstance(t, torch.Tensor) for t in ts):
        refuse("every argument must be a tensor")
    if not all(t.is_cuda for t in ts) or any(t.device != target.device for t in ts):
        refuse("every tensor must be on the same CUDA device")
    if (target.dtype, drafts.dtype, n_draft.dtype, seq_lens.dtype) != (torch.int64, torch.int64, torch.int32,
                                                                       torch.int32):
        refuse("target and drafts must be int64, n_draft and seq_lens int32")
    if target.dim() != 2 or target.shape[1] < 2:
        refuse(f"target must be [B, k + 1] with k >= 1, not {tuple(target.shape)}")
    B, k = target.shape[0], target.shape[1] - 1
    if tuple(drafts.shape) != (B, k) or tuple(n_draft.shape) != (B,) or tuple(seq_lens.shape) != (B,):
        refuse(f"drafts must be [{B}, {k}], n_draft and seq_lens [{B}]")
    if not all(t.is_contiguous() for t in ts):
        refuse("every tensor must be contiguous")
    out = torch.empty(B, k + 1, dtype=torch.int64, device=target.device)
    accepted = torch.empty(B, dtype=torch.int32, device=target.device)
    nxt = torch.empty(B, dtype=torch.int64, device=target.device)
    check(_lib.load().chitu_b200_spec_accept_greedy(ptr(target), ptr(drafts), ptr(n_draft), ptr(seq_lens), ptr(out),
                                                    ptr(accepted), ptr(nxt), B, k, current_stream()),
          "spec_accept_greedy")
    return out, accepted, nxt


def accept_draft_tokens_sampled(logits: torch.Tensor, drafts: torch.Tensor, n_draft: torch.Tensor,
                                seq_lens: torch.Tensor, temperatures: torch.Tensor, top_ks: torch.Tensor,
                                top_ps: torch.Tensor, u_accept: torch.Tensor, u_draw: torch.Tensor,
                                draft_probs: Optional[torch.Tensor] = None):
    """Speculative sampling of k drafts per request after a verify step, in two launches: the emitted tokens have the
    distribution of sampling the target one token at a time with each request's temperature / top_k / top_p (the rule
    of `sample_top_k_top_p`; T <= 0 is greedy, as `accept_draft_tokens_greedy` on the first maximal index).

    logits [B * (k + 1), V] bf16 / fp16 / fp32 with unit column stride (row b * (k + 1) + i: request b's position i);
    drafts int64 [B, k]; n_draft int32 [B] (0..k); seq_lens int32 [B], advanced in place; temperatures, top_ps fp32 [B];
    top_ks int32 [B] (<= 0: no top-k); u_accept fp32 [B, k] and u_draw fp32 [B], uniforms in [0, 1); draft_probs: fp32
    [B, k, V] with unit last stride, the drafter's distributions (None: token-only drafts, q one-hot at the draft).
    Draft i is accepted iff u_accept[b, i] * q_i(d_i) < p_i(d_i); at the first rejection the token is drawn from
    max(p - q, 0), after n accepted drafts from p_n.  Returns (out_tokens int64 [B, k + 1] with -1 after the emitted
    tokens, accepted int32 [B], next_tokens int64 [B]).  No host synchronisation (capturable)."""
    def refuse(why):
        raise ValueError(f"accept_draft_tokens_sampled: {why}")

    ts = (logits, drafts, n_draft, seq_lens, temperatures, top_ks, top_ps, u_accept, u_draw)
    if not all(isinstance(t, torch.Tensor) for t in ts) or not (draft_probs is None or
                                                                isinstance(draft_probs, torch.Tensor)):
        refuse("every argument must be a tensor")
    every = ts + (() if draft_probs is None else (draft_probs,))
    if not all(t.is_cuda for t in every) or any(t.device != logits.device for t in every):
        refuse("every tensor must be on the same CUDA device")
    if logits.dtype not in (torch.bfloat16, torch.float16, torch.float32):
        refuse(f"logits must be bf16, fp16 or fp32, not {logits.dtype}")
    if (drafts.dtype, n_draft.dtype, seq_lens.dtype, top_ks.dtype) != (torch.int64, torch.int32, torch.int32,
                                                                       torch.int32):
        refuse("drafts must be int64, n_draft, seq_lens and top_ks int32")
    if any(t.dtype != torch.float32 for t in (temperatures, top_ps, u_accept, u_draw)):
        refuse("temperatures, top_ps, u_accept and u_draw must be fp32")
    if drafts.dim() != 2 or drafts.shape[1] < 1:
        refuse(f"drafts must be [B, k] with k >= 1, not {tuple(drafts.shape)}")
    B, k = drafts.shape
    if logits.dim() != 2 or logits.shape[0] != B * (k + 1) or logits.shape[1] < 1 or logits.stride(1) != 1:
        refuse(f"logits must be [{B * (k + 1)}, V] with unit column stride, not {tuple(logits.shape)} "
               f"(strides {logits.stride()})")
    V = logits.shape[1]
    if any(tuple(t.shape) != (B,) for t in (n_draft, seq_lens, temperatures, top_ks, top_ps, u_draw)):
        refuse(f"n_draft, seq_lens, temperatures, top_ks, top_ps and u_draw must be [{B}]")
    if tuple(u_accept.shape) != (B, k):
        refuse(f"u_accept must be [{B}, {k}], not {tuple(u_accept.shape)}")
    if not all(t.is_contiguous() for t in ts[1:]):
        refuse("every tensor but logits and draft_probs must be contiguous")
    q_stride = 0
    if draft_probs is not None:
        if draft_probs.dtype != torch.float32 or tuple(draft_probs.shape) != (B, k, V):
            refuse(f"draft_probs must be fp32 [{B}, {k}, {V}], not {draft_probs.dtype} {tuple(draft_probs.shape)}")
        q_stride = draft_probs.stride(1)
        if draft_probs.stride(2) != 1 or draft_probs.stride(0) != k * q_stride:
            refuse(f"draft_probs must have unit last stride and rows at a fixed stride, not {draft_probs.stride()}")
    lib = _lib.load()
    dev = logits.device
    ws = torch.empty(lib.chitu_b200_spec_accept_sampled_workspace_bytes(B, k), dtype=torch.uint8, device=dev)
    out = torch.empty(B, k + 1, dtype=torch.int64, device=dev)
    accepted = torch.empty(B, dtype=torch.int32, device=dev)
    nxt = torch.empty(B, dtype=torch.int64, device=dev)
    check(lib.chitu_b200_spec_accept_sampled(ptr(logits), logits.stride(0), V, dtype_code(logits.dtype),
                                             ptr(temperatures), ptr(top_ks), ptr(top_ps), ptr(drafts), ptr(n_draft),
                                             ptr(draft_probs), q_stride, ptr(u_accept), ptr(u_draw), ptr(seq_lens),
                                             ptr(out), ptr(accepted), ptr(nxt), B, k, ptr(ws), ws.numel(),
                                             current_stream()), "spec_accept_sampled")
    return out, accepted, nxt
