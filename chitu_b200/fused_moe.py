"""Drop-in for the hot-path entry points of `chitu/fused_moe.py`: moe_align_block_size,
per_token_group_quant_fp8, SiluAndMul, fused_experts (+ the DeepSeek gate as `moe_gate`).
Reference: thu-pacman/chitu, chitu/fused_moe.py (file:line cited per function).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from . import _lib, chitu_backend, workspace
from ._lib import check, current_stream, dtype_code, ptr, require_cuda
from .ops import silu_and_mul

__all__ = ["moe_align_block_size", "per_token_group_quant_fp8", "fused_experts", "SiluAndMul", "moe_gate",
           "invoke_fused_moe_kernel"]


def ceil_div(a, b):
    return (a + b - 1) // b


class SiluAndMul(torch.nn.Module):
    """fused_moe.py:24-39."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return silu_and_mul(x.contiguous())


def moe_align_block_size(topk_ids: torch.Tensor, block_size: int, num_experts: int,
                         expert_map: torch.Tensor = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """fused_moe.py:445-519 / 599-610: same allocations (sorted_ids pre-filled with numel,
    expert_ids zero-filled), same return tuple."""
    max_num_tokens_padded = topk_ids.numel() + num_experts * (block_size - 1)
    sorted_ids = torch.empty((max_num_tokens_padded,), dtype=torch.int32, device=topk_ids.device)
    sorted_ids.fill_(topk_ids.numel())
    max_num_m_blocks = ceil_div(max_num_tokens_padded, block_size)
    expert_ids = torch.zeros((max_num_m_blocks,), dtype=torch.int32, device=topk_ids.device)
    num_tokens_post_pad = torch.empty((1), dtype=torch.int32, device=topk_ids.device)
    cumsum_buffer = torch.zeros((num_experts + 1,), dtype=torch.int32, device=topk_ids.device)
    chitu_backend.cuda_moe_align_block_size(topk_ids.contiguous(), num_experts, block_size, sorted_ids,
                                            expert_ids, num_tokens_post_pad, cumsum_buffer)
    if expert_map is not None:
        expert_ids = expert_map[expert_ids]
    return sorted_ids, expert_ids, num_tokens_post_pad


def per_token_group_quant_fp8(x: torch.Tensor, group_size: int, eps: float = 1e-10,
                              dtype: Optional[torch.dtype] = None,
                              column_major_scales: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """fused_moe.py:713-793."""
    if dtype is None:
        dtype = torch.float8_e4m3fn
    assert dtype == torch.float8_e4m3fn, "only float8_e4m3fn is supported (as in the reference)"
    assert x.shape[-1] % group_size == 0, (
        f"the last dimension of `x` {x.shape[-1]} must be divisible by `group_size` {group_size}")
    assert x.stride(-1) == 1, "`x` groups must be contiguous"
    assert not column_major_scales, "column_major_scales is never used by the reference's callers"
    require_cuda(x)
    x = x.contiguous()
    x_q = torch.empty_like(x, dtype=dtype)
    x_s = torch.empty(x.shape[:-1] + (x.shape[-1] // group_size,), device=x.device, dtype=torch.float32)
    K = x.shape[-1]
    check(_lib.load().chitu_b200_act_quant_fp8(ptr(x), ptr(x_q), ptr(x_s), x.numel() // K, K, group_size, 1,
                                               float(eps), dtype_code(x.dtype), current_stream()),
          "per_token_group_quant_fp8")
    return x_q, x_s


def moe_gate(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], topk: int, n_groups: int,
             topk_groups: int, score_func: str, route_scale: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """GateDeepSeekV3.forward (models/model_deepseek_v3.py:810-842) -> (weights.type_as(x), indices int64).
    score_func "softmax_renorm" = the routing of SparseMoeBlockHFMixtral (model_hf_mixtral.py:57-64): softmax in fp32,
    top-k, weights /= their sum (fp32), cast to x.dtype."""
    assert x.dim() == 2 and x.is_contiguous() and weight.is_contiguous()
    assert x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16
    require_cuda(x, weight, bias)
    T, dim = x.shape
    E = weight.shape[0]
    w = torch.empty((T, topk), dtype=x.dtype, device=x.device)
    idx = torch.empty((T, topk), dtype=torch.int64, device=x.device)
    bcode = dtype_code(bias.dtype) if bias is not None else 0
    lib = _lib.load()
    ws = workspace.get("moe_gate", lib.chitu_b200_moe_gate_workspace_bytes(T, E), x.device)
    check(lib.chitu_b200_moe_gate(ptr(x), ptr(weight), ptr(bias), bcode, T, dim, E, n_groups, topk_groups,
                                  topk, {"sigmoid": 1, "softmax": 0, "softmax_renorm": 2}[score_func], float(route_scale), ptr(w),
                                  ptr(idx), topk, ptr(ws), ws.numel(), current_stream()), "moe_gate")
    return w, idx


def invoke_fused_moe_kernel(A: torch.Tensor, B: torch.Tensor, C: torch.Tensor, A_scale: Optional[torch.Tensor],
                            B_scale: Optional[torch.Tensor], B_zp: Optional[torch.Tensor], topk_weights: torch.Tensor,
                            topk_ids: torch.Tensor, sorted_token_ids: torch.Tensor, expert_ids: torch.Tensor,
                            num_tokens_post_padded: torch.Tensor, mul_routed_weight: bool, top_k: int, config: dict,
                            compute_type=None, use_fp8_w8a8: bool = False, use_int8_w8a16: bool = False,
                            use_int4_w4a16: bool = False, block_shape: Optional[List[int]] = None,
                            soft_fp8: bool = False) -> None:
    """fused_moe.py:796-891 — same signature, writes C in place.  One grouped wgmma GEMM over the blocks that
    `moe_align_block_size(topk_ids, config["BLOCK_SIZE_M"], E)` produced (BLOCK_SIZE_M in {16, 32, 64, 128}; the Triton
    tiling keys BLOCK_SIZE_N / K / GROUP_SIZE_M have no meaning here and are ignored)."""
    if use_int8_w8a16 or use_int4_w4a16 or B_zp is not None:
        raise NotImplementedError("int8_w8a16 / int4_w4a16 expert weights are outside the hot path of this library")
    assert topk_weights.stride(1) == 1
    assert sorted_token_ids.stride(0) == 1
    assert A.dtype == torch.bfloat16 and A.is_contiguous() and B.is_contiguous() and C.is_contiguous()
    require_cuda(A, B, C, topk_weights, sorted_token_ids, expert_ids, num_tokens_post_padded)
    if use_fp8_w8a8:
        assert B_scale is not None and block_shape is not None and list(block_shape) == [128, 128]
        assert A_scale is None, "the reference quantises A inside (per_token_group_quant_fp8, :826); so does the kernel"
        wmode = 2 if soft_fp8 else 1
    else:
        assert A_scale is None and B_scale is None and B.dtype == torch.bfloat16
        wmode = 0
    E, N, K = B.shape
    block_m = int(config["BLOCK_SIZE_M"])
    EM = sorted_token_ids.shape[0]
    numel = topk_ids.numel()
    tw = topk_weights.contiguous()
    if tw.dtype not in (torch.bfloat16, torch.float32):
        tw = tw.float()
    lib = _lib.load()
    ws = workspace.get("moe_gg", lib.chitu_b200_moe_grouped_gemm_workspace_bytes(EM, N, K), A.device)
    check(lib.chitu_b200_moe_grouped_gemm(
        ptr(A), ptr(B), ptr(C), ptr(B_scale.contiguous()) if B_scale is not None else None, ptr(tw), dtype_code(tw.dtype),
        ptr(sorted_token_ids), ptr(expert_ids), ptr(num_tokens_post_padded), EM, numel, int(bool(mul_routed_weight)), int(top_k),
        block_m, E, N, K, wmode, ptr(ws), ws.numel(), current_stream()), "moe_grouped_gemm")


def fused_experts(hidden_states: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, topk_weights: torch.Tensor,
                  topk_ids: torch.Tensor, inplace: bool = False, activation: str = "silu",
                  use_fp8_w8a8: bool = False, use_int8_w8a16: bool = False, use_int4_w4a16: bool = False,
                  global_num_experts: int = -1, expert_map: Optional[torch.Tensor] = None,
                  w1_scale: Optional[torch.Tensor] = None, w2_scale: Optional[torch.Tensor] = None,
                  w1_zp: Optional[torch.Tensor] = None, w2_zp: Optional[torch.Tensor] = None,
                  a1_scale: Optional[torch.Tensor] = None, a2_scale: Optional[torch.Tensor] = None,
                  block_shape: Optional[List[int]] = None, soft_fp8: bool = False) -> torch.Tensor:
    """fused_moe.py:1060-1307 — same signature.  Quantisation flags that are outside the
    north-star path are accepted and rejected with NotImplementedError (SURVEY §8b)."""
    if use_int8_w8a16 or use_int4_w4a16:
        raise NotImplementedError("int8_w8a16 / int4_w4a16 expert weights are outside the hot path of this library")
    if activation != "silu":
        raise ValueError(f"Unsupported FusedMoe activation: {activation}")
    if a1_scale is not None or a2_scale is not None or w1_zp is not None or w2_zp is not None:
        raise NotImplementedError("static activation scales / zero points are not used by the reference callers")
    assert hidden_states.shape[1] == w1.shape[2], "Hidden size mismatch"
    assert topk_weights.shape == topk_ids.shape, "topk shape mismatch"
    assert hidden_states.is_contiguous(), "Hidden_states must be contiguous"
    assert w1.is_contiguous(), "Expert weights1 must be contiguous"
    assert w2.is_contiguous(), "Expert weights2 must be contiguous"
    assert hidden_states.dtype == torch.bfloat16, "this path computes in bf16"
    require_cuda(hidden_states, w1, w2, topk_weights, topk_ids)
    T, K1 = hidden_states.shape
    E, N1, _ = w1.shape
    topk = topk_ids.shape[1]
    if use_fp8_w8a8:
        assert block_shape is not None and list(block_shape) == [128, 128], "block-wise 128x128 fp8 only"
        assert w1_scale is not None and w2_scale is not None
        wmode = 2 if soft_fp8 else 1
        w1_s, w2_s = w1_scale.contiguous(), w2_scale.contiguous()
    else:
        assert w1.dtype == torch.bfloat16 and w2.dtype == torch.bfloat16
        wmode, w1_s, w2_s = 0, None, None
    ids = topk_ids.contiguous()
    if expert_map is not None:  # expert parallelism: global -> local id, -1 = not on this rank
        ids = expert_map[ids.long()].to(torch.int32).contiguous()
    if ids.dtype not in (torch.int32, torch.int64):
        ids = ids.to(torch.int32)
    tw = topk_weights.contiguous()
    if tw.dtype not in (torch.bfloat16, torch.float32):
        tw = tw.float()
    out = hidden_states if inplace else torch.empty_like(hidden_states)
    lib = _lib.load()
    # (token, slot) pairs per launch: <= 8192 keeps every chunk on the grouped wgmma path (each distinct expert streamed
    # once per chunk); the C side accepts up to 65535 pairs (SIMT fallback above 8192)
    CHUNK = max(1, 8192 // max(topk, 1))
    for t0 in range(0, T, CHUNK):
        t1 = min(T, t0 + CHUNK)
        n = lib.chitu_b200_moe_workspace_bytes(t1 - t0, topk, E, N1, K1)
        ws = workspace.get("moe", n, hidden_states.device)
        check(lib.chitu_b200_fused_experts(
            ptr(hidden_states[t0:t1]), ptr(w1), ptr(w2), ptr(w1_s), ptr(w2_s), ptr(tw[t0:t1]), dtype_code(tw.dtype),
            ptr(ids[t0:t1]), dtype_code(ids.dtype), t1 - t0, topk, E, N1, K1, wmode, ptr(out[t0:t1]), None, ptr(ws),
            ws.numel(), current_stream()), "fused_experts")
    return out
