"""CPU oracle for Chitu's decode hot path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
leg may import this file (prompt ③).  The product path (chitu_b200/*) never does.

Each function restates one reference operator in numpy (integer / byte arithmetic) or torch-CPU
fp32 (floating point), citing the reference file:line it follows (paths relative to the
thu-pacman/chitu tree).  Pinning: `oracle/gen_golden.py` runs the REAL reference code (its Triton
kernels under TRITON_INTERPRET=1, its torch code as is) in the authoring container and commits
the outputs under tests/golden/; tests/test_oracle_vs_golden.py checks this file against them,
plus the reference's own KAT (fused_moe.py:478-490 docstring).  Third-party arithmetic that is
not in the reference tree (flash_attn's paged decode, the closed w8a8gemm/w8a8gemv) is anchored
on the in-tree restatements (RefAttnBackend attn_backend.py:294-392; test/pytest/test_w8a8.py)
— "parity unpinned" for those two beyond that (SURVEY.md §8c).
"""
from __future__ import annotations

import math
import struct
from typing import Optional, Tuple

import numpy as np
import torch

FP8_MAX = 448.0


# ------------------------------------------------------------------------------------------------
# a3  append_to_paged_kv_cache — chitu/ops.py:50-91, kernel triton_kernels.py:18-48
# ------------------------------------------------------------------------------------------------
def append_to_paged_kv_cache(kv_cache: np.ndarray, page_table: np.ndarray, this_kv: np.ndarray,
                             old_seq_lens: np.ndarray) -> None:
    """In place. kv_cache:(num_pages, page_size, ...) ; literal 64 as in triton_kernels.py:38,42:
    row = page_table[b, len//64] * PAGE_SIZE + len % 64."""
    page_size = kv_cache.shape[1]
    flat = kv_cache.reshape(kv_cache.shape[0] * page_size, -1)
    kv = this_kv.reshape(this_kv.shape[0], -1)
    for b in range(page_table.shape[0]):
        L = int(old_seq_lens[b])
        page = int(page_table[b, L // 64])
        flat[page * page_size + L % 64] = kv[b]


# ------------------------------------------------------------------------------------------------
# a13 moe_align_block_size — fused_moe.py:314-442 (Triton 4-stage order), csrc/moe_align_kernel.cu
# ------------------------------------------------------------------------------------------------
def moe_align_block_size(topk_ids: np.ndarray, block_size: int, num_experts: int):
    """Returns (sorted_ids, expert_ids, num_tokens_post_pad, cumsum) with the reference's
    allocation conventions (fused_moe.py:491-505): sorted_ids pre-filled with numel, expert_ids
    zero-filled.  Order inside a segment: ascending flat token index (== the Triton fallback:
    program p scans its contiguous token chunk in order and chunks are ordered by p)."""
    ids = np.asarray(topk_ids).reshape(-1).astype(np.int64)
    numel = ids.size
    max_padded = numel + num_experts * (block_size - 1)
    sorted_ids = np.full(max_padded, numel, dtype=np.int32)
    expert_ids = np.zeros((max_padded + block_size - 1) // block_size, dtype=np.int32)
    counts = np.bincount(ids, minlength=num_experts)[:num_experts]
    padded = (counts + block_size - 1) // block_size * block_size
    cumsum = np.zeros(num_experts + 1, dtype=np.int32)
    cumsum[1:] = np.cumsum(padded)
    for e in range(num_experts):
        for i in range(cumsum[e], cumsum[e + 1], block_size):
            expert_ids[i // block_size] = e
    fill = cumsum[:-1].astype(np.int64).copy()
    for i in range(numel):
        e = ids[i]
        sorted_ids[fill[e]] = i
        fill[e] += 1
    return sorted_ids, expert_ids, np.array([cumsum[-1]], dtype=np.int32), cumsum


# ------------------------------------------------------------------------------------------------
# a6  rotary — ops.py:243-308 (torch reference of both layouts), kernels triton_kernels.py:51-190
# ------------------------------------------------------------------------------------------------
def rotary_interleaved(q: torch.Tensor, k: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, out_dtype=None):
    """rotary_type="llama": pairs (2i, 2i+1); cos/sin [bs, rot/2] fp32; q [bs,h,rot], k [bs,(h,)rot].
    Follows the Triton kernel (triton_kernels.py:159-163): products in fp32, one rounding
    (out_dtype=torch.float32 returns the unrounded value, used to pin against the interpreter)."""
    def rot(x):
        shape = x.shape
        x3 = x.reshape(shape[0], -1, shape[-1]).float()
        x0, x1 = x3[..., 0::2], x3[..., 1::2]
        c, s = cos.float()[:, None, :], sin.float()[:, None, :]
        o = torch.stack([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1).flatten(-2)
        return o.to(out_dtype or x.dtype).reshape(shape)
    return rot(q), rot(k)


def rotary_half(q: torch.Tensor, k: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor):
    """rotary_type="hf-llama": halves; cos/sin [bs, hd/2] in the tensor dtype
    (triton_kernels.py:87-98: every product / sum is rounded to the tensor dtype)."""
    def rot(x):
        hd = x.shape[-1]
        x0, x1 = x[..., : hd // 2], x[..., hd // 2:]
        c, s = cos.to(x.dtype)[:, None, :], sin.to(x.dtype)[:, None, :]
        return torch.cat([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1)
    return rot(q), rot(k)


# ------------------------------------------------------------------------------------------------
# a19 RMSNorm — models/model.py:50-78 ; SiluAndMul — fused_moe.py:24-39
# ------------------------------------------------------------------------------------------------
def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, compute_dtype=torch.float32):
    dtype = x.dtype
    return torch.nn.functional.rms_norm(x.to(compute_dtype), (x.shape[-1],), weight, eps).to(dtype)


def silu_and_mul(x: torch.Tensor) -> torch.Tensor:
    d = x.shape[-1] // 2
    return torch.nn.functional.silu(x[..., :d]) * x[..., d:]


# ------------------------------------------------------------------------------------------------
# a7 / a14 fp8 group quantisers
# ------------------------------------------------------------------------------------------------
def _to_fp8(v: torch.Tensor) -> torch.Tensor:
    """fp32 -> float8_e4m3fn, round-to-nearest-even, saturating (Triton's GPU conversion is
    cvt.rn.satfinite; inputs here are pre-clamped or <= 448 by construction)."""
    return v.clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)


def act_quant_deepseek_v3(x: torch.Tensor, block_size: int = 128):
    """ops.py:329-353, kernel triton_kernels.py:193-214: s = max|x|/448 (no eps), y = fp8(x/s)."""
    xf = x.float().reshape(-1, block_size)
    s = xf.abs().amax(dim=-1) / FP8_MAX
    y = _to_fp8(xf / s[:, None])
    return y.reshape(x.shape), s.reshape(*x.shape[:-1], x.shape[-1] // block_size)


def per_token_group_quant_fp8(x: torch.Tensor, group_size: int, eps: float = 1e-10):
    """fused_moe.py:667-710: s = max(max|x|, eps)/448 ; q = fp8(clamp(x/s, -448, 448))."""
    xf = x.float().reshape(-1, group_size)
    s = xf.abs().amax(dim=-1).clamp(min=eps) / FP8_MAX
    q = _to_fp8((xf / s[:, None]).clamp(-FP8_MAX, FP8_MAX))
    return q.reshape(x.shape), s.reshape(*x.shape[:-1], x.shape[-1] // group_size)


# ------------------------------------------------------------------------------------------------
# a10 weight dequant — ops.py:356-449
# ------------------------------------------------------------------------------------------------
def _expand_block_scale(s: torch.Tensor, M: int, N: int, block: int = 128) -> torch.Tensor:
    return s.repeat_interleave(block, dim=-2)[..., :M, :].repeat_interleave(block, dim=-1)[..., :N]


def weight_dequant(x_fp8: torch.Tensor, s: torch.Tensor, block: int = 128, out_dtype=torch.bfloat16):
    """triton_kernels.py:217-247: y = fp32(x) * s[block] -> default dtype (bf16 for DeepSeek)."""
    M, N = x_fp8.shape[-2:]
    return (x_fp8.float() * _expand_block_scale(s, M, N, block)).to(out_dtype)


def soft_fp8_bits_to_f32(x_fp8: torch.Tensor) -> torch.Tensor:
    """The bit trick of triton_kernels.py:250-262 / 474-491: ((x&0x80)<<24 | (x&0x7f)<<20) as fp32
    (value = fp8 value * 2^-120)."""
    u = x_fp8.view(torch.uint8).numpy().astype(np.uint32)
    bits = ((u & 0x80) << 24) | ((u & 0x7F) << 20)
    return bits.view(np.float32)


def weight_dequant_soft_fp8(x_fp8: torch.Tensor, s: torch.Tensor, block: int = 128, out_dtype=torch.bfloat16):
    """ops.py:395-449: y = bits_f32 * (s * 2^120) -> bf16."""
    M, N = x_fp8.shape[-2:]
    two120 = struct.unpack(">f", bytes.fromhex("7b800000"))[0]
    f = torch.from_numpy(soft_fp8_bits_to_f32(x_fp8).copy()).reshape(x_fp8.shape)
    return (f * (_expand_block_scale(s, M, N, block) * two120)).to(out_dtype)


# ------------------------------------------------------------------------------------------------
# a8 fp8 block GEMM — ops.py:452-483, kernel triton_kernels.py:303-365 ; a9 soft fp8 GEMM
# ------------------------------------------------------------------------------------------------
def fp8_gemm(a_fp8: torch.Tensor, a_s: torch.Tensor, b_fp8: torch.Tensor, b_s: torch.Tensor,
             out_dtype=torch.bfloat16) -> torch.Tensor:
    """c = sum_kb (a_kb · b_kb^T) * a_s[:,kb] * b_s[n//128,kb]  (fp32 accumulate per 128-K block)."""
    K = a_fp8.shape[-1]
    a = a_fp8.float().reshape(-1, K)
    M = a.shape[0]
    N = b_fp8.shape[0]
    b = b_fp8.float()
    a_s = a_s.reshape(M, -1)
    acc = torch.zeros(M, N, dtype=torch.float32)
    for kb in range((K + 127) // 128):
        sl = slice(kb * 128, min((kb + 1) * 128, K))
        part = a[:, sl] @ b[:, sl].T
        bs = b_s[:, kb].repeat_interleave(128)[:N]
        acc += part * a_s[:, kb:kb + 1] * bs[None, :]
    return acc.to(out_dtype).reshape(*a_fp8.shape[:-1], N)


def soft_fp8_gemm(a: torch.Tensor, b_fp8: torch.Tensor, b_s: torch.Tensor) -> torch.Tensor:
    """triton_kernels.py:388-508: weight -> bf16(bits * (s*2^120)), then a(bf16) x w(bf16), fp32 acc."""
    K = a.shape[-1]
    w = weight_dequant_soft_fp8(b_fp8, b_s, 128, torch.bfloat16).float()
    c = a.float().reshape(-1, K) @ w.T
    return c.to(a.dtype).reshape(*a.shape[:-1], b_fp8.shape[0])


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.linear with fp32 accumulation, one rounding (cuBLAS semantics of the reference path)."""
    y = x.float() @ w.float().T
    if bias is not None:
        y = y + bias.float()
    return y.to(x.dtype)


# ------------------------------------------------------------------------------------------------
# a17 W8A8 — quantize/w8a8.py:18-35, 96-133 ; closed kernels pinned by test/pytest/test_w8a8.py
# ------------------------------------------------------------------------------------------------
def quant_act(act: torch.Tensor):
    scales = act.abs().max(dim=-1, keepdim=True)[0].to(torch.float)
    scales.clamp_(min=1e-5).div_(127.0)
    aa = act.div(scales).round_()
    return aa.to(torch.int8).view(-1, act.shape[-1]), scales.view(-1)


def quant_weight(w: torch.Tensor):
    return quant_act(w)


def w8a8_mm(a_i8: torch.Tensor, b_i8: torch.Tensor, a_scales: torch.Tensor, b_scales: torch.Tensor,
            bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = fp16( (a·b^T in int32) * a_scale[m] * b_scale[n] ) (+ bias, fp16 add)."""
    acc = a_i8.to(torch.int32).numpy().astype(np.int64) @ b_i8.to(torch.int32).numpy().astype(np.int64).T
    out = torch.from_numpy(acc.astype(np.float32)) * a_scales.float()[:, None] * b_scales.float()[None, :]
    out = out.to(torch.float16)
    if bias is not None:
        out = out + bias
    return out


# ------------------------------------------------------------------------------------------------
# a2/a4 MLA paged decode — triton_decode_attention.py:20-290 restated as fp32 SDPA over gathered
# pages (third_party/FlashMLA/tests/test_flash_mla.py:11-28 is the same formulation)
# ------------------------------------------------------------------------------------------------
def gather_pages(cache: torch.Tensor, block_table_row: torch.Tensor, length: int) -> torch.Tensor:
    page = cache.shape[1]
    n_pages = (length + page - 1) // page
    rows = cache[block_table_row[:n_pages].long()].reshape(n_pages * page, *cache.shape[2:])
    return rows[:length]


def mla_decode(q_nope: torch.Tensor, q_pe: torch.Tensor, kv_cache: torch.Tensor, seqlens_incl: torch.Tensor,
               block_table: torch.Tensor, softmax_scale: float) -> torch.Tensor:
    """q_nope [B,H,C], q_pe [B,H,R], kv_cache [num_blocks,page,C+R] -> [B,H,C] (latent)."""
    B, H, C = q_nope.shape
    out = torch.empty(B, H, C, dtype=torch.float32)
    for b in range(B):
        L = int(seqlens_incl[b])
        rows = gather_pages(kv_cache, block_table[b], L).float()          # [L, C+R]
        q = torch.cat([q_nope[b], q_pe[b]], dim=-1).float()               # [H, C+R]
        s = (q @ rows.T) * softmax_scale
        p = torch.softmax(s, dim=-1)
        out[b] = p @ rows[:, :C]
    return out.to(q_nope.dtype)


def mla_attn_with_kvcache(q_nope, q_pe, kv_cache, kv, seqlens_excl, block_table, softmax_scale):
    """attn_backend.py:707-774: append (literal-64 paging) then decode over len+1 keys. In place."""
    B = q_nope.shape[0]
    cache_np = kv_cache.view(torch.int16).numpy()
    append_to_paged_kv_cache(cache_np, block_table.numpy(), kv.reshape(B, -1).view(torch.int16).numpy(),
                             seqlens_excl.numpy())
    return mla_decode(q_nope, q_pe, kv_cache, seqlens_excl + 1, block_table, softmax_scale)


# ------------------------------------------------------------------------------------------------
# a5 GQA paged decode with append — AttnBackend.attn_with_kvcache (attn_backend.py:92-164);
# arithmetic = RefAttnBackend._attention (attn_backend.py:294-392), paging = flash_attn semantics
# (true page_size indexing).
# ------------------------------------------------------------------------------------------------
def gqa_paged_decode(q, k_cache, v_cache, k_new, v_new, cache_seqlens, block_table, softmax_scale=None):
    """q [B,1,Hq,D]; caches [num_blocks,page,Hkv,D]; k_new/v_new [B,1,Hkv,D] or None. In place append."""
    B, _, Hq, D = q.shape
    page, Hkv = k_cache.shape[1], k_cache.shape[2]
    g = Hq // Hkv
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
    out = torch.empty(B, 1, Hq, D, dtype=torch.float32)
    for b in range(B):
        L = int(cache_seqlens[b])
        if k_new is not None:
            blk = int(block_table[b, L // page])
            k_cache[blk, L % page] = k_new[b, 0]
            v_cache[blk, L % page] = v_new[b, 0]
            L += 1
        kk = gather_pages(k_cache, block_table[b], L).float().repeat_interleave(g, dim=1)   # [L,Hq,D]
        vv = gather_pages(v_cache, block_table[b], L).float().repeat_interleave(g, dim=1)
        s = torch.einsum("hd,shd->hs", q[b, 0].float() * scale, kk)
        p = torch.softmax(s, dim=-1)
        out[b, 0] = torch.einsum("hs,shd->hd", p, vv)
    return out.to(q.dtype)


# ------------------------------------------------------------------------------------------------
# a12 gate — GateDeepSeekV3.forward, models/model_deepseek_v3.py:810-842 (verbatim semantics)
# ------------------------------------------------------------------------------------------------
def moe_gate(x, weight, bias, topk, n_groups, topk_groups, score_func, route_scale):
    scores = torch.nn.functional.linear(x, weight)
    if score_func == "softmax":
        scores = scores.softmax(dim=-1, dtype=torch.float32)
    else:
        scores = scores.sigmoid()
    original_scores = scores
    if bias is not None:
        scores = scores + bias
    if n_groups > 1:
        scores = scores.view(x.size(0), n_groups, -1)
        if bias is None:
            group_scores = scores.amax(dim=-1)
        else:
            group_scores = scores.topk(2, dim=-1)[0].sum(dim=-1)
        indices = group_scores.topk(topk_groups, dim=-1)[1]
        mask = torch.zeros_like(scores[..., 0]).scatter_(1, indices, True)
        scores = (scores * mask.unsqueeze(-1)).flatten(1)
    indices = torch.topk(scores, topk, dim=-1)[1]
    weights = original_scores.gather(1, indices)
    if score_func == "sigmoid":
        weights = weights / weights.sum(dim=-1, keepdim=True)
    weights = weights * route_scale
    return weights.type_as(x), indices, scores


# ------------------------------------------------------------------------------------------------
# a16 fused_experts — fused_moe.py:1130-1307 restated with torch (cf. the non-Triton branch of
# MoEDeepSeekV3.forward, model_deepseek_v3.py:1012-1060)
# ------------------------------------------------------------------------------------------------
def fused_experts(x, w1, w2, topk_weights, topk_ids, w1_scale=None, w2_scale=None, mode="bf16"):
    """mode: "bf16" | "fp8_w8a8" (per_token_group_quant_fp8 + block-scaled GEMM) | "soft_fp8".
    Intermediate tensors are rounded to bf16 where the reference stores them (C1, silu*mul, C3)."""
    T, K1 = x.shape
    topk = topk_ids.shape[1]
    dt = x.dtype

    def gemm(a, w, ws):
        if mode == "bf16":
            return (a.float() @ w.float().T).to(dt)
        if mode == "fp8_w8a8":
            aq, a_s = per_token_group_quant_fp8(a, 128)
            return fp8_gemm(aq, a_s, w, ws, dt)
        return soft_fp8_gemm(a, w, ws)

    c3 = torch.zeros(T, topk, K1, dtype=dt)
    for t in range(T):
        for j in range(topk):
            e = int(topk_ids[t, j])
            h = gemm(x[t:t + 1], w1[e], None if w1_scale is None else w1_scale[e])
            a2 = silu_and_mul(h)
            if mode == "bf16":
                y = a2.float() @ w2[e].float().T
            elif mode == "fp8_w8a8":
                aq, a_s = per_token_group_quant_fp8(a2, 128)
                y = fp8_gemm(aq, a_s, w2[e], w2_scale[e], torch.float32)
            else:
                wbf = weight_dequant_soft_fp8(w2[e], w2_scale[e]).float()
                y = a2.float() @ wbf.T
            c3[t, j] = (y * float(topk_weights[t, j])).to(dt)[0]
    return c3.float().sum(dim=1).to(dt)


# ------------------------------------------------------------------------------------------------
# LLaMA decode step (config 1/2 plumbing, BASELINE.md §3): the reference's model code path
# (models/model_llama.py, models/model.py:167-198, 467-474) restated for the CPU baseline.
# ------------------------------------------------------------------------------------------------
class LlamaWeights:
    """Random-init LLaMA-shaped weights (bf16) — `infer.do_load=False` in the reference."""

    def __init__(self, dim, n_layers, n_heads, n_kv_heads, ffn_dim, vocab, seed=0, n_layers_alloc=None,
                 dtype=torch.bfloat16):
        g = torch.Generator().manual_seed(seed)
        self.dim, self.n_layers, self.n_heads, self.n_kv_heads = dim, n_layers, n_heads, n_kv_heads
        self.head_dim = dim // n_heads
        self.ffn_dim, self.vocab = ffn_dim, vocab
        L = n_layers_alloc or n_layers

        def r(*shape):
            return (torch.randn(*shape, generator=g) * 0.02).to(dtype)

        kvd = n_kv_heads * self.head_dim
        self.embed = r(vocab, dim)
        self.layers = [dict(attn_norm=torch.ones(dim, dtype=dtype), ffn_norm=torch.ones(dim, dtype=dtype),
                            wq=r(dim, dim), wk=r(kvd, dim), wv=r(kvd, dim), wo=r(dim, dim), w1=r(ffn_dim, dim),
                            w3=r(ffn_dim, dim), w2=r(dim, ffn_dim)) for _ in range(L)]
        self.norm = torch.ones(dim, dtype=dtype)
        self.output = r(vocab, dim)


def llama_decode_step(wts: LlamaWeights, tokens, k_caches, v_caches, seqlens, block_table, cos, sin,
                      n_layers=None, eps=1e-5):
    """One decode step on CPU following TransformerLlama.decode_single_device (model.py:467-474).
    tokens [B] int64 ; k_caches/v_caches: list per layer [num_blocks,page,Hkv,D] ; cos/sin [B, D/2] fp32."""
    B = tokens.shape[0]
    h = wts.embed[tokens]
    H, Hkv, D = wts.n_heads, wts.n_kv_heads, wts.head_dim
    for li in range(n_layers or wts.n_layers):
        lw = wts.layers[li % len(wts.layers)]
        xn = rms_norm(h, lw["attn_norm"], eps)
        q = linear(xn, lw["wq"]).view(B, H, D)
        k = linear(xn, lw["wk"]).view(B, Hkv, D)
        v = linear(xn, lw["wv"]).view(B, Hkv, D)
        q, k = rotary_interleaved(q, k, cos, sin)
        o = gqa_paged_decode(q.view(B, 1, H, D), k_caches[li], v_caches[li], k.view(B, 1, Hkv, D),
                             v.view(B, 1, Hkv, D), seqlens, block_table)
        h = linear(o.reshape(B, H * D), lw["wo"]) + h
        xn = rms_norm(h, lw["ffn_norm"], eps)
        ff = torch.nn.functional.silu(linear(xn, lw["w1"])) * linear(xn, lw["w3"])
        h = h + linear(ff, lw["w2"])
    h = rms_norm(h, wts.norm, eps)
    return linear(h, wts.output).float()


def llama_block(lw, h, k_cache, v_cache, seqlens, block_table, cos, sin, n_heads, n_kv_heads, eps=1e-5):
    """One TransformerBlockLlama.forward in decode mode (models/model_llama.py:172-185 + Attention.decode_forward
    models/model.py:142-172): the per-layer body of `llama_decode_step`, exposed so that it can be pinned against
    the reference block (tests/golden/block_llama.npz).  h [B, dim]; paged caches are appended in place."""
    B = h.shape[0]
    H, Hkv = n_heads, n_kv_heads
    D = lw["wq"].shape[0] // H
    xn = rms_norm(h, lw["attn_norm"], eps)
    q = linear(xn, lw["wq"]).view(B, H, D)
    k = linear(xn, lw["wk"]).view(B, Hkv, D)
    v = linear(xn, lw["wv"]).view(B, Hkv, D)
    q, k = rotary_interleaved(q, k, cos, sin)
    o = gqa_paged_decode(q.view(B, 1, H, D), k_cache, v_cache, k.view(B, 1, Hkv, D), v.view(B, 1, Hkv, D), seqlens,
                         block_table)
    h = linear(o.reshape(B, H * D), lw["wo"]) + h
    xn = rms_norm(h, lw["ffn_norm"], eps)
    ff = torch.nn.functional.silu(linear(xn, lw["w1"])) * linear(xn, lw["w3"])
    return h + linear(ff, lw["w2"])


# ------------------------------------------------------------------------------------------------
# DeepSeek-V3 decode step restated from the reference model code (tp=1 shard arithmetic):
# TransformerBlockDeepSeekV3.forward (model_deepseek_v3.py:1100-1114), decode_forward_paged (:672-699),
# _run_linear absorb-without-precomp (:475-536), MLPDeepSeekV3 (:755-771), MoEDeepSeekV3 (:921-1011),
# linear_deepseek_v3 fp8 branch (:53-106).
# ------------------------------------------------------------------------------------------------
def fp8_linear(x, w, w_s):
    xq, xs = act_quant_deepseek_v3(x.contiguous(), 128)
    return fp8_gemm(xq, xs, w, w_s, x.dtype)


def deepseek_attn_half(L, h, kv_cache, seqlens, block_table, cos, sin, cfg, n_heads_local):
    """h + attn(attn_norm(h)) of TransformerBlockDeepSeekV3.forward in paged decode mode (model_deepseek_v3.py:1106-1111,
    672-699, 475-536).  h [B, dim] bf16; the paged latent cache is appended in place."""
    B = h.shape[0]
    H, C, R = n_heads_local, cfg.kv_lora_rank, cfg.qk_rope_head_dim
    dn, dv, eps = cfg.qk_nope_head_dim, cfg.v_head_dim, cfg.norm_eps
    bf = torch.bfloat16
    xn = rms_norm(h, L["attn_norm"], eps, bf)
    qkv_a = fp8_linear(xn, L["wqkv_a"], L["wqkv_a_s"])
    q_a, kv, k_pe = torch.split(qkv_a, [cfg.q_lora_rank, C, R], dim=-1)
    q = fp8_linear(rms_norm(q_a.contiguous(), L["q_norm"], eps, bf), L["wq_b"], L["wq_b_s"]).view(B, H, dn + R)
    q_nope, q_pe = torch.split(q, [dn, R], dim=-1)
    q_pe, k_pe = rotary_interleaved(q_pe, k_pe, cos, sin)
    wkv_b = weight_dequant(L["wkv_b"], L["wkv_b_s"]).view(H, dn + dv, C)
    q_abs = torch.einsum("shd,hdc->shc", q_nope.float(), wkv_b[:, :dn].float()).to(bf)
    this_kv = torch.cat([rms_norm(kv.contiguous(), L["kv_norm"], eps, bf), k_pe], dim=-1)
    x = mla_attn_with_kvcache(q_abs, q_pe.contiguous(), kv_cache, this_kv.view(B, 1, 1, -1), seqlens, block_table,
                              cfg.softmax_scale)
    o = torch.einsum("bhc,hdc->bhd", x.float(), wkv_b[:, -dv:].float()).to(bf)
    return h + fp8_linear(o.reshape(B, H * dv), L["wo"], L["wo_s"])


def deepseek_ffn_half(L, h, cfg, route_out=None):
    """h + ffn(ffn_norm(h)) (model_deepseek_v3.py:1112-1113): MLPDeepSeekV3 (:755-771) for the dense layers,
    MoEDeepSeekV3 (:921-1011: gate, shared expert = last stacked expert, fused routed experts) otherwise."""
    xn = rms_norm(h, L["ffn_norm"], cfg.norm_eps, torch.bfloat16)
    if "w13" in L:
        y = fp8_linear(silu_and_mul(fp8_linear(xn, L["w13"], L["w13_s"])), L["w2"], L["w2_s"])
    else:
        w, idx, _ = moe_gate(xn, L["gate_w"], L["gate_b"], cfg.n_activated_experts, cfg.n_expert_groups,
                             cfg.n_limited_groups, cfg.score_func, cfg.route_scale)
        if route_out is not None:
            route_out.append(idx)
        y = fp8_linear(silu_and_mul(fp8_linear(xn, L["ws13"], L["ws13_s"])), L["ws2"], L["ws2_s"])
        ne = cfg.n_routed_experts
        y = y + fused_experts(xn, L["we1"][:ne], L["we2"][:ne], w, idx, L["we1_s"][:ne], L["we2_s"][:ne], mode="fp8_w8a8")
    return h + y


def deepseek_block(L, h, kv_cache, seqlens, block_table, cos, sin, cfg, n_heads_local, route_out=None):
    """One TransformerBlockDeepSeekV3.forward in paged decode mode: the per-layer body of `deepseek_decode_step`,
    exposed in two halves so that each can be pinned against the reference block
    (tests/golden/block_deepseek_*.npz, tests/test_oracle_vs_reference_blocks.py)."""
    h = deepseek_attn_half(L, h, kv_cache, seqlens, block_table, cos, sin, cfg, n_heads_local)
    return deepseek_ffn_half(L, h, cfg, route_out)


def deepseek_decode_step(layers, embed, norm_w, head, cfg, tokens, kv_caches, seqlens, block_table, cos, sin,
                         n_heads_local, routes_out=None):
    """layers: list of dicts with the engine's tensor names (CPU copies). Returns fp32 logits."""
    B = tokens.shape[0]
    H, C, R = n_heads_local, cfg.kv_lora_rank, cfg.qk_rope_head_dim
    dn, dv, eps = cfg.qk_nope_head_dim, cfg.v_head_dim, cfg.norm_eps
    bf = torch.bfloat16
    h = embed[tokens]
    for li, L in enumerate(layers):
        xn = rms_norm(h, L["attn_norm"], eps, bf)
        qkv_a = fp8_linear(xn, L["wqkv_a"], L["wqkv_a_s"])
        q_a, kv, k_pe = torch.split(qkv_a, [cfg.q_lora_rank, C, R], dim=-1)
        q = fp8_linear(rms_norm(q_a.contiguous(), L["q_norm"], eps, bf), L["wq_b"], L["wq_b_s"]).view(B, H, dn + R)
        q_nope, q_pe = torch.split(q, [dn, R], dim=-1)
        q_pe, k_pe = rotary_interleaved(q_pe, k_pe, cos, sin)
        wkv_b = weight_dequant(L["wkv_b"], L["wkv_b_s"]).view(H, dn + dv, C)
        q_abs = torch.einsum("shd,hdc->shc", q_nope.float(), wkv_b[:, :dn].float()).to(bf)
        this_kv = torch.cat([rms_norm(kv.contiguous(), L["kv_norm"], eps, bf), k_pe], dim=-1)
        x = mla_attn_with_kvcache(q_abs, q_pe.contiguous(), kv_caches[li], this_kv.view(B, 1, 1, -1), seqlens,
                                  block_table, cfg.softmax_scale)
        o = torch.einsum("bhc,hdc->bhd", x.float(), wkv_b[:, -dv:].float()).to(bf)
        h = h + fp8_linear(o.reshape(B, H * dv), L["wo"], L["wo_s"])
        xn = rms_norm(h, L["ffn_norm"], eps, bf)
        if "w13" in L:
            y = fp8_linear(silu_and_mul(fp8_linear(xn, L["w13"], L["w13_s"])), L["w2"], L["w2_s"])
        else:
            w, idx, _ = moe_gate(xn, L["gate_w"], L["gate_b"], cfg.n_activated_experts, cfg.n_expert_groups,
                                 cfg.n_limited_groups, cfg.score_func, cfg.route_scale)
            if routes_out is not None:
                routes_out.append((li, idx))
            y = fp8_linear(silu_and_mul(fp8_linear(xn, L["ws13"], L["ws13_s"])), L["ws2"], L["ws2_s"])
            ne = cfg.n_routed_experts      # engine storage: expert index ne is the shared expert (reference :1178)
            y1 = fused_experts(xn, L["we1"][:ne], L["we2"][:ne], w, idx, L["we1_s"][:ne], L["we2_s"][:ne], mode="fp8_w8a8")
            y = y + y1
        h = h + y
    return linear(rms_norm(h, norm_w, eps, bf), head).float()


def check_kv_append(after, before, ref_after, table, lens, page: int) -> float:
    """KV-page indexing is bit exact: the step touched exactly one row per request — page table[b, L // page], slot
    L % page — and nothing else.  The appended VALUES come out of a GEMM (accumulation order differs between two correct
    implementations), so they are compared with the reference's appended rows within 1e-2 instead of bit for bit.
    Returns that max relative difference."""
    nb, pg = after.shape[0], after.shape[1]
    mask = torch.zeros(nb, pg, dtype=torch.bool, device=after.device)
    for b, L in enumerate(lens.tolist()):
        mask[int(table[b, L // page]), L % page] = True
    flat_a, flat_b = after.view(torch.int16).reshape(nb, pg, -1), before.view(torch.int16).reshape(nb, pg, -1)
    assert torch.equal(flat_a[~mask], flat_b[~mask]), "a cache row other than the appended ones changed"
    got = after.reshape(nb, pg, -1)[mask].double()
    want = ref_after.to(after.device).reshape(nb, pg, -1)[mask].double()
    rel = ((got - want).abs().max() / want.abs().max().clamp(min=1e-30)).item()
    assert rel < 1e-2, f"appended rows differ from the reference: max rel {rel}"
    return rel
