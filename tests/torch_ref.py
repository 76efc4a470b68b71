"""TEST INFRASTRUCTURE — device-agnostic fp32 torch restatements of the oracle's model-level functions, so that
full-width parity (dim 7168, 257 experts, S = 4096) can be checked ON THE GPU in seconds (SURVEY Appendix A:
"full-size parity on the GPU is checked against the torch fp32 restatements running on GPU").

Every function mirrors the function of the same name in oracle/chitu_oracle.py (which cites the reference lines and is
pinned against the reference's goldens); `tests/test_torch_ref_cpu.py` proves the two agree on CPU at small shapes.
Only tests import this module.
"""
from __future__ import annotations

import math

import torch

FP8_MAX = 448.0
BF = torch.bfloat16


def rms_norm(x, w, eps, compute_dtype=torch.float32):
    return torch.nn.functional.rms_norm(x.to(compute_dtype), (x.shape[-1],), w.to(compute_dtype), eps).to(x.dtype)


def silu_and_mul(x):
    d = x.shape[-1] // 2
    return torch.nn.functional.silu(x[..., :d]) * x[..., d:]


def act_quant(x, block=128):
    """act_quant_deepseek_v3 (ops.py:329-353): s = max|x|/448, y = fp8(x/s)."""
    xf = x.float().reshape(-1, block)
    s = xf.abs().amax(dim=-1) / FP8_MAX
    y = (xf / s[:, None]).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
    return y.reshape(x.shape), s.reshape(*x.shape[:-1], x.shape[-1] // block)


def group_quant(x, group=128, eps=1e-10):
    """per_token_group_quant_fp8 (fused_moe.py:667-710)."""
    xf = x.float().reshape(-1, group)
    s = xf.abs().amax(dim=-1).clamp(min=eps) / FP8_MAX
    q = (xf / s[:, None]).clamp(-FP8_MAX, FP8_MAX).to(torch.float8_e4m3fn)
    return q.reshape(x.shape), s.reshape(*x.shape[:-1], x.shape[-1] // group)


def fp8_gemm(a_q, a_s, b_q, b_s, out_dtype=BF):
    """c = sum_kb (a_kb . b_kb^T) * a_s[:,kb] * b_s[n//128,kb]   (triton_kernels.py:303-365), batched over K blocks."""
    K = a_q.shape[-1]
    M = a_q.numel() // K
    N = b_q.shape[0]
    kb = (K + 127) // 128
    assert K % 128 == 0
    a = a_q.float().reshape(M, kb, 128)
    b = b_q.float().reshape(N, kb, 128)
    part = torch.einsum("mkc,nkc->kmn", a, b)                                   # [kb, M, N] fp32 dots per K block
    bs = b_s.float().repeat_interleave(128, dim=0)[:N]                          # [N, kb]
    acc = torch.zeros(M, N, dtype=torch.float32, device=a_q.device)
    for k in range(kb):                                                         # same accumulation order as the oracle
        acc += part[k] * a_s.reshape(M, kb)[:, k:k + 1] * bs[:, k][None, :]
    return acc.to(out_dtype)


def fp8_linear(x, w, w_s):
    xq, xs = act_quant(x.contiguous())
    return fp8_gemm(xq, xs, w, w_s, x.dtype)


def weight_dequant(w, s, out_dtype=BF):
    N, K = w.shape[-2:]
    se = s.repeat_interleave(128, dim=-2)[..., :N, :].repeat_interleave(128, dim=-1)[..., :K]
    return (w.float() * se).to(out_dtype)


def rotary_interleaved(q, k, cos, sin):
    def rot(x):
        shape = x.shape
        x3 = x.reshape(shape[0], -1, shape[-1]).float()
        x0, x1 = x3[..., 0::2], x3[..., 1::2]
        c, s = cos.float()[:, None, :], sin.float()[:, None, :]
        return torch.stack([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1).flatten(-2).to(x.dtype).reshape(shape)
    return rot(q), rot(k)


def mla_attn_with_kvcache(q_nope, q_pe, kv_cache, kv, seqlens_excl, block_table, scale):
    """append (literal-64 paging, ops.py:50-91) then fp32 softmax attention over len+1 rows; in place."""
    B, H, C = q_nope.shape
    page = kv_cache.shape[1]
    out = torch.empty(B, H, C, dtype=torch.float32, device=q_nope.device)
    lens = seqlens_excl.tolist()
    for b in range(B):
        L = lens[b]
        kv_cache[block_table[b, L // 64].long(), L % 64] = kv.reshape(B, -1)[b]
        n_pages = (L + 1 + page - 1) // page
        rows = kv_cache[block_table[b, :n_pages].long()].reshape(n_pages * page, -1)[: L + 1].float()
        q = torch.cat([q_nope[b], q_pe[b]], dim=-1).float()
        p = torch.softmax((q @ rows.T) * scale, dim=-1)
        out[b] = p @ rows[:, :C]
    return out.to(q_nope.dtype)


def gqa_paged_decode(q, k_cache, v_cache, k_new, v_new, lens, block_table, scale=None):
    B, _, Hq, D = q.shape
    page, Hkv = k_cache.shape[1], k_cache.shape[2]
    g = Hq // Hkv
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    out = torch.empty(B, 1, Hq, D, dtype=torch.float32, device=q.device)
    ll = lens.tolist()
    for b in range(B):
        L = ll[b]
        if k_new is not None:
            blk = block_table[b, L // page].long()
            k_cache[blk, L % page] = k_new[b, 0]
            v_cache[blk, L % page] = v_new[b, 0]
            L += 1
        n_pages = (L + page - 1) // page
        kk = k_cache[block_table[b, :n_pages].long()].reshape(n_pages * page, Hkv, D)[:L].float()
        vv = v_cache[block_table[b, :n_pages].long()].reshape(n_pages * page, Hkv, D)[:L].float()
        qb = (q[b, 0].float() * scale).view(Hkv, g, D)
        s = torch.einsum("kgd,skd->kgs", qb, kk)
        p = torch.softmax(s, dim=-1)
        out[b, 0] = torch.einsum("kgs,skd->kgd", p, vv).reshape(Hq, D)
    return out.to(q.dtype)


def moe_gate(x, weight, bias, topk, n_groups, topk_groups, score_func, route_scale):
    """GateDeepSeekV3.forward (model_deepseek_v3.py:810-842), verbatim semantics (== oracle.moe_gate)."""
    scores = torch.nn.functional.linear(x, weight)
    scores = scores.softmax(dim=-1, dtype=torch.float32) if score_func == "softmax" else scores.sigmoid()
    original = scores
    if bias is not None:
        scores = scores + bias
    if n_groups > 1:
        scores = scores.view(x.size(0), n_groups, -1)
        gs = scores.amax(dim=-1) if bias is None else scores.topk(2, dim=-1)[0].sum(dim=-1)
        idx = gs.topk(topk_groups, dim=-1)[1]
        mask = torch.zeros_like(scores[..., 0]).scatter_(1, idx, True)
        scores = (scores * mask.unsqueeze(-1)).flatten(1)
    indices = torch.topk(scores, topk, dim=-1)[1]
    weights = original.gather(1, indices)
    if score_func == "sigmoid":
        weights = weights / weights.sum(dim=-1, keepdim=True)
    weights = weights * route_scale
    return weights.type_as(x), indices, scores


def fused_experts(x, w1, w2, topk_w, topk_ids, w1_s=None, w2_s=None, mode="bf16"):
    """fused_moe.py:1130-1307 restated per DISTINCT expert (all of its tokens at once) instead of per pair; the
    per-element arithmetic and the bf16 roundings (C1, silu*mul, C3, final sum) are those of oracle.fused_experts."""
    T, K1 = x.shape
    topk = topk_ids.shape[1]
    c3 = torch.zeros(T, topk, K1, dtype=x.dtype, device=x.device)
    xq = xs = None
    if mode == "fp8_w8a8":
        xq, xs = group_quant(x)
    for e in torch.unique(topk_ids).tolist():
        tok, slot = (topk_ids == e).nonzero(as_tuple=True)
        if mode == "bf16":
            h = (x[tok].float() @ w1[e].float().T).to(x.dtype)
            a2 = silu_and_mul(h)
            y = a2.float() @ w2[e].float().T
        elif mode == "fp8_w8a8":
            h = fp8_gemm(xq[tok], xs[tok], w1[e], w1_s[e], x.dtype)
            a2 = silu_and_mul(h)
            aq, a_s = group_quant(a2)
            y = fp8_gemm(aq, a_s, w2[e], w2_s[e], torch.float32)
        else:
            raise ValueError(mode)
        c3[tok, slot] = (y * topk_w[tok, slot].float()[:, None]).to(x.dtype)
    return c3.float().sum(dim=1).to(x.dtype)


def llama_decode_step(layers, embed, norm_w, head, tokens, k_caches, v_caches, lens, block_table, cos, sin, n_heads,
                      n_kv_heads, eps):
    """== oracle.llama_decode_step with the ENGINE's merged weights (wqkv = [wq; wk; wv], w13 = [w1; w3])."""
    B = tokens.shape[0]
    h = embed[tokens]
    D = layers[0]["wqkv"].shape[0] // (n_heads + 2 * n_kv_heads)

    def lin(x, w):
        return (x.float() @ w.float().T).to(x.dtype)

    for li, lw in enumerate(layers):
        xn = rms_norm(h, lw["attn_norm"], eps)
        qkv = lin(xn, lw["wqkv"])
        q = qkv[:, : n_heads * D].reshape(B, n_heads, D)
        k = qkv[:, n_heads * D: (n_heads + n_kv_heads) * D].reshape(B, n_kv_heads, D)
        v = qkv[:, (n_heads + n_kv_heads) * D:].reshape(B, n_kv_heads, D)
        q, k = rotary_interleaved(q, k, cos, sin)
        o = gqa_paged_decode(q.view(B, 1, n_heads, D), k_caches[li], v_caches[li], k.view(B, 1, n_kv_heads, D),
                             v.view(B, 1, n_kv_heads, D), lens, block_table)
        h = lin(o.reshape(B, n_heads * D), lw["wo"]) + h
        xn = rms_norm(h, lw["ffn_norm"], eps)
        F = lw["w13"].shape[0] // 2
        gu = lin(xn, lw["w13"])
        ff = torch.nn.functional.silu(gu[:, :F]) * gu[:, F:]
        h = h + lin(ff, lw["w2"])
    return lin(rms_norm(h, norm_w, eps), head).float()


def deepseek_layer(L, h, kv_cache, lens, block_table, cos, sin, cfg, H, route_out=None):
    """One TransformerBlockDeepSeekV3.forward in paged decode mode (== oracle.deepseek_block): h [B, dim] -> h'."""
    B = h.shape[0]
    C, R = cfg.kv_lora_rank, cfg.qk_rope_head_dim
    dn, dv, eps = cfg.qk_nope_head_dim, cfg.v_head_dim, cfg.norm_eps
    xn = rms_norm(h, L["attn_norm"], eps, BF)
    qkv_a = fp8_linear(xn, L["wqkv_a"], L["wqkv_a_s"])
    q_a, kv, k_pe = torch.split(qkv_a, [cfg.q_lora_rank, C, R], dim=-1)
    q = fp8_linear(rms_norm(q_a.contiguous(), L["q_norm"], eps, BF), L["wq_b"], L["wq_b_s"]).view(B, H, dn + R)
    q_nope, q_pe = torch.split(q, [dn, R], dim=-1)
    q_pe, k_pe = rotary_interleaved(q_pe, k_pe, cos, sin)
    wkv_b = weight_dequant(L["wkv_b"], L["wkv_b_s"]).view(H, dn + dv, C)
    q_abs = torch.einsum("shd,hdc->shc", q_nope.float(), wkv_b[:, :dn].float()).to(BF)
    this_kv = torch.cat([rms_norm(kv.contiguous(), L["kv_norm"], eps, BF), k_pe], dim=-1)
    x = mla_attn_with_kvcache(q_abs, q_pe.contiguous(), kv_cache, this_kv, lens, block_table, cfg.softmax_scale)
    o = torch.einsum("bhc,hdc->bhd", x.float(), wkv_b[:, -dv:].float()).to(BF)
    h = h + fp8_linear(o.reshape(B, H * dv), L["wo"], L["wo_s"])
    xn = rms_norm(h, L["ffn_norm"], eps, BF)
    if "w13" in L:
        y = fp8_linear(silu_and_mul(fp8_linear(xn, L["w13"], L["w13_s"])), L["w2"], L["w2_s"])
    else:
        w, idx, sc = moe_gate(xn, L["gate_w"], L["gate_b"], cfg.n_activated_experts, cfg.n_expert_groups,
                              cfg.n_limited_groups, cfg.score_func, cfg.route_scale)
        if route_out is not None:
            route_out.append((idx, sc))
        ne = cfg.n_routed_experts
        y = fp8_linear(silu_and_mul(fp8_linear(xn, L["we1"][ne], L["we1_s"][ne])), L["we2"][ne], L["we2_s"][ne])
        y = y + fused_experts(xn, L["we1"][:ne], L["we2"][:ne], w, idx, L["we1_s"][:ne], L["we2_s"][:ne], "fp8_w8a8")
    return h + y


def deepseek_decode_step(layers, embed, norm_w, head, cfg, tokens, kv_caches, lens, block_table, cos, sin, H,
                         routes_out=None, trace=None):
    """== oracle.deepseek_decode_step (model_deepseek_v3.py:1100-1114, :672-699, :475-536, :755-771, :921-1011)."""
    h = embed[tokens]
    for li, L in enumerate(layers):
        r = []
        h = deepseek_layer(L, h, kv_caches[li], lens, block_table, cos, sin, cfg, H, r)
        if routes_out is not None and r:
            routes_out.append((li, r[0][0], r[0][1]))
        if trace is not None:
            trace.append(dict(h_out=h.clone()))
    h = rms_norm(h, norm_w, cfg.norm_eps, BF)
    return (h.float() @ head.float().T).to(BF).float()

def rotary_half(q, k, cos, sin):
    """rotary_type="hf-llama" (triton_kernels.py:87-98): halves, every product / sum rounded to the tensor dtype."""
    def rot(x):
        hd = x.shape[-1]
        x0, x1 = x[..., : hd // 2], x[..., hd // 2:]
        c, s = cos.to(x.dtype)[:, None, :], sin.to(x.dtype)[:, None, :]
        return torch.cat([x0 * c - x1 * s, x1 * c + x0 * s], dim=-1)
    return rot(q), rot(k)


def mixtral_moe_block(x, gate_w, w1, w2, topk):
    """SparseMoeBlockHFMixtral.forward (model_hf_mixtral.py:51-96) through the fused-experts arithmetic (== the pinned
    oracle formulation of tests/test_oracle_vs_reference_blocks.py::test_mixtral_sparse_moe_block_vs_reference)."""
    logits = (x.float() @ gate_w.float().T).to(x.dtype)
    probs = torch.softmax(logits, dim=-1, dtype=torch.float32)
    w, idx = torch.topk(probs, topk, dim=-1)
    w = (w / w.sum(dim=-1, keepdim=True)).to(x.dtype)
    return fused_experts(x, w1, w2, w, idx), idx


def mixtral_decode_step(layers, embed, norm_w, head, tokens, k_caches, v_caches, lens, block_table, cos, sin, n_heads,
                        n_kv_heads, topk, eps):
    """hf-llama attention (model_hf_llama.py:139-252) + the Mixtral sparse-MoE block, engine weight names."""
    B = tokens.shape[0]
    h = embed[tokens]
    D = layers[0]["wqkv"].shape[0] // (n_heads + 2 * n_kv_heads)

    def lin(x, w):
        return (x.float() @ w.float().T).to(x.dtype)

    routes = []
    for li, lw in enumerate(layers):
        xn = rms_norm(h, lw["attn_norm"], eps)
        qkv = lin(xn, lw["wqkv"])
        q = qkv[:, : n_heads * D].reshape(B, n_heads, D)
        k = qkv[:, n_heads * D: (n_heads + n_kv_heads) * D].reshape(B, n_kv_heads, D)
        v = qkv[:, (n_heads + n_kv_heads) * D:].reshape(B, n_kv_heads, D)
        q, k = rotary_half(q, k, cos, sin)
        o = gqa_paged_decode(q.view(B, 1, n_heads, D), k_caches[li], v_caches[li], k.view(B, 1, n_kv_heads, D),
                             v.view(B, 1, n_kv_heads, D), lens, block_table)
        h = lin(o.reshape(B, n_heads * D), lw["wo"]) + h
        xn = rms_norm(h, lw["ffn_norm"], eps)
        y, idx = mixtral_moe_block(xn, lw["gate_w"], lw["w1"], lw["w2"], topk)
        routes.append(idx)
        h = h + y
    return lin(rms_norm(h, norm_w, eps), head).float(), routes
