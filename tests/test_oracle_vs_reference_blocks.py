"""Pins the oracle's MODEL-LEVEL restatements against whole transformer blocks of the real reference
(tests/golden/block_*.npz, written by oracle/gen_golden_models.py from the reference).  CPU only."""
import numpy as np
import torch

from conftest import Golden, cos_diff, max_rel
from oracle import chitu_oracle as O

BF = torch.bfloat16


def trunc_bf16(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16 by truncation (what the Triton 3.6 CPU interpreter does on a bf16 store)."""
    return (t.contiguous().view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)


def paged_from_contiguous(cache, page):
    """[B, max_len, Hkv, D] -> ([B*max_len/page, page, Hkv, D], block_table [B, max_len/page]) with shuffled pages."""
    B, max_len = cache.shape[:2]
    per = max_len // page
    g = torch.Generator().manual_seed(5)
    perm = torch.randperm(B * per, generator=g)
    table = perm.view(B, per).to(torch.int32)
    paged = torch.empty(B * per, page, *cache.shape[2:], dtype=cache.dtype)
    for b in range(B):
        for j in range(per):
            paged[table[b, j]] = cache[b, j * page:(j + 1) * page]
    return paged, table


def test_llama_block_vs_reference():
    """TransformerBlockLlama decode (models/model_llama.py:172-185, models/model.py:142-172, RefAttnBackend) on
    CPU in bf16 vs the oracle's per-layer body, fed through a PAGED cache with shuffled pages."""
    g = Golden("block_llama")
    dim, H, Hkv = (int(v) for v in g.np("cfg"))
    lw = dict(attn_norm=g.t("attention_norm__weight", BF), ffn_norm=g.t("ffn_norm__weight", BF),
              wq=g.t("attention__wq__weight", BF), wk=g.t("attention__wk__weight", BF),
              wv=g.t("attention__wv__weight", BF), wo=g.t("attention__wo__weight", BF),
              w1=g.t("feed_forward__w1__weight", BF), w2=g.t("feed_forward__w2__weight", BF),
              w3=g.t("feed_forward__w3__weight", BF))
    x = g.t("x", BF)[:, 0]
    seqlens = g.t("seqlens").to(torch.int32)
    page = 16
    kp, table = paged_from_contiguous(g.t("k_cache", BF), page)
    vp, _ = paged_from_contiguous(g.t("v_cache", BF), page)
    y = O.llama_block(lw, x, kp, vp, seqlens, table, g.t("cos"), g.t("sin"), H, Hkv, eps=1e-5)
    ref = g.t("y", BF)[:, 0].float()
    assert cos_diff(y.float(), ref) < 1e-5
    # bf16 end to end on both sides: a few roundings apart at most
    assert (y.float() - ref).abs().max() <= 2 * 2.0 ** -7 * ref.abs().max()
    # the appended K / V rows landed on the right page.  V is bit exact; K went through the reference's Triton
    # rotary kernel whose bf16 store TRUNCATES under the CPU interpreter (see test_oracle_vs_golden.py), so it is
    # compared with the truncated fp32 rotary and is within one bf16 ulp of the oracle's RNE value.
    k_after, v_after = g.t("k_after", BF), g.t("v_after", BF)
    xn = O.rms_norm(x, lw["attn_norm"], 1e-5)
    D = dim // H
    q32, k32 = O.rotary_interleaved(O.linear(xn, lw["wq"]).view(-1, H, D), O.linear(xn, lw["wk"]).view(-1, Hkv, D),
                                    g.t("cos"), g.t("sin"), out_dtype=torch.float32)
    for b in range(x.shape[0]):
        L = int(seqlens[b])
        blk = int(table[b, L // page])
        assert torch.equal(vp[blk, L % page], v_after[b, L])
        assert torch.equal(trunc_bf16(k32[b]), k_after[b, L])
        assert (kp[blk, L % page].float() - k_after[b, L].float()).abs().max() <= 2.0 ** -7 * k_after[b, L].float().abs().max()
        # rows that were not appended are untouched
        assert torch.equal(g.t("k_cache", BF)[b, :L], k_after[b, :L])


def test_llama_decode_step_is_the_block_composition():
    """`llama_decode_step` (used by smoke(), the engine tests and the CPU baseline) = embedding + llama_block per
    layer + norm + head, bit for bit."""
    W = O.LlamaWeights(dim=128, n_layers=2, n_heads=4, n_kv_heads=2, ffn_dim=256, vocab=97, seed=3)
    B, page, per = 2, 16, 3
    g = torch.Generator().manual_seed(9)
    kc = [torch.randn(B * per, page, 2, 32, generator=g).to(BF) for _ in range(2)]
    vc = [torch.randn(B * per, page, 2, 32, generator=g).to(BF) for _ in range(2)]
    table = torch.arange(B * per, dtype=torch.int32).view(B, per)
    seqlens = torch.tensor([20, 7], dtype=torch.int32)
    tokens = torch.tensor([5, 60])
    ang = torch.rand(B, 16, generator=g) * 6.28
    cos, sin = torch.cos(ang), torch.sin(ang)
    kc2, vc2 = [c.clone() for c in kc], [c.clone() for c in vc]
    logits = O.llama_decode_step(W, tokens, kc, vc, seqlens, table, cos, sin)
    h = W.embed[tokens]
    for li in range(2):
        h = O.llama_block(W.layers[li], h, kc2[li], vc2[li], seqlens, table, cos, sin, 4, 2)
    ref = O.linear(O.rms_norm(h, W.norm, 1e-5), W.output).float()
    assert torch.equal(logits, ref)
    assert all(torch.equal(a, b) for a, b in zip(kc, kc2))


# ------------------------------------------------------------------------------------------- DeepSeek-V3 blocks
def _deepseek_case(tag):
    from types import SimpleNamespace

    from oracle.synth_blocks import checksum, deepseek_args, synth_deepseek_block
    g = Golden(f"block_deepseek_{tag}")
    a = deepseek_args()
    layer_id, seed = int(g.np("layer_id")[0]), int(g.np("seed")[0])
    P, I = synth_deepseek_block(a, layer_id, seed)
    if int(checksum(P, I)[0]) != int(g.np("checksum")[0]):
        import pytest
        pytest.skip("seed-regenerated weights differ from the generator's (torch CPU RNG differs from the authoring image)")
    L = dict(attn_norm=P["attn_norm.weight"], ffn_norm=P["ffn_norm.weight"], q_norm=P["attn.q_norm.weight"],
             kv_norm=P["attn.kv_norm.weight"], wqkv_a=P["attn.wqkv_a.weight"], wqkv_a_s=P["attn.wqkv_a.scale"],
             wq_b=P["attn.wq_b.weight"], wq_b_s=P["attn.wq_b.scale"], wkv_b=P["attn.wkv_b.weight"],
             wkv_b_s=P["attn.wkv_b.scale"], wo=P["attn.wo.weight"], wo_s=P["attn.wo.scale"])
    if layer_id < a.n_dense_layers:
        L.update(w13=P["ffn.w1w3.weight"], w13_s=P["ffn.w1w3.scale"], w2=P["ffn.w2.weight"], w2_s=P["ffn.w2.scale"])
    else:
        # reference storage: experts [0, n_routed) routed, the last one shared (model_deepseek_v3.py:935-947, 1178)
        L.update(gate_w=P["ffn.gate.weight"], gate_b=P["ffn.gate.bias"], we1=P["ffn.w1w3.weight"],
                 we1_s=P["ffn.w1w3.scale"], we2=P["ffn.w2.weight"], we2_s=P["ffn.w2.scale"],
                 ws13=P["ffn.w1w3.weight"][-1], ws13_s=P["ffn.w1w3.scale"][-1], ws2=P["ffn.w2.weight"][-1],
                 ws2_s=P["ffn.w2.scale"][-1])
    cfg = SimpleNamespace(**vars(a))
    cfg.softmax_scale = float(g.np("softmax_scale")[0])
    return g, a, cfg, L, I


class interpreter_arithmetic:
    """The golden blocks were produced by the reference's Triton kernels under the Triton 3.6 CPU interpreter, whose
    fp32->bf16 cast truncates and whose fp32->fp8 cast rounds half up and can lose the carry into the exponent
    (triton/runtime/interpreter.py::_convert_float).  Inside this context the oracle's roundings AT THE OUTPUTS OF
    THE REFERENCE'S TRITON KERNELS (act_quant / group quant -> fp8, fp8 GEMM / weight_dequant / rotary -> bf16) use
    that arithmetic — the interpreter's own conversion routine for fp8 — so that the comparison with the reference
    is (nearly) bit for bit instead of being drowned in interpreter noise.  Everything else (torch ops of the model
    code: RMSNorm, einsum, SiLU, residuals) is untouched."""

    def __enter__(self):
        import triton.language as tl
        from triton._C.libtriton import ir as _ir
        from triton.runtime.interpreter import _convert_float

        def interp_fp8(v):
            a = v.float().contiguous().numpy()
            out = _convert_float(a, tl.float32, tl.float8e4nv, _ir.ROUNDING_MODE.RTNE)
            return torch.from_numpy(np.array(out, dtype=np.uint8).reshape(a.shape)).view(torch.float8_e4m3fn)

        self.saved = dict(_to_fp8=O._to_fp8, fp8_gemm=O.fp8_gemm, weight_dequant=O.weight_dequant,
                          rotary_interleaved=O.rotary_interleaved)
        sv = self.saved

        def fp8_gemm(a, a_s, b, b_s, out_dtype=BF):
            c = sv["fp8_gemm"](a, a_s, b, b_s, torch.float32)
            return trunc_bf16(c) if out_dtype == BF else c.to(out_dtype)

        def weight_dequant(x, s, block=128, out_dtype=BF):
            assert out_dtype == BF
            return trunc_bf16(sv["weight_dequant"](x, s, block, torch.float32))

        def rotary_interleaved(q, k, cos, sin, out_dtype=None):
            assert out_dtype is None and q.dtype == BF
            a, b = sv["rotary_interleaved"](q, k, cos, sin, out_dtype=torch.float32)
            return trunc_bf16(a), trunc_bf16(b)

        O._to_fp8, O.fp8_gemm, O.weight_dequant, O.rotary_interleaved = interp_fp8, fp8_gemm, weight_dequant, rotary_interleaved
        return self

    def __exit__(self, *exc):
        for k, v in self.saved.items():
            setattr(O, k, v)
        return False


def close_bf16(a, b, ulps=2):
    """max |a - b| within `ulps` bf16 spacings of the largest reference element (the residual stream adds numbers
    of that size, so a per-element relative bound is meaningless near its zero crossings)"""
    a, b = a.float(), b.float()
    top = float(b.abs().max())
    return float((a - b).abs().max()) <= ulps * 2.0 ** (np.floor(np.log2(top)) - 7)


def _check_deepseek_block(tag):
    g, a, cfg, L, I = _deepseek_case(tag)
    # the reference's own softmax scale (compute_softmax_scale_deepseek_v3, :1441-1445): 192^-1/2 * (0.1 ln 40 + 1)^2
    assert abs(cfg.softmax_scale - 192 ** -0.5 * (0.1 * np.log(40.0) + 1.0) ** 2) < 1e-12
    x = I["x"][:, 0]
    h_mid_ref, y_ref = g.t("h_mid", BF)[:, 0], g.t("y", BF)[:, 0]
    page = I["kv_cache"].shape[1]
    rows = g.t("kv_new_rows", BF)

    # ---- (1) interpreter arithmetic: attention half from x, FFN half teacher-forced from the reference's h_mid
    with interpreter_arithmetic():
        cache = I["kv_cache"].clone()
        h_mid = O.deepseek_attn_half(L, x, cache, I["seqlens"], I["table"], I["cos"], I["sin"], cfg, a.n_heads)
        route = []
        y = O.deepseek_ffn_half(L, h_mid_ref, cfg, route)
    # appended latent rows [kv_norm(kv) | rotary(k_pe)]: bit exact, on the right page, nothing else touched
    touched = torch.zeros(cache.shape[:2], dtype=torch.bool)
    for b in range(rows.shape[0]):
        Lb = int(I["seqlens"][b])
        blk = int(I["table"][b, Lb // page])
        touched[blk, Lb % page] = True
        assert torch.equal(cache[blk, Lb % page], rows[b])
    assert torch.equal(cache[~touched], I["kv_cache"][~touched])
    # residual stream after attention: q/k/v chain is bit exact, the absorb einsums and the softmax accumulate in a
    # different order (torch bf16 einsum / Triton split-KV vs fp32 here) -> a couple of bf16 ulps
    assert cos_diff(h_mid.float(), h_mid_ref.float()) < 1e-6
    assert close_bf16(h_mid, h_mid_ref)
    if route:   # routing: indices exact, weights within one bf16 ulp
        assert torch.equal(route[0], g.t("route_idx"))
    # dense MLP: bit-level agreement up to accumulation order.  MoE: the routed-weight multiply + bf16 store inside
    # the reference's fused_moe_kernel truncates (interpreter) where the oracle rounds, one ulp per (token, expert)
    # before the top-k sum -> a few 1e-6 of cos_diff
    assert cos_diff(y.float(), y_ref.float()) < (2e-5 if route else 1e-6)
    assert close_bf16(y, y_ref, ulps=3 if route else 2)

    # ---- (2) the oracle as the GPU tests use it (RNE everywhere): same structure, interpreter noise on top
    cache2 = I["kv_cache"].clone()
    y2 = O.deepseek_block(L, x, cache2, I["seqlens"], I["table"], I["cos"], I["sin"], cfg, a.n_heads)
    assert cos_diff(y2.float(), y_ref.float()) < 1e-2
    for b in range(rows.shape[0]):
        Lb = int(I["seqlens"][b])
        got = cache2[int(I["table"][b, Lb // page]), Lb % page].float()
        assert cos_diff(got, rows[b].float()) < 1e-2


def test_deepseek_dense_block_vs_reference():
    _check_deepseek_block("dense")


def test_deepseek_moe_block_vs_reference():
    _check_deepseek_block("moe")


def test_deepseek_decode_step_is_the_block_composition():
    """`deepseek_decode_step` (the checker of the engine tests) = embedding + deepseek_block per layer + norm + head."""
    from types import SimpleNamespace

    from oracle.synth_blocks import deepseek_args, synth_deepseek_block
    a = deepseek_args()
    cfg = SimpleNamespace(**vars(a))
    cfg.softmax_scale = 0.1352
    layers, I = [], None
    for layer_id, tag in ((0, "dense"), (1, "moe")):
        g, _, _, L, I = _deepseek_case(tag)
        layers.append(L)
    gen = torch.Generator().manual_seed(4)
    embed = (torch.randn(64, a.dim, generator=gen)).to(BF)
    head = (torch.randn(32, a.dim, generator=gen) / a.dim ** 0.5).to(BF)
    norm_w = torch.ones(a.dim, dtype=BF)
    tokens = torch.tensor([3, 17, 40])
    caches = [I["kv_cache"].clone(), I["kv_cache"].clone()]
    caches2 = [c.clone() for c in caches]
    logits = O.deepseek_decode_step(layers, embed, norm_w, head, cfg, tokens, caches, I["seqlens"], I["table"],
                                    I["cos"], I["sin"], a.n_heads)
    h = embed[tokens]
    for li in range(2):
        h = O.deepseek_block(layers[li], h, caches2[li], I["seqlens"], I["table"], I["cos"], I["sin"], cfg, a.n_heads)
    ref = O.linear(O.rms_norm(h, norm_w, cfg.norm_eps, BF), head).float()
    assert torch.equal(logits, ref)
    assert all(torch.equal(x, y) for x, y in zip(caches, caches2))


# ------------------------------------------------------------------------------------------- Mixtral sparse MoE
def test_mixtral_sparse_moe_block_vs_reference():
    """SparseMoeBlockHFMixtral (model_hf_mixtral.py:51-96, SURVEY a21) = router linear -> softmax(fp32) -> top-2 ->
    renormalise -> the fused-experts arithmetic with bf16 weights.  Pure torch on the reference side: no interpreter
    involved, so this is a clean pin of `fused_experts(mode="bf16")` and of the softmax routing."""
    g = Golden("block_mixtral_moe")
    E, topk = (int(v) for v in g.np("cfg"))
    x = g.t("x", BF)
    logits = O.linear(x, g.t("gate_w", BF))
    probs = torch.softmax(logits, dim=-1, dtype=torch.float32)
    w, idx = torch.topk(probs, topk, dim=-1)
    w = (w / w.sum(dim=-1, keepdim=True)).to(BF)
    y = O.fused_experts(x, g.t("w1", BF), g.t("w2", BF), w, idx, mode="bf16")
    ref = g.t("y", BF).float()
    assert cos_diff(y.float(), ref) < 1e-5
    # bf16 on both sides; the reference adds the two expert outputs in bf16 (index_add_), the oracle in fp32
    assert (y.float() - ref).abs().max() <= 2 * 2.0 ** -8 * ref.abs().max()
    # the oracle's own gate with score_func="softmax" returns the UNnormalised softmax weights of the same experts
    w2, idx2, _ = O.moe_gate(x, g.t("gate_w", BF), None, topk, 1, 1, "softmax", 1.0)
    assert torch.equal(idx2, idx)
