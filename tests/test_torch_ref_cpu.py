"""tests/torch_ref.py (the device-agnostic restatement the full-width GPU tests run on the GPU) must agree with the
pinned oracle on CPU — bit for bit where both do the same fp32 arithmetic in the same order."""
import torch

import torch_ref as R
from oracle import chitu_oracle as O
from oracle.synth_blocks import quant_fp8_block

BF = torch.bfloat16


def _w(g, n, k):
    return quant_fp8_block(torch.randn(n, k, generator=g) * 0.02)


def test_fp8_linear_and_quantisers_match_oracle():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 512, generator=g).to(BF)
    w, ws = _w(g, 384, 512)
    assert torch.equal(R.fp8_linear(x, w, ws), O.fp8_linear(x, w, ws))
    q1, s1 = R.group_quant(x)
    q2, s2 = O.per_token_group_quant_fp8(x, 128)
    assert torch.equal(q1.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s1, s2)
    assert torch.equal(R.weight_dequant(w, ws), O.weight_dequant(w, ws))


def test_fused_experts_matches_oracle():
    g = torch.Generator().manual_seed(1)
    T, K, F, E, topk = 6, 256, 128, 8, 3
    x = torch.randn(T, K, generator=g).to(BF)
    w1 = torch.stack([_w(g, 2 * F, K)[0] for _ in range(E)])
    g = torch.Generator().manual_seed(2)
    pairs1 = [_w(g, 2 * F, K) for _ in range(E)]
    pairs2 = [_w(g, K, F) for _ in range(E)]
    w1, w1s = torch.stack([p[0] for p in pairs1]), torch.stack([p[1] for p in pairs1])
    w2, w2s = torch.stack([p[0] for p in pairs2]), torch.stack([p[1] for p in pairs2])
    ids = torch.stack([torch.randperm(E, generator=g)[:topk] for _ in range(T)])
    tw = torch.rand(T, topk, generator=g).to(BF)
    a = R.fused_experts(x, w1, w2, tw, ids, w1s, w2s, "fp8_w8a8")
    b = O.fused_experts(x, w1, w2, tw, ids, w1s, w2s, mode="fp8_w8a8")
    assert torch.equal(a, b)
    wb1, wb2 = O.weight_dequant(w1, w1s), O.weight_dequant(w2, w2s)
    assert torch.equal(R.fused_experts(x, wb1, wb2, tw, ids), O.fused_experts(x, wb1, wb2, tw, ids))


def test_gate_matches_oracle():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(7, 256, generator=g).to(BF)
    w = (torch.randn(32, 256, generator=g) * 0.05).to(BF)
    b = torch.randn(32, generator=g) * 0.01
    for a, o in zip(R.moe_gate(x, w, b, 4, 4, 2, "sigmoid", 2.5), O.moe_gate(x, w, b, 4, 4, 2, "sigmoid", 2.5)):
        assert torch.equal(a, o)


def test_mla_and_gqa_attention_match_oracle():
    g = torch.Generator().manual_seed(4)
    B, H, C, Rr, page, nblk = 3, 4, 512, 64, 64, 12
    cache = torch.randn(nblk, page, C + Rr, generator=g).to(BF)
    table = torch.randperm(nblk, generator=g).to(torch.int32).view(B, 4)
    lens = torch.tensor([100, 63, 128], dtype=torch.int32)
    qn, qp = torch.randn(B, H, C, generator=g).to(BF), torch.randn(B, H, Rr, generator=g).to(BF)
    kv = torch.randn(B, C + Rr, generator=g).to(BF)
    c1, c2 = cache.clone(), cache.clone()
    a = R.mla_attn_with_kvcache(qn, qp, c1, kv, lens, table, 0.135)
    b = O.mla_attn_with_kvcache(qn, qp, c2, kv.view(B, 1, 1, -1), lens, table, 0.135)
    assert torch.equal(c1.view(torch.int16), c2.view(torch.int16))
    assert (a.float() - b.float()).abs().max() <= 1e-2 * b.float().abs().max()
    Hq, Hkv, D, page = 8, 2, 64, 16
    kc = torch.randn(24, page, Hkv, D, generator=g).to(BF)
    vc = torch.randn(24, page, Hkv, D, generator=g).to(BF)
    table = torch.randperm(24, generator=g).to(torch.int32).view(B, 8)
    q = torch.randn(B, 1, Hq, D, generator=g).to(BF)
    kn, vn = torch.randn(B, 1, Hkv, D, generator=g).to(BF), torch.randn(B, 1, Hkv, D, generator=g).to(BF)
    lens = torch.tensor([100, 15, 16], dtype=torch.int32)
    k1, v1, k2, v2 = kc.clone(), vc.clone(), kc.clone(), vc.clone()
    a = R.gqa_paged_decode(q, k1, v1, kn, vn, lens, table)
    b = O.gqa_paged_decode(q, k2, v2, kn, vn, lens, table)
    assert torch.equal(k1.view(torch.int16), k2.view(torch.int16)) and torch.equal(v1.view(torch.int16), v2.view(torch.int16))
    assert (a.float() - b.float()).abs().max() <= 1e-2 * b.float().abs().max()


def test_rotary_half_and_mixtral_block_match_oracle(golden):
    g = torch.Generator().manual_seed(5)
    q, k = torch.randn(3, 4, 64, generator=g).to(BF), torch.randn(3, 2, 64, generator=g).to(BF)
    cos, sin = torch.randn(3, 32, generator=g).to(BF), torch.randn(3, 32, generator=g).to(BF)
    for a, b in zip(R.rotary_half(q, k, cos, sin), O.rotary_half(q, k, cos, sin)):
        assert torch.equal(a, b)
    G = golden("block_mixtral_moe")
    E, topk = (int(v) for v in G.np("cfg"))
    y, _, _ = R.mixtral_moe_block(G.t("x", BF), G.t("gate_w", BF), G.t("w1", BF), G.t("w2", BF), topk)
    ref = G.t("y", BF).float()
    assert (y.float() - ref).abs().max() <= 2 * 2.0 ** -8 * ref.abs().max()      # the reference block's own output


def _llama_case(g, B=3, Hq=8, Hkv=2, D=64, F=256, n_layers=2, page=16, nblk=24):
    dim = Hq * D

    def r(*shape, scale=0.02):
        return (torch.randn(*shape, generator=g) * scale).to(BF)

    layers = [dict(attn_norm=(0.5 + torch.rand(dim, generator=g)).to(BF), ffn_norm=(0.5 + torch.rand(dim, generator=g)).to(BF),
                   wqkv=r((Hq + 2 * Hkv) * D, dim), wo=r(dim, Hq * D), w13=r(2 * F, dim), w2=r(dim, F))
              for _ in range(n_layers)]
    kc = [torch.randn(nblk, page, Hkv, D, generator=g).to(BF) for _ in range(n_layers)]
    vc = [torch.randn(nblk, page, Hkv, D, generator=g).to(BF) for _ in range(n_layers)]
    table = torch.randperm(nblk, generator=g).to(torch.int32).view(B, nblk // B)
    lens = torch.tensor([0, 15, 100], dtype=torch.int32)[:B]
    ang = torch.rand(B, D // 2, generator=g) * 6
    return layers, kc, vc, table, lens, ang.cos(), ang.sin()


def test_llama_layers_match_oracle_step():
    """R.llama_decode_step (a loop over R.llama_layer) against the oracle's step, with distinct norm weights; the layer
    in fp64 stays within bf16 rounding of the fp32 one."""
    g = torch.Generator().manual_seed(6)
    Hq, Hkv, D, F = 8, 2, 64, 256
    layers, kc, vc, table, lens, cos, sin = _llama_case(g, Hq=Hq, Hkv=Hkv, D=D, F=F)
    dim, vocab = Hq * D, 96
    embed, head = (torch.randn(vocab, dim, generator=g) * 0.02).to(BF), (torch.randn(vocab, dim, generator=g) * 0.02).to(BF)
    norm = (0.5 + torch.rand(dim, generator=g)).to(BF)
    tokens = torch.tensor([3, 50, 95])
    W = O.LlamaWeights(dim, len(layers), Hq, Hkv, F, vocab)
    W.embed, W.norm, W.output = embed, norm, head
    for ow, lw in zip(W.layers, layers):
        ow.update(attn_norm=lw["attn_norm"], ffn_norm=lw["ffn_norm"], wo=lw["wo"], w2=lw["w2"], w1=lw["w13"][:F],
                  w3=lw["w13"][F:], wq=lw["wqkv"][: Hq * D], wk=lw["wqkv"][Hq * D: (Hq + Hkv) * D],
                  wv=lw["wqkv"][(Hq + Hkv) * D:])
    k1, v1 = [c.clone() for c in kc], [c.clone() for c in vc]
    k2, v2 = [c.clone() for c in kc], [c.clone() for c in vc]
    a = R.llama_decode_step(layers, embed, norm, head, tokens, k1, v1, lens, table, cos, sin, Hq, Hkv, 1e-5)
    b = O.llama_decode_step(W, tokens, k2, v2, lens, table, cos, sin, eps=1e-5)
    for x, y in zip(k1 + v1, k2 + v2):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16))
    assert (a - b).abs().max() <= 1e-2 * b.abs().max()
    h = embed[tokens]
    h32 = R.llama_layer(layers[0], h, kc[0].clone(), vc[0].clone(), lens, table, cos, sin, Hq, Hkv, 1e-5)
    h64 = R.llama_layer(layers[0], h, kc[0].clone(), vc[0].clone(), lens, table, cos, sin, Hq, Hkv, 1e-5,
                        compute_dtype=torch.float64)
    assert h64.dtype == BF and ((h64.float() - h32.float()).abs() <= 2.0 ** -7 * h32.float().abs() + 1e-6).all()


def test_mixtral_layer_matches_oracle_pieces():
    """R.mixtral_layer against the oracle's operators composed in the engine's order (hf-llama attention, then the
    renormalised top-2 sparse-MoE block), fp32 and fp64 compute."""
    g = torch.Generator().manual_seed(7)
    Hq, Hkv, D, F, E, topk = 4, 2, 64, 128, 4, 2
    layers, kc, vc, table, lens, _, _ = _llama_case(g, Hq=Hq, Hkv=Hkv, D=D, F=F, n_layers=1)
    dim, eps = Hq * D, 1e-5
    lw = dict(layers[0], gate_w=(torch.randn(E, dim, generator=g) * 0.05).to(BF),
              w1=(torch.randn(E, 2 * F, dim, generator=g) * 0.02).to(BF), w2=(torch.randn(E, dim, F, generator=g) * 0.02).to(BF))
    ang = torch.rand(3, D // 2, generator=g) * 6
    cos, sin = ang.cos().to(BF), ang.sin().to(BF)
    h = (torch.randn(3, dim, generator=g) * 0.3).to(BF)
    k1, v1, k2, v2 = kc[0].clone(), vc[0].clone(), kc[0].clone(), vc[0].clone()
    routes = []
    got = R.mixtral_layer(lw, h, k1, v1, lens, table, cos, sin, Hq, Hkv, topk, eps, route_out=routes)
    xn = O.rms_norm(h, lw["attn_norm"], eps)
    qkv = O.linear(xn, lw["wqkv"])
    q, k, v = qkv.split([Hq * D, Hkv * D, Hkv * D], dim=-1)
    q, k = O.rotary_half(q.reshape(3, Hq, D), k.reshape(3, Hkv, D), cos, sin)
    o = O.gqa_paged_decode(q.view(3, 1, Hq, D), k2, v2, k.view(3, 1, Hkv, D), v.reshape(3, 1, Hkv, D), lens, table)
    h2 = O.linear(o.reshape(3, Hq * D), lw["wo"]) + h
    xn = O.rms_norm(h2, lw["ffn_norm"], eps)
    probs = torch.softmax(O.linear(xn, lw["gate_w"]), dim=-1, dtype=torch.float32)
    w, idx = torch.topk(probs, topk, dim=-1)
    want = h2 + O.fused_experts(xn, lw["w1"], lw["w2"], (w / w.sum(dim=-1, keepdim=True)).to(BF), idx)
    assert torch.equal(k1.view(torch.int16), k2.view(torch.int16)) and torch.equal(v1.view(torch.int16), v2.view(torch.int16))
    assert torch.equal(routes[0][0], idx)
    assert (got.float() - want.float()).abs().max() <= 2.0 ** -7 * want.float().abs().max()
    got64 = R.mixtral_layer(lw, h, kc[0].clone(), vc[0].clone(), lens, table, cos, sin, Hq, Hkv, topk, eps,
                            compute_dtype=torch.float64)
    assert (got64.float() - want.float()).abs().max() <= 2.0 ** -7 * want.float().abs().max()
