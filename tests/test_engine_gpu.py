"""End-to-end decode steps of the two engines against the CPU oracle (tiny dims, same weights)."""
import pytest
import torch

from conftest import cos_diff, max_rel
from oracle import chitu_oracle as O

pytestmark = pytest.mark.gpu


def test_llama_engine_step_and_graph_vs_oracle():
    import __graft_entry__ as ge
    ge.smoke()


def test_llama_engine_cuda_graph_two_steps():
    from chitu_b200.engine import LlamaConfig, LlamaDecodeEngine
    cfg = LlamaConfig(dim=512, n_layers=2, n_heads=8, n_kv_heads=2, vocab_size=1024, multiple_of=256, ffn_dim_multiplier=None)
    eng = LlamaDecodeEngine(cfg, max_reqs=4, max_seq_len=1024, device="cuda:0")
    eng.set_synthetic_context(200)
    toks = torch.tensor([1, 2, 3, 4], dtype=torch.int64).pin_memory()
    a = eng.decode(toks)
    lens_after = eng.seq_lens.clone()
    eng.seq_lens.fill_(200)                 # same cache contents (the append rewrote identical rows)
    eng.capture()
    b = eng.decode(toks)                    # graph replay must give the same tokens and advance seq_lens
    assert torch.equal(a, b) and torch.equal(eng.seq_lens, lens_after)
    assert eng.launches_per_step > 0


def _deepseek_case(n_layers, n_dense, B=3, S=150):
    from chitu_b200.engine_deepseek import DeepSeekConfig, DeepSeekDecodeEngine
    cfg = DeepSeekConfig(vocab_size=1024, dim=512, inter_dim=1024, moe_inter_dim=256, n_layers=n_layers,
                         n_dense_layers=n_dense, n_heads=4, n_routed_experts=16, n_activated_experts=4,
                         n_expert_groups=4, n_limited_groups=2, q_lora_rank=256)
    eng = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=512, device="cuda:0", tp_size=1)
    eng.set_synthetic_context(S)
    eng.seq_lens.copy_(torch.tensor([S, 63, 128], dtype=torch.int32))
    tokens = torch.tensor([5, 17, 900], dtype=torch.int64)
    layers = [{k: v.cpu() for k, v in L.items()} for L in eng.layers]
    kc = [eng.kv_cache[l].cpu() for l in range(cfg.n_layers)]
    kv0_before = kc[0].clone()
    lens = eng.seq_lens.cpu()
    cos, sin = eng.cos_table[lens.long()].cpu(), eng.sin_table[lens.long()].cpu()
    routes = []
    ref = O.deepseek_decode_step(layers, eng.embed.cpu(), eng.norm.cpu(), eng.head.cpu(), cfg, tokens, kc, lens,
                                 eng.block_table.cpu(), cos, sin, eng.H, routes_out=routes)
    eng.decode(tokens.pin_memory())
    torch.cuda.synchronize()
    got = eng.logits.float().cpu()
    same_routes = all(torch.equal(eng.gate_i_all[li][:, :cfg.n_activated_experts].cpu().sort(dim=-1)[0], r.sort(dim=-1)[0]) for li, r in routes)
    O.check_kv_append(eng.kv_cache[0].cpu(), kv0_before, kc[0], eng.block_table.cpu(), lens, 64)
    return cos_diff(got, ref), max_rel(got, ref), same_routes


def test_deepseek_engine_step_vs_oracle():
    """Whole-step check.  KV-page indexing is bit exact.  Logits: every FP8 linear re-quantises its input,
    so a 1-ulp bf16 difference upstream flips a few e4m3 roundings (6-12 % each) and two CORRECT
    implementations differ by ~1 % per GEMM (cos_diff ~1e-3 after a layer) — the tight, teacher-forced
    comparison is test_deepseek_engine_wiring_stage_by_stage; here only gross errors are caught."""
    for n_layers, n_dense in [(1, 1), (2, 1), (3, 1)]:
        cd, mr, same_routes = _deepseek_case(n_layers, n_dense)
        print(f"deepseek engine vs oracle L={n_layers}: cos_diff {cd:.3e} max_rel {mr:.3e} same_routes {same_routes}")
        if same_routes:
            assert cd < 1e-2, (n_layers, cd)
            assert mr < 0.15, (n_layers, mr)


def test_deepseek_engine_wiring_stage_by_stage():
    """Teacher-forced check of every stage of the DeepSeek layer: each engine intermediate is compared with
    the oracle operator applied to the ENGINE's own inputs of that stage, so fp8 re-quantisation noise cannot
    accumulate and every comparison is tight (wiring, strides, views, residuals)."""
    from chitu_b200.engine_deepseek import DeepSeekConfig, DeepSeekDecodeEngine
    cfg = DeepSeekConfig(vocab_size=1024, dim=512, inter_dim=1024, moe_inter_dim=256, n_layers=2, n_dense_layers=1,
                         n_heads=4, n_routed_experts=16, n_activated_experts=4, n_expert_groups=4, n_limited_groups=2,
                         q_lora_rank=256)
    B, S = 3, 150
    eng = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=512, device="cuda:0", tp_size=1)
    eng.set_synthetic_context(S)
    eng.seq_lens.copy_(torch.tensor([S, 63, 128], dtype=torch.int32))
    eng.trace = []
    eng.decode(torch.tensor([5, 17, 900], dtype=torch.int64).pin_memory())
    torch.cuda.synchronize()
    bf, eps = torch.bfloat16, cfg.norm_eps
    H, C, R, dn, dv = eng.H, eng.C, eng.R, cfg.qk_nope_head_dim, cfg.v_head_dim
    table = eng.block_table.cpu()

    def close(name, got, ref, tol=8e-3):
        mr = max_rel(got.float().cpu(), ref.float())
        assert mr < tol, (name, mr)

    for li, tr in enumerate(eng.trace):
        t = {k: v.cpu() for k, v in tr.items()}
        L = {k: v.cpu() for k, v in eng.layers[li].items()}
        close("xn_attn", t["xn_attn"], O.rms_norm(t["h_in"], L["attn_norm"], eps, bf))
        close("qkv_a", t["qkv_a"], O.fp8_linear(t["xn_attn"], L["wqkv_a"], L["wqkv_a_s"]))
        q_a, kv, k_pe = torch.split(t["qkv_a"], [cfg.q_lora_rank, C, R], dim=-1)
        close("qa_n", t["qa_n"], O.rms_norm(q_a.contiguous(), L["q_norm"], eps, bf))
        close("q", t["q"].view(B, -1), O.fp8_linear(t["qa_n"], L["wq_b"], L["wq_b_s"]))
        q = t["q"].view(B, H, dn + R)
        lens = t["lens"]
        cos, sin = eng.cos_table[lens.long().to("cuda")].cpu(), eng.sin_table[lens.long().to("cuda")].cpu()
        q_pe_r, k_pe_r = O.rotary_interleaved(q[..., dn:], k_pe, cos, sin)
        assert torch.equal(t["q_pe"], q_pe_r)
        assert torch.equal(t["new_kv"][:, C:], k_pe_r)
        close("kv_norm", t["new_kv"][:, :C], O.rms_norm(kv.contiguous(), L["kv_norm"], eps, bf))
        wkv = O.weight_dequant(L["wkv_b"], L["wkv_b_s"]).view(H, dn + dv, C)
        close("q_abs", t["q_abs"], torch.einsum("shd,hdc->shc", q[..., :dn].float(), wkv[:, :dn].float()))
        cache = t["cache_before"].clone()
        ref_lat = O.mla_attn_with_kvcache(t["q_abs"], t["q_pe"], cache, t["new_kv"].view(B, 1, 1, -1), lens, table,
                                          cfg.softmax_scale)
        close("o_lat", t["o_lat"], ref_lat, 1e-2)
        assert torch.equal(eng.kv_cache[li].cpu().view(torch.int16), cache.view(torch.int16))     # append bit exact
        close("o", t["o"].view(B, H, dv), torch.einsum("bhc,hdc->bhd", t["o_lat"].float(), wkv[:, -dv:].float()))
        close("attn_out", t["attn_out"], O.fp8_linear(t["o"], L["wo"], L["wo_s"]))
        close("h_mid", t["h_mid"], t["attn_out"] + t["h_in"])
        close("xn_ffn", t["xn_ffn"], O.rms_norm(t["h_mid"], L["ffn_norm"], eps, bf))
        if "w13" in L:
            ff = O.fp8_linear(t["xn_ffn"], L["w13"], L["w13_s"])
            close("ff", t["ff"][:, : ff.shape[1]], ff)
            close("act", t["act"][:, : ff.shape[1] // 2], O.silu_and_mul(t["ff"][:, : ff.shape[1]].contiguous()))
            close("y", t["y"], O.fp8_linear(t["act"][:, : ff.shape[1] // 2].contiguous(), L["w2"], L["w2_s"]))
        else:
            w, idx, scores = O.moe_gate(t["xn_ffn"], L["gate_w"], L["gate_b"], cfg.n_activated_experts, cfg.n_expert_groups,
                                        cfg.n_limited_groups, cfg.score_func, cfg.route_scale)
            k = cfg.n_activated_experts
            gi, gw = eng.gate_i_all[li][:, :k].cpu(), eng.gate_w_all[li][:, :k].cpu()
            assert torch.equal(gi, idx)                                           # routing bit exact
            close("gate_w", gw, w)
            assert bool((eng.gate_i_all[li][:, k] == cfg.n_routed_experts).all()) and bool((eng.gate_w_all[li][:, k] == 1).all())
            sh = O.fp8_linear(O.silu_and_mul(O.fp8_linear(t["xn_ffn"], L["ws13"], L["ws13_s"])), L["ws2"], L["ws2_s"])
            routed = O.fused_experts(t["xn_ffn"], L["we1"][:-1], L["we2"][:-1], gw, gi, L["we1_s"][:-1], L["we2_s"][:-1],
                                     mode="fp8_w8a8")
            close("y", t["y"], sh.float() + routed.float(), 2e-2)   # shared expert rides as expert #E in the grouped GEMM
        close("h_out", t["h_out"], t["y"] + t["h_mid"])
