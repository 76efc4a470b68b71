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
    comparison of every layer against fp64 is tests/test_engine_steps_gpu.py; here only gross errors are caught."""
    for n_layers, n_dense in [(1, 1), (2, 1), (3, 1)]:
        cd, mr, same_routes = _deepseek_case(n_layers, n_dense)
        print(f"deepseek engine vs oracle L={n_layers}: cos_diff {cd:.3e} max_rel {mr:.3e} same_routes {same_routes}")
        if same_routes:
            assert cd < 1e-2, (n_layers, cd)
            assert mr < 0.15, (n_layers, mr)
