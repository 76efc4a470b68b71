"""Generate tests/golden/*.npz by running the REAL reference (a thu-pacman/chitu checkout at $CHITU_REFERENCE).

Needs that checkout (CPU only):
    python oracle/gen_golden.py
The reference's Triton kernels run under TRITON_INTERPRET=1 on CPU (SURVEY.md §8c / Appendix A);
its torch code runs as is.  bf16 tensors are stored as uint16 bit patterns, fp8 as uint8.
Caveat (SURVEY §8c): bf16 `tl.dot` is broken in the Triton 3.6 CPU interpreter, so kernels that
reach tl.dot are fed fp32 tensors holding bf16-rounded values.
"""
import os
import sys
import types

os.environ["TRITON_INTERPRET"] = "1"
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
os.environ.setdefault("MASTER_PORT", "29577")
REF = os.environ.get("CHITU_REFERENCE", "reference")   # checkout of thu-pacman/chitu
sys.path.insert(0, REF)

import numpy as np
import torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from oracle.golden_inputs import compact  # noqa: E402

sys.modules["chitu_backend"] = types.ModuleType("chitu_backend")
for name in ("w8a8gemm", "w8a8gemv"):
    sys.modules[name] = types.ModuleType(name)
import chitu.device_type as D  # noqa: E402

D._device_name = "cpu"
torch.cuda.synchronize = lambda *a, **k: None

from chitu import fused_moe, ops  # noqa: E402
from chitu import triton_decode_attention as tda  # noqa: E402
from chitu import triton_kernels as tk  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
os.makedirs(OUT, exist_ok=True)


def bits(t: torch.Tensor) -> np.ndarray:
    if t.dtype == torch.bfloat16:
        return t.contiguous().view(torch.int16).numpy().view(np.uint16)
    if t.dtype == torch.float8_e4m3fn:
        return t.contiguous().view(torch.uint8).numpy()
    return t.contiguous().numpy()


def save(name, **arrs):
    """Writes the stored form (oracle/golden_inputs.compact): large seeded inputs as SHA-256, near-copies as deltas."""
    full = {k: (bits(v) if torch.is_tensor(v) else np.asarray(v)) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **compact(name, full))
    print("wrote", name, {k: tuple(v.shape) for k, v in full.items()})


def bf16r(t):
    return t.bfloat16().float()


def gen_moe_align():
    g = torch.Generator().manual_seed(11)
    cases = {}
    kat = torch.tensor([[2, 3, 4], [1, 2, 4], [1, 3, 4], [1, 2, 3]], dtype=torch.int32)
    for tag, ids, blk, E in [
        ("kat", kat, 4, 5),
        ("e256", torch.randint(0, 256, (1000,), generator=g, dtype=torch.int32), 64, 256),
        ("e64", torch.randint(0, 64, (37, 6), generator=g, dtype=torch.int32), 16, 64),
        ("skew", (torch.randint(0, 8, (300,), generator=g, dtype=torch.int32) ** 2) % 32, 32, 32),
    ]:
        s, e, n = fused_moe.moe_align_block_size_native(ids, blk, E)
        cases[f"{tag}_ids"] = ids
        cases[f"{tag}_cfg"] = np.array([blk, E])
        cases[f"{tag}_sorted"] = s
        cases[f"{tag}_experts"] = e
        cases[f"{tag}_npp"] = n
    save("moe_align", **cases)


def gen_append():
    g = torch.Generator().manual_seed(12)
    B, pages_per, page, dim = 5, 4, 64, 576
    nblk = B * pages_per
    cache = torch.randn(nblk, page, dim, generator=g).bfloat16()
    table = torch.randperm(nblk, generator=g).to(torch.int32).view(B, pages_per).contiguous()
    lens = torch.tensor([0, 63, 64, 130, 255], dtype=torch.int32)
    kv = torch.randn(B, dim, generator=g).bfloat16()
    before = cache.clone()
    ops.append_to_paged_kv_cache(cache, table, kv, lens)
    save("append_kv", cache_before=before, cache_after=cache, table=table, lens=lens, kv=kv)
    # page_size 256 (GQA layout [nblk, page, heads, dim]): exposes the literal-64 arithmetic
    cache2 = torch.randn(6, 256, 2, 8, generator=g).half()
    table2 = torch.tensor([[3, 1, 0], [5, 2, 4]], dtype=torch.int32)
    lens2 = torch.tensor([70, 130], dtype=torch.int32)
    kv2 = torch.randn(2, 2, 8, generator=g).half()
    before2 = cache2.clone()
    ops.append_to_paged_kv_cache(cache2, table2, kv2, lens2)
    save("append_kv_p256", cache_before=before2, cache_after=cache2, table=table2, lens=lens2, kv=kv2)


def gen_rotary():
    g = torch.Generator().manual_seed(13)
    bs, h, d = 6, 5, 64
    q = torch.randn(bs, h, d, generator=g)
    k = torch.randn(bs, d, generator=g)
    cos = torch.randn(bs, d // 2, generator=g) * 2
    sin = torch.randn(bs, d // 2, generator=g)
    oq, ok = ops.apply_rotary_pos_emb_triton(q, k, cos, sin, rotary_type="llama")
    tq, tk_ = ops.apply_rotary_pos_emb_torch(q, k, cos, sin, rotary_type="llama")
    qb, kb = q.bfloat16(), k.bfloat16()
    oqb, okb = ops.apply_rotary_pos_emb_triton(qb, kb, cos, sin, rotary_type="llama")
    save("rotary_llama", q=q, k=k, cos=cos, sin=sin, out_q=oq, out_k=ok, torch_q=tq, torch_k=tk_, q_bf16=qb,
         k_bf16=kb, out_q_bf16=oqb, out_k_bf16=okb)
    # hf-llama: [bs, heads, 128]
    q2 = torch.randn(3, 4, 128, generator=g)
    k2 = torch.randn(3, 2, 128, generator=g)
    cos2 = torch.randn(3, 64, generator=g)
    sin2 = torch.randn(3, 64, generator=g)
    oq2, ok2 = ops.apply_rotary_pos_emb_triton(q2, k2, cos2, sin2, rotary_type="hf-llama")
    tq2, tk2 = ops.apply_rotary_pos_emb_torch(q2, k2, cos2, sin2, rotary_type="hf-llama")
    save("rotary_hf", q=q2, k=k2, cos=cos2, sin=sin2, out_q=oq2, out_k=ok2, torch_q=tq2, torch_k=tk2)


def gen_quant():
    g = torch.Generator().manual_seed(14)
    x = (torch.randn(7, 512, generator=g) * 3).bfloat16()
    x[2, 128:256] *= 50.0
    y, s = ops.act_quant_deepseek_v3(x)
    save("act_quant", x=x, y=y, s=s)
    x2 = (torch.randn(5, 256, generator=g) * 2).bfloat16()
    x2[1, :128] = 0  # all-zero group exercises eps
    q, qs = fused_moe.per_token_group_quant_fp8(x2, 128)
    save("group_quant", x=x2, q=q, s=qs)


def make_fp8_weight(N, K, g, scale=0.05):
    w = torch.randn(N, K, generator=g) * scale
    nb, kb = (N + 127) // 128, (K + 127) // 128
    wp = torch.zeros(nb * 128, kb * 128)
    wp[:N, :K] = w
    blocks = wp.view(nb, 128, kb, 128)
    s = blocks.abs().amax(dim=(1, 3)) / 448.0
    q = (blocks / s[:, None, :, None]).view(nb * 128, kb * 128)[:N, :K].to(torch.float8_e4m3fn)
    return q.contiguous(), s.float().contiguous()


def gen_dequant_and_gemm():
    g = torch.Generator().manual_seed(15)
    torch.set_default_dtype(torch.bfloat16)
    wq, ws = make_fp8_weight(256, 384, g)
    deq = ops.weight_dequant_deepseek_v3(wq, ws)
    deq_soft = ops.weight_dequant_soft_fp8_deepseek_v3(wq, ws)
    wq3 = torch.stack([wq, make_fp8_weight(256, 384, g)[0]])
    ws3 = torch.stack([ws, ws * 1.5])
    deq3 = ops.weight_dequant_deepseek_v3(wq3, ws3)
    save("weight_dequant", w=wq, s=ws, deq=deq, deq_soft=deq_soft, w3=wq3, s3=ws3, deq3=deq3)

    # fp8 block GEMM through the reference kernel body (autotune wrapper needs a GPU: call .fn)
    M, N, K = 5, 256, 512
    a = (torch.randn(M, K, generator=g) * 2).bfloat16()
    aq, a_s = ops.act_quant_deepseek_v3(a)
    bq, b_s = make_fp8_weight(N, K, g)
    c = torch.empty(M, N, dtype=torch.bfloat16)
    BM, BN, BK = 16, 64, 128
    grid = ((M + BM - 1) // BM, (N + BN - 1) // BN)
    tk.fp8_gemm_deepseek_v3_kernel.fn[grid](aq, bq, c, a_s, b_s, M, N, K, group_n=128, group_k=128,
                                            BLOCK_SIZE_M=BM, BLOCK_SIZE_N=BN, BLOCK_SIZE_K=BK)
    # soft-fp8 linear: the reference's own non-fused path (model_deepseek_v3.py:95-99)
    wsoft = ops.weight_dequant_soft_fp8_deepseek_v3(bq, b_s)
    c_soft = torch.nn.functional.linear(a, wsoft)
    save("fp8_gemm", a=a, aq=aq, a_s=a_s, bq=bq, b_s=b_s, c=c, c_soft=c_soft)
    torch.set_default_dtype(torch.float32)


def gen_mla():
    g = torch.Generator().manual_seed(16)
    B, H, C, R, page = 3, 16, 512, 64, 64
    lens = torch.tensor([1, 77, 130], dtype=torch.int32)
    pages_per = 3
    nblk = B * pages_per
    cache = bf16r(torch.randn(nblk, page, C + R, generator=g))
    table = torch.randperm(nblk, generator=g).to(torch.int32).view(B, pages_per).contiguous()
    q_nope = bf16r(torch.randn(B, H, C, generator=g))
    q_pe = bf16r(torch.randn(B, H, R, generator=g))
    scale = 0.1352337788
    splits = 4
    logits = torch.zeros(B, H, splits, C + 1)
    o = torch.zeros(B, H, C)
    kv_c, k_pe = cache[..., :C], cache[..., C:]
    grid = (B, 1, splits)
    tda._mla_attn_kernel.fn[grid](q_nope, q_pe, kv_c, k_pe, table, lens, logits, scale, q_nope.stride(0),
                                  q_nope.stride(1), q_pe.stride(0), q_pe.stride(1), kv_c.stride(-2),
                                  k_pe.stride(-2), table.stride(0), logits.stride(0), logits.stride(1),
                                  logits.stride(2), BLOCK_H=16, BLOCK_N=64, NUM_KV_SPLITS=splits, PAGE_SIZE=page,
                                  HEAD_DIM_CKV=C, HEAD_DIM_KPE=R)
    tda._mla_softmax_reducev(logits, o, lens, splits)
    save("mla_decode", q_nope=q_nope.bfloat16(), q_pe=q_pe.bfloat16(), cache=cache.bfloat16(), table=table, lens=lens,
         scale=np.float32(scale), out=o)


def gen_fused_experts():
    g = torch.Generator().manual_seed(17)
    T, K1, N1, E, topk = 3, 256, 256, 8, 2
    x = bf16r(torch.randn(T, K1, generator=g))
    w1 = bf16r(torch.randn(E, N1, K1, generator=g) * 0.05)
    w2 = bf16r(torch.randn(E, K1, N1 // 2, generator=g) * 0.05)
    ids = torch.stack([torch.randperm(E, generator=g)[:topk] for _ in range(T)]).to(torch.int32)
    tw = bf16r(torch.rand(T, topk, generator=g))
    out = fused_moe.fused_experts_impl(x.clone(), w1, w2, tw, ids, inplace=False)
    # fp8 block-quantised experts
    w1q, w1s, w2q, w2s = [], [], [], []
    for e in range(E):
        q, s = make_fp8_weight(N1, K1, g)
        w1q.append(q), w1s.append(s)
        q, s = make_fp8_weight(K1, N1 // 2, g)
        w2q.append(q), w2s.append(s)
    w1q, w1s, w2q, w2s = torch.stack(w1q), torch.stack(w1s), torch.stack(w2q), torch.stack(w2s)
    out_fp8 = fused_moe.fused_experts_impl(x.clone(), w1q, w2q, tw, ids, inplace=False, use_fp8_w8a8=True,
                                           w1_scale=w1s, w2_scale=w2s, block_shape=[128, 128])
    save("fused_experts", x=x.bfloat16(), w1=w1.bfloat16(), w2=w2.bfloat16(), ids=ids, tw=tw.bfloat16(), out=out,
         w1q=w1q, w1s=w1s, w2q=w2q, w2s=w2s, out_fp8=out_fp8)


def gen_gate():
    from types import SimpleNamespace
    import importlib
    g = torch.Generator().manual_seed(18)
    import chitu.global_vars as gv
    args = SimpleNamespace(infer=SimpleNamespace(soft_fp8=False, tp_size=1, pp_size=1, op_impl="torch"),
                           models=SimpleNamespace())
    try:
        gv.set_global_variables(args)
    except Exception as e:  # pragma: no cover
        print("set_global_variables:", e)
    if not torch.distributed.is_initialized():
        torch.distributed.init_process_group("gloo", rank=0, world_size=1)
    mdl = importlib.import_module("chitu.models.model_deepseek_v3")
    margs = SimpleNamespace(dim=7168, n_activated_experts=8, n_expert_groups=8, n_limited_groups=4,
                            score_func="sigmoid", route_scale=2.5, n_routed_experts=256)
    gate = mdl.GateDeepSeekV3(margs)
    T = 6
    with torch.no_grad():
        gate.weight.copy_(torch.randn(256, 7168, generator=g) * 0.02)
        gate.bias.copy_(torch.randn(256, generator=g) * 0.01)
    gate.weight.data = gate.weight.data.bfloat16()
    x = torch.randn(T, 7168, generator=g).bfloat16()
    with torch.no_grad():
        w, idx = gate(x)          # bias fp32 (keep_dtype_in_checkpoint) -> fp32 score path
    save("gate_sigmoid_f32bias", x=x, weight=gate.weight.data, bias=gate.bias.data.float(), w=w, idx=idx)
    # small softmax / no-bias / grouped-amax variant (dim != 7168 -> bias None)
    margs2 = SimpleNamespace(dim=512, n_activated_experts=6, n_expert_groups=4, n_limited_groups=2,
                             score_func="softmax", route_scale=1.0, n_routed_experts=64)
    gate2 = mdl.GateDeepSeekV3(margs2)
    with torch.no_grad():
        gate2.weight.copy_(torch.randn(64, 512, generator=g) * 0.1)
    gate2.weight.data = gate2.weight.data.bfloat16()
    x2 = torch.randn(5, 512, generator=g).bfloat16()
    with torch.no_grad():
        w2, idx2 = gate2(x2)
    save("gate_softmax", x=x2, weight=gate2.weight.data, w=w2, idx=idx2)


def gen_w8a8_and_norm():
    g = torch.Generator().manual_seed(19)
    from chitu.quantize import w8a8 as rw
    act = (torch.randn(4, 1, 512, generator=g) * 3).half()
    q, s = rw.quant_act(act.clone())
    w = (torch.randn(96, 512, generator=g) * 0.1).half()
    wq, ws = rw.quant_weight(w.clone())
    save("w8a8_quant", act=act, q=q, s=s, w=w, wq=wq, ws=ws)
    from chitu.models.model import RMSNorm
    n = RMSNorm(384, eps=1e-5)
    with torch.no_grad():
        n.weight.copy_(torch.rand(384, generator=g) + 0.5)
    x = (torch.randn(5, 384, generator=g) * 2).bfloat16()
    n.weight.data = n.weight.data.bfloat16()
    with torch.no_grad():
        y32 = n(x)                                   # LLaMA: compute_dtype fp32
        y16 = n(x, compute_dtype=torch.bfloat16)     # DeepSeek: compute_dtype = x.dtype
    act2 = fused_moe.SiluAndMul()(x)
    save("rmsnorm_silu", x=x, w=n.weight.data, y_f32=y32, y_bf16=y16, silu_mul=act2)


def gen_ref_attn():
    g = torch.Generator().manual_seed(20)
    from chitu.attn_backend import RefAttnBackend
    be = RefAttnBackend()
    B, Hq, Hkv, Dh, S = 3, 8, 2, 128, 300
    k_cache = torch.randn(B, S, Hkv, Dh, generator=g).bfloat16()
    v_cache = torch.randn(B, S, Hkv, Dh, generator=g).bfloat16()
    lens = torch.tensor([0, 150, 299], dtype=torch.long)
    q = torch.randn(B, 1, Hq, Dh, generator=g).bfloat16()
    k = torch.randn(B, 1, Hkv, Dh, generator=g).bfloat16()
    v = torch.randn(B, 1, Hkv, Dh, generator=g).bfloat16()
    kc, vc = k_cache.clone(), v_cache.clone()
    out = be.attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=lens)
    save("ref_attn_gqa", q=q, k_cache=k_cache, v_cache=v_cache, k=k, v=v, lens=lens.to(torch.int32), out=out,
         k_cache_after=kc, v_cache_after=vc)


if __name__ == "__main__":
    gens = [gen_moe_align, gen_append, gen_rotary, gen_quant, gen_dequant_and_gemm, gen_mla, gen_fused_experts,
            gen_gate, gen_w8a8_and_norm, gen_ref_attn]
    only = sys.argv[1:]
    for fn in gens:
        if only and fn.__name__ not in only:
            continue
        print("==", fn.__name__)
        fn()
