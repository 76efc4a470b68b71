"""GPU parity: every CUDA operator (called through the Python mirror -> C ABI) against the CPU
oracle on seeded inputs, against the committed reference goldens, and at full size through
size-independent properties.  Bit-exact for integer / byte / index work; stated tolerances for
floating point (north_star: logits within 1e-2 relative; FlashMLA's cos_diff < 1e-5)."""
import numpy as np
import pytest
import torch

from conftest import Golden, cos_diff, max_rel
from oracle import chitu_oracle as O

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F8 = torch.float8_e4m3fn
DEV = "cuda:0"


def cu(t):
    return t.to(DEV)


# ---------------------------------------------------------------------------- append (bit exact)
def test_append_golden_and_oracle():
    from chitu_b200 import ops
    for name in ("append_kv", "append_kv_p256"):
        g = Golden(name)
        dt = BF if name == "append_kv" else torch.float16
        cache = g.t("cache_before", BF) if dt == BF else g.t("cache_before")
        after = g.t("cache_after", BF) if dt == BF else g.t("cache_after")
        kv = g.t("kv", BF) if dt == BF else g.t("kv")
        c = cu(cache.clone())
        ops.append_to_paged_kv_cache(c, cu(g.t("table")), cu(kv), cu(g.t("lens")))
        assert torch.equal(c.cpu().view(torch.int16), after.view(torch.int16)), name


def test_append_full_size_round_trip():
    from chitu_b200 import ops
    torch.manual_seed(3)
    B, pages_per, page, dim = 256, 65, 64, 576      # DeepSeek-R1 max_reqs=256, S=4096 (+1 page)
    nblk = B * pages_per
    cache = torch.zeros(nblk, page, dim, dtype=BF, device=DEV)
    table = torch.randperm(nblk, device=DEV).to(torch.int32).view(B, pages_per).contiguous()
    lens = torch.randint(0, 4096, (B,), device=DEV, dtype=torch.int32)
    kv = torch.randn(B, dim, device=DEV).to(BF)
    ops.append_to_paged_kv_cache(cache, table, kv, lens)
    pg = table[torch.arange(B, device=DEV), (lens // 64).long()].long()
    got = cache[pg, (lens % 64).long()]
    assert torch.equal(got, kv)                                  # appended rows read back exactly
    assert int((cache != 0).any(dim=-1).sum()) == B              # nothing else was touched


# ------------------------------------------------------------------------- moe_align (bit exact)
@pytest.mark.parametrize("tag", ["kat", "e256", "e64", "skew"])
def test_moe_align_golden(tag):
    from chitu_b200 import fused_moe
    g = Golden("moe_align")
    blk, E = g.np(f"{tag}_cfg").tolist()
    ids = cu(g.t(f"{tag}_ids"))
    s, e, npp = fused_moe.moe_align_block_size(ids, blk, E)
    assert np.array_equal(npp.cpu().numpy(), g.np(f"{tag}_npp"))
    assert np.array_equal(s.cpu().numpy(), g.np(f"{tag}_sorted"))          # raw array == Triton fallback
    nb = int(npp.item()) // blk
    assert np.array_equal(e.cpu().numpy()[:nb], g.np(f"{tag}_experts")[:nb])


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.int32, torch.int64])
def test_moe_align_oracle_dtypes_and_reference_property(dtype):
    from chitu_b200 import chitu_backend
    torch.manual_seed(5)
    E, blk = 256, 64
    ids = torch.randint(0, 256 if dtype != torch.uint8 else 255, (1000,), dtype=dtype)
    numel = ids.numel()
    max_padded = numel + E * (blk - 1)
    sorted_ids = torch.full((max_padded,), numel, dtype=torch.int32, device=DEV)
    expert_ids = torch.zeros(((max_padded + blk - 1) // blk,), dtype=torch.int32, device=DEV)
    npp = torch.empty((1,), dtype=torch.int32, device=DEV)
    cumsum = torch.zeros((E + 1,), dtype=torch.int32, device=DEV)
    chitu_backend.cuda_moe_align_block_size(cu(ids), E, blk, sorted_ids, expert_ids, npp, cumsum)
    s, e, n, c = O.moe_align_block_size(ids.numpy(), blk, E)
    assert np.array_equal(sorted_ids.cpu().numpy(), s)
    assert np.array_equal(cumsum.cpu().numpy(), c)
    assert np.array_equal(npp.cpu().numpy(), n)
    assert np.array_equal(expert_ids.cpu().numpy()[: int(n[0]) // blk], e[: int(n[0]) // blk])
    # the reference's own test property (test/pytest/test_moe_align.py:52-74): segment membership
    sid, cs = sorted_ids.cpu(), cumsum.cpu()
    for ex in torch.unique(ids).tolist():
        seg = set(sid[cs[ex]: cs[ex + 1]].tolist())
        assert set(torch.nonzero(ids == ex).flatten().tolist()) <= seg


def test_moe_align_edge_cases():
    from chitu_b200 import fused_moe
    # empty input, one expert, > 256 experts (the reference CUDA kernel caps at 256), ragged
    for ids, blk, E in [
        (torch.zeros((0,), dtype=torch.int32), 16, 8),
        (torch.zeros((33,), dtype=torch.int32), 16, 1),
        (torch.randint(0, 1024, (5000,), dtype=torch.int32), 8, 1024),
        (torch.full((257,), 7, dtype=torch.int32), 64, 16),
    ]:
        s, e, npp = fused_moe.moe_align_block_size(cu(ids), blk, E)
        so, eo, no, _ = O.moe_align_block_size(ids.numpy(), blk, E)
        assert np.array_equal(s.cpu().numpy(), so)
        assert np.array_equal(npp.cpu().numpy(), no)
        nb = int(no[0]) // blk
        assert np.array_equal(e.cpu().numpy()[:nb], eo[:nb])


# -------------------------------------------------------------------------------------- rotary
def test_rotary_reference_test_shape():
    # test/pytest/test_rotary_triton.py:16-32: B=16, H=64, D=256, rtol=atol=1e-5 (fp32)
    from chitu_b200 import ops
    torch.manual_seed(0)
    q = torch.randn(16, 64, 256)
    k = torch.randn(16, 256)
    cos = torch.randn(16, 128) * 2
    sin = torch.randn(16, 128)
    oq, ok = ops.apply_rotary_pos_emb(cu(q), cu(k), cu(cos), cu(sin), rotary_type="llama")
    rq, rk = O.rotary_interleaved(q, k, cos, sin)
    assert torch.allclose(oq.cpu(), rq, rtol=1e-5, atol=1e-5)
    assert torch.allclose(ok.cpu(), rk, rtol=1e-5, atol=1e-5)


def test_rotary_golden_and_bf16():
    from chitu_b200 import ops
    g = Golden("rotary_llama")
    oq, ok = ops.apply_rotary_pos_emb(cu(g.t("q")), cu(g.t("k")), cu(g.t("cos")), cu(g.t("sin")), rotary_type="llama")
    assert torch.allclose(oq.cpu(), g.t("out_q"), rtol=1e-5, atol=1e-5)
    assert torch.allclose(ok.cpu(), g.t("out_k"), rtol=1e-5, atol=1e-5)
    # bf16 io with strided q_pe view (as AttentionDeepSeekV3._run_linear passes it)
    torch.manual_seed(1)
    q = torch.randn(16, 16, 192).to(BF)
    q_pe = q[..., 128:]
    k_pe = torch.randn(16, 64).to(BF)
    cos, sin = torch.randn(16, 32), torch.randn(16, 32)
    oq, ok = ops.apply_rotary_pos_emb(cu(q)[..., 128:], cu(k_pe), cu(cos), cu(sin), rotary_type="llama")
    rq, rk = O.rotary_interleaved(q_pe, k_pe, cos, sin)
    assert torch.equal(oq.cpu(), rq) and torch.equal(ok.cpu(), rk)          # fp32 math, RNE: bit exact
    g = Golden("rotary_hf")
    oq, ok = ops.apply_rotary_pos_emb(cu(g.t("q")), cu(g.t("k")), cu(g.t("cos")), cu(g.t("sin")), rotary_type="hf-llama")
    assert torch.allclose(oq.cpu(), g.t("out_q"), rtol=1e-5, atol=1e-5)
    assert torch.allclose(ok.cpu(), g.t("out_k"), rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------ norms / activations
def test_rmsnorm_silu():
    from chitu_b200 import ops
    g = Golden("rmsnorm_silu")
    x, w = g.t("x", BF), g.t("w", BF)
    y = ops.rms_norm(cu(x), cu(w), 1e-5).cpu()
    # <= 1 bf16 ulp vs both reference compute dtypes (fp32 / bf16 opmath differ by rounding only)
    for key in ("y_f32", "y_bf16"):
        assert max_rel(y.float(), g.t(key, BF).float()) < 8e-3
    assert (y != g.t("y_f32", BF)).float().mean() < 0.01
    assert torch.equal(ops.silu_and_mul(cu(x)).cpu(), g.t("silu_mul", BF))
    torch.manual_seed(2)
    for dim in (7168, 1536, 512, 4096):
        x = (torch.randn(16, dim) * 2).to(BF)
        w = (torch.rand(dim) + 0.5).to(BF)
        y = ops.rms_norm(cu(x), cu(w), 1e-6).cpu()
        r = O.rms_norm(x, w, 1e-6)
        assert max_rel(y.float(), r.float()) < 8e-3 and (y != r).float().mean() < 0.01


# ----------------------------------------------------------------------------- fp8 quantisers
def test_act_quant_fp8_bit_exact_vs_oracle():
    from chitu_b200 import fused_moe, ops
    torch.manual_seed(7)
    for shape in [(1, 7168), (16, 7168), (16, 1536), (128, 256), (3, 2048)]:
        x = (torch.randn(*shape) * 3).to(BF)
        x[0, :128] *= 40
        y, s = ops.act_quant_deepseek_v3(cu(x))
        yo, so = O.act_quant_deepseek_v3(x)
        assert torch.equal(s.cpu(), so)
        assert torch.equal(y.cpu().view(torch.uint8), yo.view(torch.uint8))
        x[-1, -128:] = 0      # all-zero group: eps path (act_quant would give NaN, as the reference)
        q, qs = fused_moe.per_token_group_quant_fp8(cu(x), 128)
        qo, qso = O.per_token_group_quant_fp8(x, 128)
        assert torch.equal(qs.cpu(), qso)
        assert torch.equal(q.cpu().view(torch.uint8), qo.view(torch.uint8))
    g = Golden("act_quant")
    y, s = ops.act_quant_deepseek_v3(cu(g.t("x", BF)))
    assert torch.equal(s.cpu(), g.t("s"))          # reference scales: bit exact


def test_weight_dequant_bit_exact_vs_oracle():
    from chitu_b200 import ops
    g = Golden("weight_dequant")
    w, s = g.t("w", F8), g.t("s")
    assert torch.equal(ops.weight_dequant_deepseek_v3(cu(w), cu(s)).cpu(), O.weight_dequant(w, s))
    assert torch.equal(ops.weight_dequant_soft_fp8_deepseek_v3(cu(w), cu(s)).cpu(), O.weight_dequant_soft_fp8(w, s))
    w3, s3 = g.t("w3", F8), g.t("s3")
    assert torch.equal(ops.weight_dequant_deepseek_v3(cu(w3), cu(s3)).cpu(), O.weight_dequant(w3, s3))


def test_quant_act_int8_bit_exact():
    from chitu_b200.quantize import quant_act
    g = Golden("w8a8_quant")
    q, s = quant_act(cu(g.t("act")))
    assert torch.equal(q.cpu(), g.t("q")) and torch.equal(s.cpu(), g.t("s"))
    torch.manual_seed(9)
    x = (torch.randn(16, 4096) * 2).half()
    x[3] = 0
    q, s = quant_act(cu(x))
    qo, so = O.quant_act(x)
    assert torch.equal(q.cpu(), qo) and torch.equal(s.cpu(), so)


# ------------------------------------------------------------------------------------ linears
def _make_fp8_weight(N, K, gen, scale=0.05):
    w = torch.randn(N, K, generator=gen) * scale
    nb, kb = (N + 127) // 128, (K + 127) // 128
    wp = torch.zeros(nb * 128, kb * 128)
    wp[:N, :K] = w
    blocks = wp.view(nb, 128, kb, 128)
    s = blocks.abs().amax(dim=(1, 3)) / 448.0
    q = (blocks / s[:, None, :, None]).reshape(nb * 128, kb * 128)[:N, :K].to(F8)
    return q.contiguous(), s.float().contiguous()


LINEAR_IMPLS = [1, 2]


def _need_impl(impl):
    from chitu_b200 import _lib
    if impl == 2 and _lib.load().chitu_b200_linear_workspace_bytes(16, 4096) <= 0:
        pytest.skip("wgmma path not built in this library")


@pytest.mark.parametrize("impl", LINEAR_IMPLS)
@pytest.mark.parametrize("M,N,K", [(1, 4096, 4096), (16, 6144, 4096), (5, 384, 1024), (16, 2112, 7168), (33, 512, 256)])
def test_linear_bf16(impl, M, N, K):
    from chitu_b200 import ops
    _need_impl(impl)
    g = torch.Generator().manual_seed(M * 7 + N)
    x = torch.randn(M, K, generator=g).to(BF)
    w = (torch.randn(N, K, generator=g) * 0.05).to(BF)
    ops.LINEAR_IMPL = impl
    try:
        y = ops.linear(cu(x), cu(w)).cpu()
        res = torch.randn(M, N, generator=g).to(BF)
        y2 = ops.linear(cu(x), cu(w), residual=cu(res)).cpu()
    finally:
        ops.LINEAR_IMPL = 0
    r = O.linear(x, w)
    assert cos_diff(y.float(), r.float()) < 1e-5
    assert max_rel(y.float(), r.float()) < 8e-3           # bf16 output rounding (1 ulp)
    assert max_rel(y2.float(), (r + res).float()) < 8e-3


@pytest.mark.parametrize("impl", LINEAR_IMPLS)
@pytest.mark.parametrize("M,N,K", [(1, 2112, 7168), (16, 3072, 1536), (16, 7168, 2048), (4, 512, 7168), (7, 7168, 256)])
def test_fp8_gemm(impl, M, N, K):
    from chitu_b200 import ops
    _need_impl(impl)
    g = torch.Generator().manual_seed(M * 3 + K)
    a = (torch.randn(M, K, generator=g) * 2).to(BF)
    aq, a_s = O.act_quant_deepseek_v3(a)
    bq, b_s = _make_fp8_weight(N, K, g)
    ops.LINEAR_IMPL = impl
    try:
        c = ops.fp8_gemm_deepseek_v3(cu(aq), cu(a_s), cu(bq), cu(b_s)).cpu()
    finally:
        ops.LINEAR_IMPL = 0
    r = O.fp8_gemm(aq, a_s, bq, b_s, out_dtype=torch.float32)
    assert cos_diff(c.float(), r) < 1e-5
    assert max_rel(c.float(), r) < 8e-3


def test_fp8_gemm_golden():
    from chitu_b200 import ops
    g = Golden("fp8_gemm")
    c = ops.fp8_gemm_deepseek_v3(cu(g.t("aq", F8)), cu(g.t("a_s")), cu(g.t("bq", F8)), cu(g.t("b_s"))).cpu()
    assert max_rel(c.float(), g.t("c", BF).float()) < 1e-2 and cos_diff(c.float(), g.t("c", BF).float()) < 1e-5
    cs = ops.soft_fp8_gemm_deepseek_v3(cu(g.t("a", BF)), cu(g.t("bq", F8)), cu(g.t("b_s"))).cpu()
    assert max_rel(cs.float(), g.t("c_soft", BF).float()) < 1e-2


@pytest.mark.parametrize("impl", LINEAR_IMPLS)
@pytest.mark.parametrize("M,N,K", [(1, 2112, 7168), (16, 1024, 2048), (16, 7168, 2048), (7, 3072, 1536), (48, 4608, 7168),
                                   (200, 7168, 2304)])
def test_soft_fp8_gemm(impl, M, N, K):
    """soft_fp8_gemm_deepseek_v3 (ops.py:486-511): impl 2 = wgmma (fp8 -> bf16 conversion warps between TMA and the
    bf16 MMA, same "weight rounded to bf16 before the MMA" semantics), impl 1 = SIMT."""
    from chitu_b200 import ops
    _need_impl(impl)
    g = torch.Generator().manual_seed(K + M)
    a = torch.randn(M, K, generator=g).to(BF)
    bq, b_s = _make_fp8_weight(N, K, g)
    ops.LINEAR_IMPL = impl
    try:
        c = ops.soft_fp8_gemm_deepseek_v3(cu(a), cu(bq), cu(b_s)).cpu()
    finally:
        ops.LINEAR_IMPL = 0
    r = O.soft_fp8_gemm(a, bq, b_s)
    assert cos_diff(c.float(), r.float()) < 1e-5 and max_rel(c.float(), r.float()) < 8e-3


@pytest.mark.parametrize("impl", LINEAR_IMPLS)
def test_w8a8_reference_tests(impl):
    # test/pytest/test_w8a8.py:13-48 — same seeds, shapes and tolerance
    from chitu_b200.quantize import w8a8gemm, w8a8gemv
    _need_impl(impl)
    w8a8gemm.IMPL = impl
    try:
        torch.manual_seed(0)
        m, n, k = 1024, 2048, 4096
        a = (torch.randn([m, k], device=DEV) * 4).to(torch.int8)
        b = (torch.randn([n, k], device=DEV) * 4).to(torch.int8)
        c = torch.zeros([m, n], dtype=torch.float16, device=DEV)
        w8a8gemm.mm(c, a, b, torch.ones([m], device=DEV), torch.ones([n], device=DEV), None)
        c1 = torch.mm(a.to(torch.float16), b.transpose(0, 1).to(torch.float16))
        assert torch.allclose(c, c1, rtol=5e-3, atol=5e-3)
        torch.manual_seed(0)
        a = (torch.randn([2, 1, 11008], device=DEV) * 4).to(torch.int8)
        b = (torch.randn([4096, 11008], device=DEV) * 4).to(torch.int8)
        c = w8a8gemv.mv(a, b, torch.ones([2], device=DEV), torch.ones([4096], device=DEV))
        c0 = torch.mm(a.reshape(2, 11008).to(torch.float16), b.transpose(0, 1).to(torch.float16)).reshape(2, 1, 4096)
        assert torch.allclose(c, c0, rtol=5e-3, atol=5e-3)
    finally:
        w8a8gemm.IMPL = 0


def test_w8a8_linear_module_vs_oracle():
    from chitu_b200.quantize import W8A8Linear
    torch.manual_seed(4)
    import copy
    lin = torch.nn.Linear(4096, 1024, bias=True).half()
    q = W8A8Linear.from_float(copy.deepcopy(lin).to(DEV))
    for shape in [(16, 4096), (2, 1, 4096), (8, 1, 4096)]:
        x = torch.randn(*shape).half()
        y = q(cu(x)).cpu()
        qx, sx = O.quant_act(x)
        wq, ws = O.quant_weight(lin.weight.data)
        r = O.w8a8_mm(qx, wq, sx, ws, lin.bias.data.cpu()).reshape(*shape[:-1], 1024)
        assert torch.allclose(y, r, rtol=5e-3, atol=5e-3)


# ---------------------------------------------------------------------------------- attention
def _paged(B, pages_per, page, tail_shape, gen, poison=True):
    nblk = B * pages_per + 3
    cache = torch.randn(nblk, page, *tail_shape, generator=gen).to(BF)
    table = torch.randperm(nblk, generator=gen)[: B * pages_per].to(torch.int32).view(B, pages_per).contiguous()
    return cache, table


def test_mla_decode_golden():
    from chitu_b200.attn_backend import B200AttnBackend
    g = Golden("mla_decode")
    be = B200AttnBackend()
    lens = g.t("lens")
    out = be.mla_attn_with_kvcache(cu(g.t("q_nope", BF)), cu(g.t("q_pe", BF)), cu(g.t("cache", BF)), None,
                                   cu(lens), cu(lens), cu(g.t("table")), softmax_scale=float(g.np("scale")))
    ref = g.t("out")
    assert cos_diff(out.cpu().float().view(ref.shape), ref) < 1e-5
    assert max_rel(out.cpu().float().view(ref.shape), ref) < 1e-2


@pytest.mark.parametrize("B,H,S", [(1, 16, 4096), (16, 16, 4096), (3, 16, 130), (2, 128, 1000), (4, 8, 64)])
def test_mla_decode_with_append_vs_oracle(B, H, S):
    from chitu_b200.attn_backend import B200AttnBackend
    g = torch.Generator().manual_seed(B * 100 + H)
    C, R, page = 512, 64, 64
    pages_per = S // page + 1
    cache, table = _paged(B, pages_per, page, (C + R,), g)
    lens = torch.randint(max(S // 2, 1), S, (B,), generator=g).to(torch.int32)
    lens[0] = S - 1 if S % page else S - 1
    if B > 1:
        lens[1] = (S // page) * page - 1 if S >= page else 0      # append lands on a page boundary
    # NaN-poison everything past the valid length (FlashMLA test_flash_mla.py:62-65): OOB reads blow up
    for b in range(B):
        L = int(lens[b])
        for pi in range(pages_per):
            lo = max(L + 1 - pi * page, 0)
            if lo < page:
                cache[table[b, pi].long(), lo:] = float("nan")
    q_nope = torch.randn(B, H, C, generator=g).to(BF)
    q_pe = torch.randn(B, H, R, generator=g).to(BF)
    kv = torch.randn(B, 1, 1, C + R, generator=g).to(BF)
    scale = 0.1352337788
    be = B200AttnBackend()
    dcache = cu(cache.clone())
    out = be.mla_attn_with_kvcache(cu(q_nope), cu(q_pe), dcache, cu(kv), cu(lens), cu(lens + 1), cu(table),
                                   softmax_scale=scale)
    ocache = cache.clone()
    ref = O.mla_attn_with_kvcache(q_nope, q_pe, ocache, kv, lens, table, scale)
    # KV-page indexing: bit exact (NaN-aware compare on the raw bits)
    assert torch.equal(dcache.cpu().view(torch.int16), ocache.view(torch.int16))
    o = out.cpu().float().view(B, H, C)
    assert not torch.isnan(o).any()
    assert cos_diff(o, ref.float()) < 1e-5
    assert max_rel(o, ref.float()) < 1e-2


@pytest.mark.parametrize("B,Hq,Hkv,D,page,S", [(1, 32, 8, 128, 256, 4096), (16, 32, 8, 128, 256, 4096),
                                                (3, 8, 2, 128, 256, 300), (2, 32, 32, 128, 256, 128),
                                                (5, 8, 8, 64, 16, 77)])
def test_gqa_paged_decode_vs_oracle(B, Hq, Hkv, D, page, S):
    from chitu_b200.attn_backend import B200AttnBackend
    g = torch.Generator().manual_seed(B + Hq + S)
    pages_per = S // page + 1
    kc, table = _paged(B, pages_per, page, (Hkv, D), g)
    vc = torch.randn(kc.shape, generator=g).to(BF)
    lens = torch.randint(max(S // 2, 1), S, (B,), generator=g).to(torch.int32)
    lens[0] = S - 1
    q = torch.randn(B, 1, Hq, D, generator=g).to(BF)
    k = torch.randn(B, 1, Hkv, D, generator=g).to(BF)
    v = torch.randn(B, 1, Hkv, D, generator=g).to(BF)
    be = B200AttnBackend()
    dk, dv = cu(kc.clone()), cu(vc.clone())
    out = be.attn_with_kvcache(cu(q), dk, dv, cu(k), cu(v), cache_seqlens=cu(lens), block_table=cu(table))
    ok_, ov_ = kc.clone(), vc.clone()
    ref = O.gqa_paged_decode(q, ok_, ov_, k, v, lens, table)
    assert torch.equal(dk.cpu(), ok_) and torch.equal(dv.cpu(), ov_)       # in-place append: bit exact
    assert cos_diff(out.cpu().float(), ref.float()) < 1e-5
    assert max_rel(out.cpu().float(), ref.float()) < 1e-2


def test_gqa_decode_ref_backend_golden():
    from chitu_b200.attn_backend import B200AttnBackend
    g = Golden("ref_attn_gqa")
    kc, vc = g.t("k_cache", BF), g.t("v_cache", BF)
    B = kc.shape[0]
    page = 100
    k_pages, v_pages = kc.reshape(B * 3, page, *kc.shape[2:]).clone(), vc.reshape(B * 3, page, *vc.shape[2:]).clone()
    table = torch.arange(B * 3, dtype=torch.int32).view(B, 3)
    be = B200AttnBackend()
    dk, dv = cu(k_pages), cu(v_pages)
    out = be.attn_with_kvcache(cu(g.t("q", BF)), dk, dv, cu(g.t("k", BF)), cu(g.t("v", BF)),
                               cache_seqlens=cu(g.t("lens")), block_table=cu(table))
    assert torch.equal(dk.cpu().reshape(kc.shape), g.t("k_cache_after", BF))
    ref = g.t("out", BF).float()
    assert cos_diff(out.cpu().float(), ref) < 1e-5 and max_rel(out.cpu().float(), ref) < 1e-2


# ---------------------------------------------------------------------------------------- MoE
def test_gate_golden_bit_exact_indices():
    from chitu_b200 import fused_moe
    g = Golden("gate_sigmoid_f32bias")
    w, idx = fused_moe.moe_gate(cu(g.t("x", BF)), cu(g.t("weight", BF)), cu(g.t("bias")), 8, 8, 4, "sigmoid", 2.5)
    assert torch.equal(idx.cpu(), g.t("idx"))                           # routing: bit exact
    assert max_rel(w.cpu().float(), g.t("w", BF).float()) < 8e-3        # <= 1 bf16 ulp
    g = Golden("gate_softmax")
    w, idx = fused_moe.moe_gate(cu(g.t("x", BF)), cu(g.t("weight", BF)), None, 6, 4, 2, "softmax", 1.0)
    assert torch.equal(idx.cpu(), g.t("idx"))
    assert max_rel(w.cpu().float(), g.t("w", BF).float()) < 8e-3


def test_gate_vs_oracle_bs16():
    from chitu_b200 import fused_moe
    g = torch.Generator().manual_seed(21)
    x = torch.randn(16, 7168, generator=g).to(BF)
    wg = (torch.randn(256, 7168, generator=g) * 0.02).to(BF)
    bias = torch.randn(256, generator=g) * 0.01
    w, idx = fused_moe.moe_gate(cu(x), cu(wg), cu(bias), 8, 8, 4, "sigmoid", 2.5)
    wo, io, scores = O.moe_gate(x, wg, bias, 8, 8, 4, "sigmoid", 2.5)
    # tie-free check of the oracle's own selection margin, then exact index equality
    top9 = scores.topk(9, dim=-1)[0]
    assert (top9[:, 7] - top9[:, 8]).min() > 0
    assert torch.equal(idx.cpu(), io)
    assert max_rel(w.cpu().float(), wo.float()) < 8e-3


@pytest.mark.parametrize("mode", ["bf16", "fp8_w8a8", "soft_fp8"])
def test_fused_experts_vs_oracle(mode):
    from chitu_b200 import fused_moe
    g = torch.Generator().manual_seed(31)
    T, K1, N1, E, topk = 5, 512, 512, 16, 4
    x = torch.randn(T, K1, generator=g).to(BF)
    ids = torch.stack([torch.randperm(E, generator=g)[:topk] for _ in range(T)])
    tw = torch.rand(T, topk, generator=g).to(BF)
    if mode == "bf16":
        w1 = (torch.randn(E, N1, K1, generator=g) * 0.05).to(BF)
        w2 = (torch.randn(E, K1, N1 // 2, generator=g) * 0.05).to(BF)
        out = fused_moe.fused_experts(cu(x), cu(w1), cu(w2), cu(tw), cu(ids), inplace=False)
        ref = O.fused_experts(x, w1, w2, tw, ids, mode="bf16")
    else:
        w1q, w1s, w2q, w2s = [], [], [], []
        for _ in range(E):
            q, s = _make_fp8_weight(N1, K1, g)
            w1q.append(q), w1s.append(s)
            q, s = _make_fp8_weight(K1, N1 // 2, g)
            w2q.append(q), w2s.append(s)
        w1q, w1s, w2q, w2s = torch.stack(w1q), torch.stack(w1s), torch.stack(w2q), torch.stack(w2s)
        out = fused_moe.fused_experts(cu(x), cu(w1q), cu(w2q), cu(tw), cu(ids), inplace=False, use_fp8_w8a8=True,
                                      w1_scale=cu(w1s), w2_scale=cu(w2s), block_shape=[128, 128],
                                      soft_fp8=(mode == "soft_fp8"))
        ref = O.fused_experts(x, w1q, w2q, tw, ids, w1s, w2s, mode=mode)
    assert cos_diff(out.cpu().float(), ref.float()) < 1e-4
    assert max_rel(out.cpu().float(), ref.float()) < 1e-2


def test_fused_experts_golden_bf16():
    from chitu_b200 import fused_moe
    g = Golden("fused_experts")
    out = fused_moe.fused_experts(cu(g.t("x", BF)), cu(g.t("w1", BF)), cu(g.t("w2", BF)), cu(g.t("tw", BF)),
                                  cu(g.t("ids")), inplace=False)
    assert cos_diff(out.cpu().float(), g.t("out")) < 1e-4 and max_rel(out.cpu().float(), g.t("out")) < 1e-2


def test_fused_experts_inplace_and_flags():
    from chitu_b200 import fused_moe
    g = Golden("fused_experts")
    x = cu(g.t("x", BF))
    y = fused_moe.fused_experts(x, cu(g.t("w1", BF)), cu(g.t("w2", BF)), cu(g.t("tw", BF)), cu(g.t("ids")), inplace=True)
    assert y.data_ptr() == x.data_ptr()
    with pytest.raises(NotImplementedError):
        fused_moe.fused_experts(x, cu(g.t("w1", BF)), cu(g.t("w2", BF)), cu(g.t("tw", BF)), cu(g.t("ids")),
                                use_int8_w8a16=True)


# ------------------------------------------------------------------------- fused decode-engine ops
def test_fused_rmsnorm_quant_and_silu_quant():
    from chitu_b200 import ops
    torch.manual_seed(12)
    for dim in (7168, 1536, 512, 2048):
        x = (torch.randn(16, dim) * 2).to(BF)
        w = (torch.rand(dim) + 0.5).to(BF)
        y, q, s = ops.rms_norm_quant(cu(x), cu(w), 1e-6)
        r = O.rms_norm(x, w, 1e-6)
        assert max_rel(y.cpu().float(), r.float()) < 8e-3 and (y.cpu() != r).float().mean() < 0.01
        qo, so = O.act_quant_deepseek_v3(y.cpu())               # quantisation of the kernel's own y: bit exact
        assert torch.equal(s.cpu(), so) and torch.equal(q.cpu().view(torch.uint8), qo.view(torch.uint8))
    x = torch.randn(9, 2 * 2304).to(BF)
    q, s = ops.silu_mul_quant(cu(x))
    qo, so = O.act_quant_deepseek_v3(O.silu_and_mul(x))
    assert torch.equal(s.cpu(), so) and torch.equal(q.cpu().view(torch.uint8), qo.view(torch.uint8))


@pytest.mark.parametrize("B,S", [(1, 4096), (16, 4096), (3, 130)])
def test_mla_deferred_merge_in_absorb_o_is_bit_identical(B, S):
    """chitu_b200_mla_decode(out = NULL) + chitu_b200_mla_absorb_o_merge_quant == decode + merge + absorb_o_quant: the merged
    latent output, the bf16 head outputs, the fp8 payload and the scales are identical bit for bit."""
    from chitu_b200 import _lib
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib.load()
    g = torch.Generator().manual_seed(B + S)
    H, C, R, dn, dv, page = 16, 512, 64, 128, 128, 64
    pages_per = S // page + 1
    cache, table = _paged(B, pages_per, page, (C + R,), g)
    lens = torch.randint(max(S // 2, 1), S, (B,), generator=g).to(torch.int32)
    lens[0] = S - 1
    q_nope, q_pe = cu(torch.randn(B, H, C, generator=g).to(BF)), cu(torch.randn(B, H, R, generator=g).to(BF))
    kv = cu(torch.randn(B, C + R, generator=g).to(BF))
    wkv = cu((torch.randn(H, dn + dv, C, generator=g) * 0.05).to(BF))
    dl, dt = cu(lens), cu(table)
    ws = torch.zeros(lib.chitu_b200_attn_workspace_bytes(B, H, C, 128), dtype=torch.uint8, device=DEV)
    outs = []
    for deferred in (False, True):
        dc = cu(cache.clone())
        x = torch.zeros(B, H, C, dtype=BF, device=DEV)
        o = torch.zeros(B, H * dv, dtype=BF, device=DEV)
        q = torch.zeros(B, H * dv, dtype=F8, device=DEV)
        qs = torch.zeros(B, H, dtype=torch.float32, device=DEV)
        check(lib.chitu_b200_mla_decode(ptr(q_nope), ptr(q_pe), ptr(dc), ptr(kv), ptr(dl), ptr(dt), dt.stride(0), B, H, C, R,
                                        page, dc.shape[0], S + 1, 0.1352337788, None if deferred else ptr(x), ptr(ws),
                                        ws.numel(), current_stream()), "mla_decode")
        if deferred:
            check(lib.chitu_b200_mla_absorb_o_merge_quant(ptr(ws), ws.numel(), S + 1, ptr(wkv), ptr(x), ptr(o), ptr(q), ptr(qs),
                                                          B, H, dn, dv, C, current_stream()), "absorb_o_merge")
        else:
            check(lib.chitu_b200_mla_absorb_o_quant(ptr(x), ptr(wkv), ptr(o), ptr(q), ptr(qs), B, H, dn, dv, C,
                                                    current_stream()), "absorb_o")
        torch.cuda.synchronize()
        outs.append((x.cpu(), o.cpu(), q.cpu().view(torch.uint8), qs.cpu(), dc.cpu()))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a.view(torch.int16) if a.dtype == BF else a, b.view(torch.int16) if b.dtype == BF else b)


@pytest.mark.parametrize("B,Hq,Hkv,S", [(16, 32, 8, 4096), (1, 32, 8, 4096), (3, 8, 2, 300), (2, 4, 1, 255)])
def test_gqa_fused_rotary_is_bit_identical(B, Hq, Hkv, S):
    """chitu_b200_gqa_paged_decode_rope (rotary of q and of the appended k inside the attention kernel, q/k/v = strided views
    of the fused qkv GEMM output) == apply_rotary_pos_emb followed by attn_with_kvcache: output and caches bit for bit."""
    from chitu_b200 import _lib
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib.load()
    g = torch.Generator().manual_seed(B * 7 + S)
    D, page = 128, 256
    pages_per = S // page + 1
    kc, table = _paged(B, pages_per, page, (Hkv, D), g)
    vc = torch.randn(kc.shape, generator=g).to(BF)
    lens = torch.randint(max(S // 2, 1), S, (B,), generator=g).to(torch.int32)
    lens[0] = S - 1
    if B > 1:
        lens[1] = (S // page) * page - 1 if S >= page else 3
    qkv_w = (Hq + 2 * Hkv) * D
    qkv = cu(torch.randn(B, qkv_w, generator=g).to(BF))
    cos, sin = cu(torch.randn(B, D // 2, generator=g)), cu(torch.randn(B, D // 2, generator=g))
    q_view, k_view, v_view = qkv, qkv[:, Hq * D:], qkv[:, (Hq + Hkv) * D:]
    dl, dt = cu(lens), cu(table)
    ws = torch.zeros(lib.chitu_b200_attn_workspace_bytes(B, Hq, D, 64), dtype=torch.uint8, device=DEV)
    res = []
    for fused in (False, True):
        dk, dv = cu(kc.clone()), cu(vc.clone())
        out = torch.zeros(B, Hq, D, dtype=BF, device=DEV)
        if fused:
            check(lib.chitu_b200_gqa_paged_decode_rope(ptr(q_view), qkv_w, ptr(dk), ptr(dv), ptr(k_view), ptr(v_view), qkv_w,
                                                       qkv_w, ptr(cos), ptr(sin), ptr(dl), ptr(dt), dt.stride(0), B, Hq, Hkv, D,
                                                       page, S + 1, 1.0 / D ** 0.5, ptr(out), ptr(ws), ws.numel(), _lib.CB_BF16,
                                                       current_stream()), "gqa_rope")
        else:
            q_rot = torch.empty(B, Hq, D, dtype=BF, device=DEV)
            k_rot = torch.empty(B, Hkv, D, dtype=BF, device=DEV)
            check(lib.chitu_b200_rotary_interleaved(ptr(q_view), ptr(k_view), ptr(q_rot), ptr(k_rot), ptr(cos), ptr(sin), B, Hq,
                                                    Hkv, D, qkv_w, D, qkv_w, D, _lib.CB_BF16, current_stream()), "rotary")
            check(lib.chitu_b200_gqa_paged_decode(ptr(q_rot), ptr(dk), ptr(dv), ptr(k_rot), ptr(v_view), Hkv * D, qkv_w, ptr(dl),
                                                  ptr(dt), dt.stride(0), B, Hq, Hkv, D, page, S + 1, 1.0 / D ** 0.5, ptr(out),
                                                  ptr(ws), ws.numel(), _lib.CB_BF16, current_stream()), "gqa")
        torch.cuda.synchronize()
        res.append((out.cpu(), dk.cpu(), dv.cpu()))
    for a, b in zip(res[0], res[1]):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))



def test_decode_prepare_matches_cache_manager_semantics():
    """chitu_b200_decode_prepare vs a numpy restatement of PagedKVCacheManager.prepare_cache_decode +
    prepare_block_table_for_decode (+ finalize_cache_single_decode), cache_manager.py:148-158,196-215: a request on a page
    boundary pops a free page into its block-table row; lengths advance; bit exact, several steps, pool exhaustion flagged."""
    from chitu_b200 import _lib
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib.load()
    B, page, max_blocks, nfree = 37, 64, 9, 40
    rng = np.random.default_rng(0)
    lens = rng.integers(1, 5 * page, size=B).astype(np.int32)
    lens[:4] = [63, 64, 127, 128]
    table = np.zeros((B, max_blocks), dtype=np.int32)
    nxt = 1000
    for b in range(B):
        for j in range((lens[b] + page - 1) // page):
            table[b, j] = nxt
            nxt += 1
    free = np.arange(500, 500 + nfree, dtype=np.int32)
    d_lens, d_incl, d_table = cu(torch.from_numpy(lens.copy())), torch.zeros(B, dtype=torch.int32, device=DEV), cu(torch.from_numpy(table.copy()))
    d_free, d_cnt = cu(torch.from_numpy(free.copy())), torch.tensor([nfree], dtype=torch.int32, device=DEV)
    d_status = torch.zeros(1, dtype=torch.int32, device=DEV)
    r_lens, r_table, r_cnt = lens.copy(), table.copy(), nfree
    for step in range(3):
        adv = 1 if step > 0 else 0
        check(lib.chitu_b200_decode_prepare(ptr(d_lens), ptr(d_incl), ptr(d_table), max_blocks, ptr(d_free), ptr(d_cnt),
                                            ptr(d_status), B, page, adv, current_stream()), "decode_prepare")
        torch.cuda.synchronize()
        if adv:
            r_lens += 1
        need = [b for b in range(B) if r_lens[b] % page == 0]
        got_tab = d_table.cpu().numpy()
        assert np.array_equal(d_lens.cpu().numpy(), r_lens) and np.array_equal(d_incl.cpu().numpy(), r_lens + 1)
        # which free page a request gets depends on the pop order (a set in the reference): check the SET of pages handed
        # out, that each needy request got exactly one new page in the right slot, and that nothing else changed
        new_pages = sorted(int(got_tab[b, r_lens[b] // page]) for b in need)
        assert new_pages == sorted(free[r_cnt - len(need): r_cnt].tolist())
        for b in need:
            r_table[b, r_lens[b] // page] = got_tab[b, r_lens[b] // page]
        r_cnt -= len(need)
        assert np.array_equal(got_tab, r_table) and int(d_cnt.item()) == r_cnt and int(d_status.item()) == 0
    d_cnt.fill_(0)
    d_lens.fill_(page - 1)
    check(lib.chitu_b200_decode_prepare(ptr(d_lens), ptr(d_incl), ptr(d_table), max_blocks, ptr(d_free), ptr(d_cnt), ptr(d_status),
                                        B, page, 1, current_stream()), "decode_prepare")
    torch.cuda.synchronize()
    assert int(d_status.item()) == 1 and int(d_cnt.item()) == 0        # "No more free blocks." is reported, not crashed on


@pytest.mark.parametrize("B,mean", [(16, 4096), (64, 1024), (5, 300)])
def test_mla_decode_with_device_plan_varlen(B, mean):
    """prepare_metadata_for_decode -> chitu_b200_attn_plan (length-aware splits, no host sync) + the MLA kernel on a ragged
    batch drawn like third_party/FlashMLA/tests/test_flash_mla.py:46-49: same output as without the plan / as the oracle."""
    from chitu_b200.attn_backend import B200AttnBackend
    g = torch.Generator().manual_seed(B)
    H, C, R, page = 16, 512, 64, 64
    lens = torch.clamp(torch.normal(float(mean), mean / 2.0, (B,), generator=g), min=1).to(torch.int32)
    lens[0] = 2 * mean
    S = int(lens.max()) + 1
    pages_per = S // page + 1
    cache, table = _paged(B, pages_per, page, (C + R,), g)
    q_nope, q_pe = torch.randn(B, H, C, generator=g).to(BF), torch.randn(B, H, R, generator=g).to(BF)
    kv = torch.randn(B, 1, 1, C + R, generator=g).to(BF)
    be = B200AttnBackend(max_seq_len=S, max_reqs=B, n_local_heads=H)
    dl = cu(lens)
    be.prepare_metadata_for_decode(dl, dl + 1, cu(table), page)
    dcache = cu(cache.clone())
    out = be.mla_attn_with_kvcache(cu(q_nope), cu(q_pe), dcache, cu(kv), dl, dl + 1, cu(table), softmax_scale=0.1352337788)
    plan = be.last_plan().cpu()
    assert plan[0] == 0x504C414E and plan[1] % page == 0 and plan[1] > 0 and plan[4] == B
    ocache = cache.clone()
    ref = O.mla_attn_with_kvcache(q_nope, q_pe, ocache, kv, lens, table, 0.1352337788)
    assert torch.equal(dcache.cpu().view(torch.int16), ocache.view(torch.int16))
    o = out.cpu().float().view(B, H, C)
    assert cos_diff(o, ref.float()) < 1e-5 and max_rel(o, ref.float()) < 1e-2


@pytest.mark.parametrize("mode", ["bf16", "fp8_w8a8", "soft_fp8"])
@pytest.mark.parametrize("gemm", [1, 2])
def test_invoke_fused_moe_kernel_standalone(mode, gemm):
    """a15: the stand-alone grouped GEMM with the reference's calling convention (fused_moe.py:796-891): blocks of
    moe_align_block_size output, row r reads A[sorted_ids[r] // top_k] and writes C.view(-1, N)[sorted_ids[r]]."""
    from chitu_b200 import fused_moe
    g = torch.Generator().manual_seed(11 + gemm)
    T, K, N, E, topk, block_m = 9, 512, 256, 12, 3, 16
    ids = torch.stack([torch.randperm(E, generator=g)[:topk] for _ in range(T)]).to(torch.int32)
    tw = torch.rand(T, topk, generator=g).to(BF)
    top_k = topk if gemm == 1 else 1
    A = torch.randn(T if gemm == 1 else T * topk, K, generator=g).to(BF)
    if mode == "bf16":
        Bw, Bs = (torch.randn(E, N, K, generator=g) * 0.05).to(BF), None
    else:
        qs = [_make_fp8_weight(N, K, g) for _ in range(E)]
        Bw, Bs = torch.stack([q for q, _ in qs]), torch.stack([s for _, s in qs])
    sorted_ids, expert_ids, npp = fused_moe.moe_align_block_size(cu(ids), block_m, E)
    C = torch.full((T, topk, N), float("nan"), dtype=BF, device=DEV)
    fused_moe.invoke_fused_moe_kernel(cu(A), cu(Bw), C, None, cu(Bs) if Bs is not None else None, None, cu(tw), cu(ids), sorted_ids,
                                      expert_ids, npp, gemm == 2, top_k, {"BLOCK_SIZE_M": block_m}, None,
                                      use_fp8_w8a8=mode != "bf16", block_shape=[128, 128] if mode != "bf16" else None,
                                      soft_fp8=mode == "soft_fp8")
    ref = torch.empty(T * topk, N)
    for p in range(T * topk):
        e = int(ids.view(-1)[p])
        a = A[p // top_k: p // top_k + 1]
        if mode == "bf16":
            y = a.float() @ Bw[e].float().T
        elif mode == "fp8_w8a8":
            aq, a_s = O.per_token_group_quant_fp8(a, 128)
            y = O.fp8_gemm(aq, a_s, Bw[e], Bs[e], torch.float32)
        else:
            y = a.float() @ O.weight_dequant_soft_fp8(Bw[e], Bs[e]).float().T
        if gemm == 2:
            y = y * float(tw.view(-1)[p])
        ref[p] = y[0]
    got = C.view(-1, N).cpu().float()
    assert not torch.isnan(got).any()
    assert cos_diff(got, ref) < 1e-5 and max_rel(got, ref) < 1e-2


@pytest.mark.parametrize("V,dtype", [(129280, torch.bfloat16), (32000, torch.float32), (1000, torch.float32)])
def test_sample_top_k_top_p_vs_reference_rule(V, dtype):
    """n3: the kept set of the sampling kernel == the reference's sort / cumsum / mask rule (utils.py:62-81) on tie-free
    rows, and the drawn token == the inverse CDF (vocabulary order) of the reference-filtered distribution at the same u."""
    from chitu_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(V)
    B = 12
    logits = (torch.randn(B, V, generator=g, device=DEV) * 3).to(dtype)
    temps = torch.tensor([1.0, 0.7, 1.3, 0.5, 1.0, 2.0, 1.0, 0.9, 1.1, 1.0, 0.8, 1.0], device=DEV)
    top_ks = torch.tensor([50, 1, 1000, 7, V, 20, 3, 100, 5, 64, 10, 2], device=DEV, dtype=torch.int32)
    top_ps = torch.tensor([0.9, 1.0, 0.5, 0.95, 0.8, 0.99, 0.3, 0.7, 1.0, 0.6, 0.85, 0.999], device=DEV)
    u = torch.rand(B, generator=g, device=DEV)
    tok, kept, mass = ops.sample_top_k_top_p(logits, temps, top_ks, top_ps, u, return_stats=True)
    # the reference's rule, verbatim (fp32 on the GPU)
    probs = torch.softmax(logits.float() / temps.view(-1, 1), dim=-1)
    ps, pi = probs.sort(dim=-1, descending=True)
    cs = torch.cumsum(ps, dim=-1)
    ps = ps.clone()
    ps[(cs - ps) > top_ps.view(-1, 1)] = 0.0
    ps[torch.arange(V, device=DEV).view(1, -1) >= top_ks.view(-1, 1)] = 0.0
    for b in range(B):
        ref_idx = pi[b][ps[b] > 0]
        n_ref = ref_idx.numel()
        # entries right at the top-p boundary may fall either way (cumsum rounding): allow +-1 there; entries TIED with the
        # smallest kept probability (bf16 logits tie often) are all kept by the kernel, whereas the reference's sort keeps
        # an arbitrary subset of them up to top_k
        p_min = probs[b][ref_idx].min()
        ties = int((probs[b] == p_min).sum()) - int((probs[b][ref_idx] == p_min).sum())
        assert -1 <= int(kept[b]) - n_ref <= 1 + ties, (b, int(kept[b]), n_ref, ties)
        keep = torch.zeros(V, dtype=torch.bool, device=DEV)
        keep[ref_idx] = True
        masked = torch.where(keep, probs[b].double(), torch.zeros((), dtype=torch.float64, device=DEV))
        cdf = torch.cumsum(masked, dim=0)
        target = float(u[b]) * float(cdf[-1])
        want = int(torch.searchsorted(cdf, torch.tensor([target], dtype=torch.float64, device=DEV), right=True)[0])
        near = torch.nonzero(keep).view(-1)
        pos = int(torch.searchsorted(near, torch.tensor([want], device=DEV))[0])
        nb = {int(near[j]) for j in range(max(pos - 1, 0), min(pos + 2, near.numel()))}      # neighbours in the kept set
        if int(kept[b]) == n_ref:
            assert int(tok[b]) in nb, (b, int(tok[b]), want)
        assert bool(keep[int(tok[b])]) or int(kept[b]) != n_ref
    assert int(tok[1]) == int(logits[1].float().argmax())                                      # top_k = 1 is greedy


@pytest.mark.parametrize("M,N,K", [(16, 28672, 4096), (1, 28672, 4096), (5, 1024, 512), (16, 7168, 4096), (40, 2048, 1024)])
def test_linear_silu_pairs_epilogue(M, N, K):
    """FeedForward gate_up + SiluAndMul in one launch (interleaved gate/up rows) == linear followed by silu_and_mul: the same
    roundings; the accumulation order of a row can differ (stream-K split points move with the row permutation) -> <= 1 ulp."""
    from chitu_b200 import _lib, ops
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib.load()
    g = torch.Generator().manual_seed(M + N)
    x = cu(torch.randn(M, K, generator=g).to(BF))
    w = cu((torch.randn(N, K, generator=g) * 0.05).to(BF))                     # [gate ; up]
    F = N // 2
    wp = w.view(2, F, K).transpose(0, 1).reshape(N, K).contiguous()           # interleaved
    y = torch.empty(M, F, dtype=BF, device=DEV)
    ws = torch.zeros(lib.chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
    check(lib.chitu_b200_linear_bf16_silu_pairs(ptr(x), ptr(wp), ptr(y), M, N, K, ptr(ws), ws.numel(), current_stream()), "pairs")
    ref = ops.silu_and_mul(ops.linear(x, w))
    r32 = O.silu_and_mul(O.linear(x.cpu(), w.cpu())).float()
    assert max_rel(y.cpu().float(), r32) < 8e-3 and cos_diff(y.cpu().float(), r32) < 1e-5
    assert (y != ref).float().mean().item() < 0.02
