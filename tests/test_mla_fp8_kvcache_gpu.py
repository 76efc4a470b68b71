"""Absorbed-MLA attention over an fp8 (e4m3fn) paged latent cache (chitu_b200_mla_attn_fp8kv behind
B200AttnBackend.mla_attn_with_kvcache, both call shapes): argument checks, the Python refusals and the fp32 reference
without a GPU; on the H100 parity over NaN-poisoned caches, the stored bytes, bit-identity with the bf16 kernels on
the decoded cache (direct, deferred merge, sq > 1), the split regimes, CUDA-graph replay, multi-token-prediction
verification against successive decodes, the e4m3 prefill scatter and the DeepSeek engine with kv_dtype=e4m3."""
import pytest
import torch

from conftest import cos_diff, max_rel
from test_mla_paged_prefill_gpu import C, PAGE, R, ROW, SCALE, check_rows, make_case, reference

F8 = torch.float8_e4m3fn
NAN_E4M3 = 0x7F


def _backend(**kw):
    from chitu_b200.attn_backend import B200AttnBackend
    return B200AttnBackend(**kw)


def quant(x):
    """The store rule of the e4m3 cache."""
    return x.float().clamp(-448.0, 448.0).to(F8)


def to_fp8_case(c, scale_rows=1.0):
    """The bf16 case of make_case as an e4m3 cache: written rows quantised (optionally scaled first), every NaN slot
    the e4m3 NaN byte."""
    kc = c["kv_cache"]
    nan = torch.isnan(kc)
    q = quant(kc.float() * scale_rows).view(torch.uint8)
    q[nan] = NAN_E4M3
    f = dict(c)
    f["kv_cache"] = q.view(F8)
    if c["kv"] is not None:
        f["kv"] = (c["kv"].float() * scale_rows).bfloat16()
    return f


def ref_fp8(q_nope, q_pe, kv_cache, kv, seq_excl, block_table, causal, scale):
    """fp32 reference: decode the cache, append quant(new rows), then the bf16 cache's reference (pinned to the
    oracle in test_mla_paged_prefill_gpu).  Returns (out, the expected e4m3 cache)."""
    dec = kv_cache.float().bfloat16()
    kvq = None if kv is None else quant(kv).float().bfloat16()
    out, kc = reference(q_nope, q_pe, dec, kvq, seq_excl, block_table, causal, scale)
    stored = kv_cache.clone()
    if kv is not None:
        B, sq = q_nope.shape[:2]
        for b in range(B):
            pos = torch.arange(int(seq_excl[b]), int(seq_excl[b]) + sq, device=kv_cache.device)
            stored[block_table[b, pos // PAGE].long(), pos % PAGE] = quant(kv.reshape(B, sq, ROW)[b])
    return out, stored


def _call(be, c, causal=True, decode_3d=False, **kw):
    qn, qp = c["q_nope"], c["q_pe"]
    if decode_3d:
        qn, qp = qn[:, 0], qp[:, 0]
    return be.mla_attn_with_kvcache(qn, qp, c["kv_cache"], c["kv"], c["seq_excl"], None, c["block_table"],
                                    causal=causal, **kw)


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ---------------------------------------------------------------- no GPU needed

def test_mla_attn_fp8kv_bad_arguments_return_status():
    from chitu_b200 import _lib
    lib = _lib.load()
    A = 16

    def call(qn=A, qpe=A, kc=A, bt=A, new_kv=None, out=A, ws=None, B=1, sq=2, H=16, c=C, r=R, page=PAGE, nb=8):
        return lib.chitu_b200_mla_attn_fp8kv(qn, qpe, kc, new_kv, A, bt, 4, B, sq, H, c, r, page, nb, 256, 1, SCALE,
                                             out, ws, 0 if ws is None else 1 << 20, None)

    bad = [dict(qn=None), dict(qpe=None), dict(kc=None), dict(bt=None), dict(out=None),   # sq > 1: out is required
           dict(sq=0), dict(H=0), dict(B=-1), dict(sq=1, H=0),
           dict(c=256), dict(r=32), dict(page=128), dict(sq=1, c=256), dict(sq=1, page=32),
           dict(qn=A + 8), dict(new_kv=A + 2), dict(kc=A + 4), dict(sq=1, qpe=A + 8),
           dict(sq=1, out=None),                                                 # deferred merge without a workspace
           dict(B=1 << 20, sq=64, H=128), dict(nb=1 << 26)]
    for kw in bad:
        assert call(**kw) < 0, kw
        assert b"chitu_b200_mla_attn_fp8kv" in lib.chitu_b200_last_error(), kw
    before = _lib.launch_count()
    assert call(B=0) == 0 and call(B=0, sq=1) == 0
    assert _lib.launch_count() == before


def test_mla_attn_fp8kv_python_refusals():
    be = _backend()
    c = to_fp8_case(make_case(1, 2, 16, [10], True, device="cpu"))
    with pytest.raises(RuntimeError):
        _call(be, c)                                                            # CPU tensors
    if not torch.cuda.is_available():
        return
    g = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()}
    for bad in (dict(q_nope=g["q_nope"].to(F8)), dict(q_pe=g["q_pe"].to(F8)), dict(kv=quant(g["kv"]))):
        with pytest.raises(RuntimeError):
            _call(be, {**g, **bad})
    for kw in (dict(window_size=(16, 0)), dict(softcap=30.0)):
        with pytest.raises(RuntimeError):
            _call(be, g, **kw)


def test_store_rule_clamps_instead_of_nan():
    x = torch.tensor([470.0, 500.0, -1000.0, 1.0e9, float("nan"), 0.0013, -3.3], dtype=torch.bfloat16)
    q = quant(x).float()
    assert q[:4].tolist() == [448.0, 448.0, -448.0, 448.0]
    assert torch.isnan(q[4]) and q[5] > 0 and q[6] < 0
    assert torch.isnan(x[:3].to(F8).float()).all()                           # what plain .to() would store


def test_reference_is_the_bf16_reference_on_the_decoded_cache():
    from oracle.chitu_oracle import mla_attn_with_kvcache
    c = to_fp8_case(make_case(3, 1, 16, [5, 300, 64], True, seed=1, device="cpu"), scale_rows=600.0)
    got, stored = ref_fp8(c["q_nope"], c["q_pe"], c["kv_cache"], c["kv"], c["seq_excl"], c["block_table"], True, SCALE)
    dec = c["kv_cache"].float().bfloat16()
    kvq = quant(c["kv"]).float().bfloat16()
    want = mla_attn_with_kvcache(c["q_nope"][:, 0], c["q_pe"][:, 0], dec.clone(), kvq, c["seq_excl"],
                                 c["block_table"], SCALE)
    torch.testing.assert_close(got[:, 0].to(want.dtype), want)
    for b in range(3):                                                          # the appended rows: quant(new row)
        p = int(c["seq_excl"][b])
        row = stored[c["block_table"][b, p // PAGE].long(), p % PAGE]
        assert _same_bits(row, quant(c["kv"][b, 0]))
        assert (row.float().abs() <= 448).all()


# ---------------------------------------------------------------- H100

gpu = pytest.mark.gpu

LENS = {1: [0, 1, 63, 64, 65, 1000], 2: [0, 5, 62, 128, 700], 4: [3, 64, 191, 333]}


@gpu
@pytest.mark.parametrize("H", [8, 16, 20, 128])
@pytest.mark.parametrize("sq", [1, 2, 4, 512])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("append", [True, False])
def test_parity_and_stored_bytes(H, sq, causal, append):
    if sq == 512 and H > 16:
        pytest.skip("the 512-token chunk is checked at H <= 16 (reference cost)")
    lens = LENS.get(sq, [0, 100, 1500])
    if not append:
        lens = [max(L, 1) for L in lens]
    B = len(lens)
    c = to_fp8_case(make_case(B, sq, H, lens, append, seed=H * 7 + sq), scale_rows=8.0)
    if append:                                     # values past +-448 and a NaN in request 0's first new row
        c["kv"].view(-1)[:4] = torch.tensor([470.0, 500.0, -1000.0, float("nan")], dtype=torch.bfloat16)
    ref, stored = ref_fp8(c["q_nope"], c["q_pe"], c["kv_cache"], c["kv"], c["seq_excl"], c["block_table"], causal, SCALE)
    be = _backend()
    got = _call(be, c, causal=causal, decode_3d=(sq == 1))
    torch.cuda.synchronize()
    assert got.shape == (B, sq, H, C)
    if append:
        # request 0 attends its NaN row (NaN scores in the reference too): checked through the stored bytes only
        ok = [b for b in range(1, B)]
        check_rows(got[ok], ref[ok], c["seq_excl"][ok], sq, append, causal, f"H={H} sq={sq}")
        assert _same_bits(c["kv_cache"], stored)
    else:
        check_rows(got, ref, c["seq_excl"], sq, append, causal, f"H={H} sq={sq}")


def _bf16_twin(c):
    """The same case on a bf16 cache holding the decoded values, with the new rows pre-rounded to e4m3 values."""
    t = dict(c)
    t["kv_cache"] = c["kv_cache"].float().bfloat16()
    if c["kv"] is not None:
        t["kv"] = quant(c["kv"]).float().bfloat16()
    return t


@gpu
@pytest.mark.parametrize("H", [16, 128])
@pytest.mark.parametrize("sq", [1, 3])
def test_bit_identical_to_bf16_kernels(H, sq):
    lens = [0, 63, 64, 500, 4000]
    c = to_fp8_case(make_case(len(lens), sq, H, lens, True, seed=3), scale_rows=300.0)
    t = _bf16_twin(c)
    for ws in (True, False):
        be = _backend(max_seq_len=4096 + 64)
        cc, tt = {**c, "kv_cache": c["kv_cache"].clone()}, {**t, "kv_cache": t["kv_cache"].clone()}
        if not ws:                                                              # no workspace: one split, direct
            from chitu_b200 import _lib
            from chitu_b200._lib import current_stream, ptr
            lib = _lib.load()
            outs = []
            for case, fn in ((cc, lib.chitu_b200_mla_attn_fp8kv), (tt, None)):
                o = torch.empty(len(lens), sq, H, C, dtype=torch.bfloat16, device="cuda")
                args = (ptr(case["q_nope"]), ptr(case["q_pe"]), ptr(case["kv_cache"]), ptr(case["kv"]),
                        ptr(case["seq_excl"]), ptr(case["block_table"]), case["block_table"].stride(0), len(lens))
                tail = (H, C, R, PAGE, case["kv_cache"].shape[0], 4160)
                if fn is not None:
                    rc = fn(*args, sq, *tail, 1, SCALE, ptr(o), None, 0, current_stream())
                elif sq == 1:
                    rc = lib.chitu_b200_mla_decode(*args, *tail, SCALE, ptr(o), None, 0, current_stream())
                else:
                    rc = lib.chitu_b200_mla_paged_prefill(*args, sq, *tail, 1, SCALE, ptr(o), None, 0, current_stream())
                assert rc == 0
                outs.append(o)
            got, want = outs
        else:
            got, want = _call(be, cc), _call(be, tt)
        torch.cuda.synchronize()
        assert _same_bits(got, want), (H, sq, ws)
        assert _same_bits(cc["kv_cache"].float().bfloat16(), tt["kv_cache"])


@gpu
def test_deferred_merge_bit_identical_through_absorb_o_merge_quant():
    from chitu_b200 import _lib, workspace
    from chitu_b200._lib import current_stream, ptr
    lib = _lib.load()
    B, H, dn, dv = 4, 16, 128, 128
    lens = [10, 700, 2000, 64]
    c = to_fp8_case(make_case(B, 1, H, lens, True, seed=5), scale_rows=100.0)
    t = _bf16_twin(c)
    wkv_b = (torch.randn(H, dn + dv, C, device="cuda") * 0.05).bfloat16()
    hint = 2048 + 64
    res = []
    for case, fp8 in ((c, True), (t, False)):
        ws = torch.zeros(workspace.attn_bytes(B, H, C), dtype=torch.uint8, device="cuda")
        args = (ptr(case["q_nope"]), ptr(case["q_pe"]), ptr(case["kv_cache"]), ptr(case["kv"]), ptr(case["seq_excl"]),
                ptr(case["block_table"]), case["block_table"].stride(0), B)
        tail = (H, C, R, PAGE, case["kv_cache"].shape[0], hint)
        if fp8:
            rc = lib.chitu_b200_mla_attn_fp8kv(*args, 1, *tail, 1, SCALE, None, ptr(ws), ws.numel(), current_stream())
        else:
            rc = lib.chitu_b200_mla_decode(*args, *tail, SCALE, None, ptr(ws), ws.numel(), current_stream())
        assert rc == 0
        x = torch.empty(B, H, C, dtype=torch.bfloat16, device="cuda")
        q = torch.empty(B, H * dv, dtype=F8, device="cuda")
        s = torch.empty(B, H * dv // 128, dtype=torch.float32, device="cuda")
        assert lib.chitu_b200_mla_absorb_o_merge_quant(ptr(ws), ws.numel(), hint, ptr(wkv_b), ptr(x), None, ptr(q),
                                                       ptr(s), B, H, dn, dv, C, current_stream()) == 0
        res.append((x, q, s))
    torch.cuda.synchronize()
    assert lib.chitu_b200_mla_num_splits(B, H, hint, workspace.attn_bytes(B, H, C)) > 1      # the merge is exercised
    for a, b in zip(*res):
        assert _same_bits(a, b)


@gpu
@pytest.mark.parametrize("lens", [[5, 64, 4096, 4100, 130], [8192] * 8, [1, 2, 3]])
def test_device_plan_honoured_bit_identical(lens):
    """prepare_metadata_for_decode's device plan: one split, a remainder split and the largest split counts."""
    B, H = len(lens), 16
    c = to_fp8_case(make_case(B, 1, H, lens, True, seed=7), scale_rows=50.0)
    t = _bf16_twin(c)
    outs = []
    for case in (c, t):
        be = _backend(max_seq_len=8192 + 64, max_reqs=B, n_local_heads=H)
        incl = case["seq_excl"] + 1
        be.prepare_metadata_for_decode(case["seq_excl"], incl, case["block_table"], PAGE)
        outs.append(_call(be, case, decode_3d=True))
    torch.cuda.synchronize()
    assert _same_bits(outs[0], outs[1])
    assert _same_bits(c["kv_cache"].float().bfloat16(), t["kv_cache"])


@gpu
def test_cuda_graph_replay_with_changed_lengths():
    B, H = 3, 16
    c = to_fp8_case(make_case(B, 1, H, [700, 700, 700], True, seed=9), scale_rows=10.0)
    be = _backend(max_seq_len=1024)
    seq = c["seq_excl"].clone()
    cache0 = c["kv_cache"].clone()
    static = {**c, "seq_excl": seq}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _call(be, static, decode_3d=True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = _call(be, static, decode_3d=True)
    for lens in ([10, 64, 699], [0, 300, 640]):
        c["kv_cache"].copy_(cache0)
        seq.copy_(torch.tensor(lens, dtype=torch.int32))
        g.replay()
        torch.cuda.synchronize()
        ref, stored = ref_fp8(c["q_nope"], c["q_pe"], cache0, c["kv"], seq, c["block_table"], True, SCALE)
        check_rows(out, ref, seq, 1, True, True, f"graph {lens}")
        assert _same_bits(c["kv_cache"], stored)


@gpu
@pytest.mark.parametrize("sq", [2, 4])
def test_mtp_verification_equals_successive_decodes(sq):
    B, H = 3, 16
    lens = [3, 62, 1000]
    c = to_fp8_case(make_case(B, sq, H, lens, True, seed=11), scale_rows=20.0)
    be = _backend(max_seq_len=2048)
    multi = {**c, "kv_cache": c["kv_cache"].clone()}
    got = _call(be, multi, causal=True)
    step = {**c, "kv_cache": c["kv_cache"].clone()}
    outs = []
    for i in range(sq):
        d = dict(step, q_nope=c["q_nope"][:, i:i + 1].contiguous(), q_pe=c["q_pe"][:, i:i + 1].contiguous(),
                 kv=c["kv"][:, i].contiguous(), seq_excl=c["seq_excl"] + i)
        outs.append(_call(be, d, decode_3d=True))
    torch.cuda.synchronize()
    assert _same_bits(multi["kv_cache"], step["kv_cache"])
    want = torch.cat(outs, dim=1)
    assert cos_diff(got.float(), want.float()) < 1e-5 and max_rel(got.float(), want.float()) < 1e-2


@gpu
def test_prefill_scatter_stores_by_the_clamp_rule():
    from chitu_b200 import ops
    B = 3
    nb = 8
    cache = torch.full((nb, PAGE, ROW), NAN_E4M3, dtype=torch.uint8, device="cuda").view(F8)
    bt = torch.tensor([[3, 1], [0, 5], [7, 2]], dtype=torch.int32, device="cuda")
    lens = torch.tensor([0, 63, 64], dtype=torch.int32, device="cuda")
    rows = (torch.randn(B, ROW, device="cuda") * 300).bfloat16()
    rows[0, :4] = torch.tensor([470.0, 500.0, -1000.0, float("nan")])
    ops.append_to_paged_kv_cache(cache, bt, rows, lens)
    torch.cuda.synchronize()
    for b in range(B):
        p = int(lens[b])
        got, want = cache[bt[b, p // PAGE].long(), p % PAGE], quant(rows[b])
        nan = torch.isnan(want.float())
        assert torch.equal(torch.isnan(got.float()), nan)                      # NaN stays NaN (either sign byte)
        assert torch.equal(got.view(torch.uint8)[~nan], want.view(torch.uint8)[~nan])


@gpu
def test_deepseek_engine_fp8_cache():
    from chitu_b200.engine_deepseek import DeepSeekConfig, DeepSeekDecodeEngine
    cfg = DeepSeekConfig(vocab_size=1024, dim=512, inter_dim=1024, moe_inter_dim=256, n_layers=2, n_dense_layers=1,
                         n_heads=4, n_routed_experts=16, n_activated_experts=4, n_expert_groups=4, n_limited_groups=2,
                         q_lora_rank=256)
    B, S = 3, 150
    lens = torch.tensor([S, 63, 128], dtype=torch.int32)
    tokens = torch.tensor([5, 17, 900], dtype=torch.int64)
    e8 = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=512, device="cuda:0", tp_size=1, kv_dtype=F8)
    e8.set_synthetic_context(S)
    e8.seq_lens.copy_(lens)
    eb = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=512, device="cuda:0", tp_size=1)
    eb.block_table.copy_(e8.block_table)
    eb.seq_lens.copy_(lens)
    eb.kv_cache.copy_(e8.kv_cache.float().bfloat16())
    eb.decode(tokens.pin_memory())
    e8.decode(tokens.pin_memory())
    torch.cuda.synchronize()
    got, want = e8.logits.float().cpu(), eb.logits.float().cpu()
    assert cos_diff(got, want) < 1e-2 and max_rel(got, want) < 0.15
