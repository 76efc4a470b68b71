"""GQA attention over the paged KV cache with seqlen_q > 1 (chitu_b200_gqa_paged_prefill behind
B200AttnBackend.attn_with_kvcache): argument checks, CPU refusal and the fp32 reference pinned to the oracle without a
GPU; on the H100 per-request parity over NaN-poisoned caches and garbage block-table tails, the bit-exact append, rows
that see no key, strided k / v views, the split path, CUDA-graph replay, speculative verification against step-by-step
decode, and dispatch."""
import math

import pytest
import torch

from conftest import cos_diff, max_rel

D, PAGE = 128, 256


def _backend():
    from chitu_b200.attn_backend import B200AttnBackend
    return B200AttnBackend()


def reference(q, k_cache, v_cache, k, v, cache_seqlens, block_table, causal, scale):
    """flash_attn_with_kvcache in fp32 on copies of the caches: scatter the sq new rows at cache_seqlens[b] + i, then
    attention over Lk keys (bottom-right causal mask; a row that sees no key is 0).  Returns (out, k_cache, v_cache)."""
    kc, vc = k_cache.clone(), v_cache.clone()
    B, sq, Hq, _ = q.shape
    page, Hkv = kc.shape[1], kc.shape[2]
    out = torch.zeros(B, sq, Hq, q.shape[-1], dtype=torch.float32, device=q.device)
    for b in range(B):
        L = int(cache_seqlens[b])
        if k is not None:
            pos = torch.arange(L, L + sq, device=q.device)
            blk = block_table[b, pos // page].long()
            kc[blk, pos % page] = k[b]
            vc[blk, pos % page] = v[b]
            L += sq
        if L == 0:
            continue
        pos = torch.arange(L, device=q.device)
        blk = block_table[b, pos // page].long()
        kk = kc[blk, pos % page].float().repeat_interleave(Hq // Hkv, dim=1)        # [L, Hq, D]
        vv = vc[blk, pos % page].float().repeat_interleave(Hq // Hkv, dim=1)
        s = torch.einsum("ihd,jhd->hij", q[b].float() * scale, kk)
        if causal:
            mask = torch.ones(sq, L, dtype=torch.bool, device=q.device).tril(diagonal=L - sq)
            s = s.masked_fill(~mask, float("-inf"))
        p = torch.softmax(s, dim=-1).nan_to_num(0.0)
        out[b] = torch.einsum("hij,jhd->ihd", p, vv)
    return out, kc, vc


def make_case(B, sq, Hq, Hkv, lens, append, dtype=torch.bfloat16, seed=0, device="cuda", spare=3, page=PAGE):
    """Caches whose unused slots and pages are NaN, a permuted block table whose entries past each request's pages are
    -1, q scaled so the running-max rescale is exercised, and new k / v rows (or None)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    need = [-(-(L + (sq if append else 0)) // page) for L in lens]
    nb = sum(need) + spare
    kc = torch.full((nb, page, Hkv, D), float("nan"), dtype=dtype)
    vc = torch.full((nb, page, Hkv, D), float("nan"), dtype=dtype)
    perm = torch.randperm(nb, generator=g)
    bt = torch.full((B, max(need + [1]) + 2), -1, dtype=torch.int32)
    o = 0
    for b, (L, n) in enumerate(zip(lens, need)):
        bt[b, :n] = perm[o:o + n].int()
        o += n
        pos = torch.arange(L)
        blk = bt[b, pos // page].long()
        kc[blk, pos % page] = torch.randn(L, Hkv, D, generator=g).to(dtype)
        vc[blk, pos % page] = torch.randn(L, Hkv, D, generator=g).to(dtype)
    q = (torch.randn(B, sq, Hq, D, generator=g) * 2.0).to(dtype)
    k = torch.randn(B, sq, Hkv, D, generator=g).to(dtype) if append else None
    v = torch.randn(B, sq, Hkv, D, generator=g).to(dtype) if append else None
    to = (lambda t: None if t is None else t.to(device))
    return dict(q=to(q), k_cache=to(kc), v_cache=to(vc), k=to(k), v=to(v),
                cache_seqlens=torch.tensor(lens, dtype=torch.int32, device=device), block_table=to(bt))


def check_rows(got, ref, cache_seqlens, sq, appended, causal, what):
    for b in range(got.shape[0]):
        g, r = got[b].float(), ref[b]
        assert not torch.isnan(g).any(), f"{what}: NaN in request {b}"
        Lk = int(cache_seqlens[b]) + (sq if appended else 0)
        blind = min(sq, max(0, sq - Lk)) if causal else (sq if Lk == 0 else 0)   # leading rows that see no key
        assert torch.equal(g[:blind], torch.zeros_like(g[:blind])), f"{what}: request {b} rows without keys must be 0"
        if blind < sq:
            cd, mr = cos_diff(g[blind:], r[blind:]), max_rel(g[blind:], r[blind:])
            assert cd < 1e-5 and mr < 1e-2, f"{what}: request {b} cos_diff {cd:.2e} max_rel {mr:.2e}"


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---------------------------------------------------------------- no GPU needed

def test_gqa_paged_prefill_bad_arguments_return_status():
    from chitu_b200 import _lib
    lib = _lib.load()
    A = 16          # a non-null, 16-byte aligned address: every case below is refused before anything is touched

    def call(q=A, kn=None, vn=None, ksb=0, kst=0, B=1, sq=4, Hq=32, Hkv=8, d=D, page=PAGE, dtype=_lib.CB_BF16):
        return lib.chitu_b200_gqa_paged_prefill(q, A, A, kn, vn, ksb, kst, 0, 0, A, A, 4, B, sq, Hq, Hkv, d, page, 8, 0,
                                                1, 0.08, A, None, 0, dtype, None)

    bad = [dict(q=None), dict(sq=0), dict(Hq=30), dict(Hq=32, Hkv=2),        # null, no query token, Hq % Hkv, G = 16
           dict(d=64), dict(page=32), dict(page=100), dict(dtype=_lib.CB_F32),
           dict(q=A + 8),                                                     # base not 16-byte aligned
           dict(kn=A),                                                        # k without v
           dict(kn=A, vn=A, ksb=100), dict(kn=A, vn=A, kst=4)]                # strides not 16-byte multiples
    for kw in bad:
        assert call(**kw) < 0, kw
        assert b"gqa_paged_prefill" in lib.chitu_b200_last_error(), kw
    before = _lib.launch_count()
    assert call(B=0) == 0                                                     # an empty batch launches nothing
    assert _lib.launch_count() == before


def test_attn_with_kvcache_multi_token_refuses_cpu_tensors():
    c = make_case(1, 4, 8, 2, [10], True, device="cpu")
    with pytest.raises(RuntimeError):
        _backend().attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                     block_table=c["block_table"], causal=True)


@pytest.mark.parametrize("append", [True, False])
def test_reference_equals_oracle_decode(append):
    from oracle.chitu_oracle import gqa_paged_decode
    c = make_case(3, 1, 8, 2, [5, 300, 256], append, seed=1, device="cpu")
    got, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], c["block_table"],
                            True, 1.0 / math.sqrt(D))
    ko, vo = c["k_cache"].clone(), c["v_cache"].clone()
    want = gqa_paged_decode(c["q"], ko, vo, c["k"], c["v"], c["cache_seqlens"], c["block_table"])
    torch.testing.assert_close(got.to(want.dtype), want)         # equal up to the one rounding to bf16
    assert _same_bits(kc, ko) and _same_bits(vc, vo)


def test_reference_causal_append_equals_successive_decodes():
    from oracle.chitu_oracle import gqa_paged_decode
    sq = 5
    c = make_case(2, sq, 8, 2, [3, 254], True, seed=2, device="cpu")
    got, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], c["block_table"],
                            True, 1.0 / math.sqrt(D))
    ko, vo = c["k_cache"].clone(), c["v_cache"].clone()
    for i in range(sq):
        step = gqa_paged_decode(c["q"][:, i:i + 1], ko, vo, c["k"][:, i:i + 1], c["v"][:, i:i + 1],
                                c["cache_seqlens"] + i, c["block_table"])
        torch.testing.assert_close(got[:, i:i + 1].to(step.dtype), step)
    assert _same_bits(kc, ko) and _same_bits(vc, vo)


# ---------------------------------------------------------------- H100

CASES = {
    "spec2": (2, [4095, 0, 17]),
    "spec7_ragged": (7, [1, 300, 64, 5000]),
    "prefill64": (64, [0]),
    "prefill2048": (2048, [0]),
    "straddle333": (333, [255, 256, 1000]),
    "prefix512": (512, [8192]),
}


def _run_and_check(Hq, Hkv, case, causal, append, dtype, seed):
    sq, lens = CASES[case]
    c = make_case(len(lens), sq, Hq, Hkv, lens, append, dtype=dtype, seed=seed)
    ref, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], c["block_table"],
                            causal, 1.0 / math.sqrt(D))
    seqlens = c["cache_seqlens"].clone()
    got = _backend().attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                       block_table=c["block_table"], causal=causal)
    torch.cuda.synchronize()
    assert got.shape == c["q"].shape and got.dtype == dtype
    assert torch.equal(c["cache_seqlens"], seqlens)
    assert _same_bits(c["k_cache"], kc) and _same_bits(c["v_cache"], vc), "the cache differs from the reference scatter"
    check_rows(got, ref, seqlens, sq, append, causal, f"{Hq}/{Hkv} {case} causal={causal} append={append} {dtype}")


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [(32, 8), (8, 2), (32, 32), (16, 2), (16, 8)], ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("append", [True, False])
def test_gqa_paged_prefill_parity_bf16(heads, case, causal, append):
    _run_and_check(*heads, case, causal, append, torch.bfloat16,
                   seed=7 * heads[0] + heads[1] + 101 * list(CASES).index(case) + causal + 2 * append)


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [(32, 8), (16, 2)], ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("case", ["spec2", "straddle333", "prefix512"])
@pytest.mark.parametrize("causal", [True, False])
def test_gqa_paged_prefill_parity_fp16(heads, case, causal):
    _run_and_check(*heads, case, causal, True, torch.float16, seed=7)


@pytest.mark.gpu
@pytest.mark.parametrize("page", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
def test_gqa_paged_prefill_small_pages(page, causal):
    sq, lens = 70, [63, 64, 200, 1000]                       # page and tile boundaries fall inside the new rows
    c = make_case(len(lens), sq, 16, 8, lens, True, seed=page + causal, page=page)
    ref, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], c["block_table"],
                            causal, 1.0 / math.sqrt(D))
    got = _backend().attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                       block_table=c["block_table"], causal=causal)
    torch.cuda.synchronize()
    assert _same_bits(c["k_cache"], kc) and _same_bits(c["v_cache"], vc)
    check_rows(got, ref, c["cache_seqlens"], sq, True, causal, f"page {page} causal={causal}")


def _c_call(lib, c, out, ws=None, wsn=0, causal=True, k=None, v=None):
    from chitu_b200 import _lib
    q, kc = c["q"], c["k_cache"]
    B, sq, Hq, _ = q.shape
    k = c["k"] if k is None else k
    v = c["v"] if v is None else v
    st = (k.stride(0), k.stride(1), v.stride(0), v.stride(1)) if k is not None else (0, 0, 0, 0)
    bt = c["block_table"]
    _lib.check(lib.chitu_b200_gqa_paged_prefill(
        q.data_ptr(), kc.data_ptr(), c["v_cache"].data_ptr(), None if k is None else k.data_ptr(),
        None if v is None else v.data_ptr(), *st, c["cache_seqlens"].data_ptr(), bt.data_ptr(), bt.stride(0), B, sq, Hq,
        kc.shape[2], D, PAGE, kc.shape[0], bt.shape[1] * PAGE, int(causal), 1.0 / math.sqrt(D), out.data_ptr(),
        None if ws is None else ws.data_ptr(), 0 if ws is None else wsn, _lib.dtype_code(q.dtype),
        _lib.current_stream()), "gqa_paged_prefill")


@pytest.mark.gpu
def test_gqa_paged_prefill_strided_kv_and_output_sentinels():
    from chitu_b200 import _lib
    lib = _lib.load()
    B, sq, Hq, Hkv, lens = 3, 9, 32, 8, [0, 250, 700]
    c = make_case(B, sq, Hq, Hkv, lens, True, seed=4)
    W = (Hq + 2 * Hkv) * D                                   # a fused qkv GEMM output row
    qkv = torch.full((B, sq, W), float("nan"), dtype=torch.bfloat16, device="cuda")
    qkv[..., Hq * D:(Hq + Hkv) * D] = c["k"].reshape(B, sq, -1)
    qkv[..., (Hq + Hkv) * D:] = c["v"].reshape(B, sq, -1)
    kv_k = qkv[..., Hq * D:(Hq + Hkv) * D].view(B, sq, Hkv, D)
    kv_v = qkv[..., (Hq + Hkv) * D:].view(B, sq, Hkv, D)
    pad, sentinel = 3 * Hq, -7.0
    obuf = torch.full((B * sq * Hq + 2 * pad, D), sentinel, dtype=torch.bfloat16, device="cuda")
    out = obuf[pad:pad + B * sq * Hq]
    ref, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], c["block_table"],
                            True, 1.0 / math.sqrt(D))
    _c_call(lib, c, out, k=kv_k, v=kv_v)
    torch.cuda.synchronize()
    assert torch.all(obuf[:pad] == sentinel) and torch.all(obuf[pad + B * sq * Hq:] == sentinel)
    assert _same_bits(c["k_cache"], kc) and _same_bits(c["v_cache"], vc)
    check_rows(out.view(B, sq, Hq, D), ref, c["cache_seqlens"], sq, True, True, "strided k / v views")


@pytest.mark.gpu
def test_gqa_paged_prefill_split_path():
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    c = make_case(1, 4, 32, 8, [16384], True, seed=5)
    ref, _, _ = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], c["block_table"],
                          True, 1.0 / math.sqrt(D))
    args = (c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"])
    before = _lib.launch_count()
    a = be.attn_with_kvcache(*args, block_table=c["block_table"], causal=True)
    assert _lib.launch_count() == before + 3                  # append, split attention, merge
    b = be.attn_with_kvcache(*args, block_table=c["block_table"], causal=True)
    nosplit = torch.empty_like(c["q"])
    before = _lib.launch_count()
    _c_call(lib, c, nosplit)                                  # workspace NULL: one split
    assert _lib.launch_count() == before + 2
    torch.cuda.synchronize()
    assert _same_bits(a, b), "the split path is not deterministic"
    check_rows(a, ref, c["cache_seqlens"], 4, True, True, "split")
    check_rows(nosplit, ref, c["cache_seqlens"], 4, True, True, "no split")
    cd, mr = cos_diff(a.float(), nosplit.float()), max_rel(a.float(), nosplit.float())
    assert cd < 1e-5 and mr < 1e-2, (cd, mr)


@pytest.mark.gpu
def test_gqa_paged_prefill_cuda_graph_with_changed_lengths():
    be = _backend()
    sq, lens_a, lens_b = 6, [100, 3000], [700, 40]
    c = make_case(2, sq, 32, 8, [max(x, y) for x, y in zip(lens_a, lens_b)], True, seed=6)
    c["cache_seqlens"].copy_(torch.tensor(lens_a, dtype=torch.int32))
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    args = (c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"])
    be.attn_with_kvcache(*args, block_table=c["block_table"], causal=True)          # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = be.attn_with_kvcache(*args, block_table=c["block_table"], causal=True)
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    c["cache_seqlens"].copy_(torch.tensor(lens_b, dtype=torch.int32))
    g.replay()
    torch.cuda.synchronize()
    replay_k, replay_v = c["k_cache"].clone(), c["v_cache"].clone()
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    eager = be.attn_with_kvcache(*args, block_table=c["block_table"], causal=True)
    torch.cuda.synchronize()
    assert _same_bits(out, eager)
    assert _same_bits(replay_k, c["k_cache"]) and _same_bits(replay_v, c["v_cache"])
    ref, _, _ = reference(c["q"], snap_k, snap_v, c["k"], c["v"], c["cache_seqlens"], c["block_table"], True,
                          1.0 / math.sqrt(D))
    check_rows(out, ref, c["cache_seqlens"], sq, True, True, "graph replay")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [2, 4, 8])
def test_speculative_verification_equals_autoregressive_decode(sq):
    be = _backend()
    c = make_case(4, sq, 32, 8, [0, 255, 1024, 4000], True, seed=8 + sq)
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    verify = be.attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                  block_table=c["block_table"], causal=True)
    ver_k, ver_v = c["k_cache"].clone(), c["v_cache"].clone()
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    steps = [be.attn_with_kvcache(c["q"][:, i:i + 1].contiguous(), c["k_cache"], c["v_cache"], c["k"][:, i:i + 1],
                                  c["v"][:, i:i + 1], c["cache_seqlens"] + i, block_table=c["block_table"], causal=True)
             for i in range(sq)]
    torch.cuda.synchronize()
    auto = torch.cat(steps, dim=1)
    assert _same_bits(ver_k, c["k_cache"]) and _same_bits(ver_v, c["v_cache"])
    for b in range(4):
        cd, mr = cos_diff(verify[b].float(), auto[b].float()), max_rel(verify[b].float(), auto[b].float())
        assert cd < 1e-5 and mr < 1e-2, (b, cd, mr)


def _entries(lib, fn):
    buf = torch.zeros(2 + 64, dtype=torch.int64, device="cuda")
    buf[1] = 64
    lib.chitu_b200_debug_timeline(buf.data_ptr())
    try:
        fn()
        torch.cuda.synchronize()
        return lib.chitu_b200_debug_timeline_names().decode().split("\n")[:-1]
    finally:
        lib.chitu_b200_debug_timeline(None)


@pytest.mark.gpu
def test_attn_with_kvcache_dispatch():
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    c = make_case(2, 1, 32, 8, [100, 5000], True, seed=9)
    q, kc, vc, k, v, cs, bt = (c[n] for n in ("q", "k_cache", "v_cache", "k", "v", "cache_seqlens", "block_table"))
    ws, wsn = be._ws(2, 32, D, q.device)
    direct_out = torch.empty_like(q)

    def direct():
        _lib.check(lib.chitu_b200_gqa_paged_decode(
            q.data_ptr(), kc.data_ptr(), vc.data_ptr(), k.data_ptr(), v.data_ptr(), k.stride(0), v.stride(0),
            cs.data_ptr(), bt.data_ptr(), bt.stride(0), 2, 32, 8, D, PAGE, bt.shape[1] * PAGE, 1.0 / math.sqrt(D),
            direct_out.data_ptr(), ws.data_ptr(), wsn, _lib.dtype_code(q.dtype), _lib.current_stream()), "decode")

    holder = {}
    via_backend = _entries(lib, lambda: holder.setdefault("o", be.attn_with_kvcache(q, kc, vc, k, v, cs,
                                                                                     block_table=bt, causal=True)))
    via_c = _entries(lib, direct)
    assert via_backend == via_c and len(via_c) >= 1
    assert _same_bits(holder["o"], direct_out)
    m = make_case(2, 3, 32, 8, [100, 5000], True, seed=10)
    multi = _entries(lib, lambda: be.attn_with_kvcache(m["q"], m["k_cache"], m["v_cache"], m["k"], m["v"],
                                                       m["cache_seqlens"], block_table=m["block_table"], causal=True))
    assert multi and all("gqa_paged_prefill" in n for n in multi)
