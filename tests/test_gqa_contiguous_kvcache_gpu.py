"""GQA attention over the NON-paged KV cache (chitu_b200_gqa_contiguous_attn behind
B200AttnBackend.attn_with_kvcache(block_table=None)), seqlen_q == 1 and > 1: argument checks, CPU refusal and the fp32
reference pinned to the oracle without a GPU; on the H100 the real reference's golden, per-request parity over
NaN-poisoned caches of any length, strided cache / k / v views and output sentinels, the capacity guard, bit-identity
with the paged path on the same data, the split path, CUDA-graph replay, speculative verification against step-by-step
decode, and dispatch."""
import math

import pytest
import torch

from conftest import Golden, cos_diff, max_rel

D = 128


def _backend():
    from chitu_b200.attn_backend import B200AttnBackend
    return B200AttnBackend()


def reference(q, k_cache, v_cache, k, v, cache_seqlens, causal, scale):
    """flash_attn_with_kvcache without a block table, in fp32 on copies of the caches: write the sq new rows at
    cache_seqlens[b] + i of cache row b, then attention over Lk keys (bottom-right causal mask; a row that sees no key is
    0).  Returns (out, k_cache, v_cache)."""
    kc, vc = k_cache.clone(), v_cache.clone()
    B, sq, Hq, _ = q.shape
    S, G = kc.shape[1], Hq // kc.shape[2]
    out = torch.zeros(B, sq, Hq, q.shape[-1], dtype=torch.float32, device=q.device)
    for b in range(B):
        L = int(cache_seqlens[b])
        if k is not None:
            n = max(0, min(sq, S - L))                      # rows at or past S are not written
            kc[b, L:L + n] = k[b, :n]
            vc[b, L:L + n] = v[b, :n]
            L += sq
        if L == 0:
            continue
        kk = kc[b, :L].float().repeat_interleave(G, dim=1)                       # [L, Hq, D]
        vv = vc[b, :L].float().repeat_interleave(G, dim=1)
        s = torch.einsum("ihd,jhd->hij", q[b].float() * scale, kk)
        if causal:
            mask = torch.ones(sq, L, dtype=torch.bool, device=q.device).tril(diagonal=L - sq)
            s = s.masked_fill(~mask, float("-inf"))
        p = torch.softmax(s, dim=-1).nan_to_num(0.0)
        out[b] = torch.einsum("hij,jhd->ihd", p, vv)
    return out, kc, vc


def make_case(B, sq, Hq, Hkv, S, lens, append, dtype=torch.bfloat16, seed=0, device="cuda", d=D):
    """[B, S, Hkv, d] caches whose rows at and past each request's length are NaN, q scaled so the running-max rescale
    is exercised, and new k / v rows (or None)."""
    g = torch.Generator(device=device).manual_seed(seed)
    kc = torch.full((B, S, Hkv, d), float("nan"), dtype=dtype, device=device)
    vc = torch.full((B, S, Hkv, d), float("nan"), dtype=dtype, device=device)
    for b, L in enumerate(lens):
        kc[b, :L] = torch.randn(L, Hkv, d, generator=g, device=device).to(dtype)
        vc[b, :L] = torch.randn(L, Hkv, d, generator=g, device=device).to(dtype)
    q = (torch.randn(B, sq, Hq, d, generator=g, device=device) * 2.0).to(dtype)
    k = torch.randn(B, sq, Hkv, d, generator=g, device=device).to(dtype) if append else None
    v = torch.randn(B, sq, Hkv, d, generator=g, device=device).to(dtype) if append else None
    return dict(q=q, k_cache=kc, v_cache=vc, k=k, v=v, cache_seqlens=torch.tensor(lens, dtype=torch.int32, device=device))


def check_rows(got, ref, cache_seqlens, sq, appended, causal, what, requests=None):
    for b in (range(got.shape[0]) if requests is None else requests):
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


def _call(c, causal=True, **kw):
    return _backend().attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                        causal=causal, **kw)


# ---------------------------------------------------------------- no GPU needed

def test_gqa_contiguous_attn_bad_arguments_return_status():
    from chitu_b200 import _lib
    lib = _lib.load()
    A = 16          # a non-null, 16-byte aligned address: every case below is refused before anything is touched
    S, Hkv = 300, 8

    def call(q=A, kn=None, vn=None, ksb=0, kst=0, csb=S * Hkv * D, rows=S, B=1, sq=4, Hq=32, hkv=Hkv, d=D,
             dtype=_lib.CB_BF16):
        return lib.chitu_b200_gqa_contiguous_attn(q, A, A, csb, rows, kn, vn, ksb, kst, 0, 0, A, B, sq, Hq, hkv, d, 0, 1,
                                                  0.08, A, None, 0, dtype, None)

    bad = [dict(q=None), dict(sq=0), dict(Hq=30), dict(Hq=32, hkv=2),          # null, no query token, Hq % Hkv, G = 16
           dict(d=96, csb=S * Hkv * 96), dict(d=64, csb=S * Hkv * 64),       # head dims: 96, and 64 with sq > 1
           dict(dtype=_lib.CB_F32),
           dict(csb=S * Hkv * D - Hkv * D),                                   # batch stride below S rows
           dict(csb=S * Hkv * D + 8), dict(csb=S * Hkv * D + 4),              # not whole rows; not a multiple of 8
           dict(rows=0),
           dict(q=A + 8),                                                     # base not 16-byte aligned
           dict(kn=A),                                                        # k without v
           dict(kn=A, vn=A, ksb=100), dict(kn=A, vn=A, kst=4)]                # strides not 16-byte multiples
    for kw in bad:
        assert call(**kw) < 0, kw
        assert b"gqa_contiguous_attn" in lib.chitu_b200_last_error(), kw
    before = _lib.launch_count()
    assert call(B=0) == 0                                                     # an empty batch launches nothing
    assert _lib.launch_count() == before


def test_attn_with_kvcache_contiguous_refuses_cpu_tensors():
    for sq in (1, 4):
        c = make_case(1, sq, 8, 2, 64, [10], True, device="cpu")
        with pytest.raises(RuntimeError):
            _call(c)


def _identity_pages(kc, page):
    """The [B, S, Hkv, D] cache as S / page pages per request and the identity block table."""
    B, S = kc.shape[:2]
    n = S // page
    return kc.reshape(B * n, page, *kc.shape[2:]), torch.arange(B * n, dtype=torch.int32).view(B, n)


@pytest.mark.parametrize("append", [True, False])
def test_reference_equals_oracle_decode(append):
    from oracle.chitu_oracle import gqa_paged_decode
    c = make_case(3, 1, 8, 2, 300, [5, 299, 256], append, seed=1, device="cpu")
    got, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], True,
                            1.0 / math.sqrt(D))
    ko, vo = c["k_cache"].clone(), c["v_cache"].clone()
    kp, table = _identity_pages(ko, 100)
    vp, _ = _identity_pages(vo, 100)
    want = gqa_paged_decode(c["q"], kp, vp, c["k"], c["v"], c["cache_seqlens"], table)
    torch.testing.assert_close(got.to(want.dtype), want)         # equal up to the one rounding to bf16
    assert _same_bits(kc, ko) and _same_bits(vc, vo)


def test_reference_causal_append_equals_successive_decodes():
    from oracle.chitu_oracle import gqa_paged_decode
    sq = 5
    c = make_case(2, sq, 8, 2, 300, [3, 254], True, seed=2, device="cpu")
    got, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], True,
                            1.0 / math.sqrt(D))
    ko, vo = c["k_cache"].clone(), c["v_cache"].clone()
    kp, table = _identity_pages(ko, 100)
    vp, _ = _identity_pages(vo, 100)
    for i in range(sq):
        step = gqa_paged_decode(c["q"][:, i:i + 1], kp, vp, c["k"][:, i:i + 1], c["v"][:, i:i + 1],
                                c["cache_seqlens"] + i, table)
        torch.testing.assert_close(got[:, i:i + 1].to(step.dtype), step)
    assert _same_bits(kc, ko) and _same_bits(vc, vo)


# ---------------------------------------------------------------- H100

@pytest.mark.gpu
def test_ref_attn_gqa_golden_without_block_table():
    g = Golden("ref_attn_gqa")                        # RefAttnBackend on contiguous [3, 300, 2, 128] caches
    kc, vc = g.t("k_cache", torch.bfloat16).cuda(), g.t("v_cache", torch.bfloat16).cuda()
    out = _backend().attn_with_kvcache(g.t("q", torch.bfloat16).cuda(), kc, vc, g.t("k", torch.bfloat16).cuda(),
                                       g.t("v", torch.bfloat16).cuda(), cache_seqlens=g.t("lens").cuda())
    torch.cuda.synchronize()
    assert torch.equal(kc.cpu(), g.t("k_cache_after", torch.bfloat16))
    assert torch.equal(vc.cpu(), g.t("v_cache_after", torch.bfloat16))
    ref = g.t("out", torch.bfloat16).float()
    assert cos_diff(out.cpu().float(), ref) < 1e-5 and max_rel(out.cpu().float(), ref) < 1e-2


# (sq, S, lengths): empty, inside the first tile, tile boundaries, the capacity boundary (L + sq == S), long
CASES = {
    "decode300": (1, 300, [0, 5, 64, 299]),
    "decode10240": (1, 10240, [10239, 4096, 17]),
    "spec2_4097": (2, 4097, [4095, 0, 17]),
    "spec7_300": (7, 300, [1, 293, 64]),
    "prefill64_300": (64, 300, [0, 236]),
    "straddle333_4097": (333, 4097, [255, 3764, 1000]),
    "prefill2048_4097": (2048, 4097, [0, 2049]),
    "prefix512_10240": (512, 10240, [8192, 9728]),
}


def _run_and_check(Hq, Hkv, case, causal, append, dtype, seed, d=D):
    sq, S, lens = CASES[case]
    c = make_case(len(lens), sq, Hq, Hkv, S, lens, append, dtype=dtype, seed=seed, d=d)
    ref, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], causal,
                            1.0 / math.sqrt(d))
    seqlens = c["cache_seqlens"].clone()
    got = _call(c, causal=causal)
    torch.cuda.synchronize()
    assert got.shape == c["q"].shape and got.dtype == dtype
    assert torch.equal(c["cache_seqlens"], seqlens)
    assert _same_bits(c["k_cache"], kc) and _same_bits(c["v_cache"], vc), "the cache differs from the reference write"
    check_rows(got, ref, seqlens, sq, append, causal, f"{Hq}/{Hkv} {case} causal={causal} append={append} {dtype}")


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [(32, 8), (8, 2), (32, 32), (16, 2), (16, 8)], ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("append", [True, False])
def test_gqa_contiguous_parity_bf16(heads, case, causal, append):
    _run_and_check(*heads, case, causal, append, torch.bfloat16,
                   seed=7 * heads[0] + heads[1] + 101 * list(CASES).index(case) + causal + 2 * append)


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [(32, 8), (16, 2)], ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("case", ["decode300", "spec2_4097", "straddle333_4097", "prefix512_10240"])
@pytest.mark.parametrize("causal", [True, False])
def test_gqa_contiguous_parity_fp16(heads, case, causal):
    _run_and_check(*heads, case, causal, True, torch.float16, seed=7)


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [(8, 2), (32, 8), (16, 16)], ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("case", ["decode300", "decode10240"])
@pytest.mark.parametrize("append", [True, False])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_gqa_contiguous_decode_head_dim_64(heads, case, append, dtype):
    _run_and_check(*heads, case, True, append, dtype, seed=3 * heads[0] + append, d=64)


def _c_call(lib, c, out, ws=None, wsn=0, causal=True, k=None, v=None, kc=None, vc=None, hint=0):
    from chitu_b200 import _lib
    q = c["q"]
    kc = c["k_cache"] if kc is None else kc
    vc = c["v_cache"] if vc is None else vc
    B, sq, Hq, d = q.shape
    k = c["k"] if k is None else k
    v = c["v"] if v is None else v
    st = (k.stride(0), k.stride(1), v.stride(0), v.stride(1)) if k is not None else (0, 0, 0, 0)
    _lib.check(lib.chitu_b200_gqa_contiguous_attn(
        q.data_ptr(), kc.data_ptr(), vc.data_ptr(), kc.stride(0), kc.shape[1], None if k is None else k.data_ptr(),
        None if v is None else v.data_ptr(), *st, c["cache_seqlens"].data_ptr(), B, sq, Hq, kc.shape[2], d, hint,
        int(causal), 1.0 / math.sqrt(d), out.data_ptr(), None if ws is None else ws.data_ptr(),
        0 if ws is None else wsn, _lib.dtype_code(q.dtype), _lib.current_stream()), "gqa_contiguous_attn")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [1, 9])
def test_gqa_contiguous_strided_views_and_sentinels(sq):
    B, Hq, Hkv, S, lens = 3, 32, 8, 1000, [0, 250, 700]
    c = make_case(B, sq, Hq, Hkv, S, lens, True, seed=4 + sq)
    # the cache is a [:B, :S] view of a larger NaN-filled buffer: one more request, 40 more positions
    kbuf = torch.full((B + 1, S + 40, Hkv, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    vbuf = torch.full_like(kbuf, float("nan"))
    kbuf[:B, :S] = c["k_cache"]
    vbuf[:B, :S] = c["v_cache"]
    kview, vview = kbuf[:B, :S], vbuf[:B, :S]
    W = (Hq + 2 * Hkv) * D                                   # a fused qkv GEMM output row
    qkv = torch.full((B, sq, W), float("nan"), dtype=torch.bfloat16, device="cuda")
    qkv[..., Hq * D:(Hq + Hkv) * D] = c["k"].reshape(B, sq, -1)
    qkv[..., (Hq + Hkv) * D:] = c["v"].reshape(B, sq, -1)
    kv_k = qkv[..., Hq * D:(Hq + Hkv) * D].view(B, sq, Hkv, D)
    kv_v = qkv[..., (Hq + Hkv) * D:].view(B, sq, Hkv, D)
    pad, sentinel = 3 * Hq, -7.0
    obuf = torch.full((B * sq * Hq + 2 * pad, D), sentinel, dtype=torch.bfloat16, device="cuda")
    out = obuf[pad:pad + B * sq * Hq]
    ref, kc, vc = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], True,
                            1.0 / math.sqrt(D))
    want_k, want_v = kbuf.clone(), vbuf.clone()
    want_k[:B, :S], want_v[:B, :S] = kc, vc                  # only the written positions of the view change
    from chitu_b200 import _lib
    be = _backend()
    ws, wsn = be._ws(B, Hq, D, c["q"].device)
    _c_call(_lib.load(), c, out, ws=ws, wsn=wsn, k=kv_k, v=kv_v, kc=kview, vc=vview)
    torch.cuda.synchronize()
    assert torch.all(obuf[:pad] == sentinel) and torch.all(obuf[pad + B * sq * Hq:] == sentinel)
    assert _same_bits(kbuf, want_k) and _same_bits(vbuf, want_v)
    check_rows(out.view(B, sq, Hq, D), ref, c["cache_seqlens"], sq, True, True, "strided views")
    # the backend accepts the same views
    kbuf[:B, :S], vbuf[:B, :S] = c["k_cache"], c["v_cache"]
    got = be.attn_with_kvcache(c["q"], kview, vview, kv_k, kv_v, c["cache_seqlens"], causal=True)
    torch.cuda.synchronize()
    assert _same_bits(got, out.view(B, sq, Hq, D))
    assert _same_bits(kbuf, want_k) and _same_bits(vbuf, want_v)


@pytest.mark.gpu
@pytest.mark.parametrize("sq,over", [(4, [-2]), (1, [0, 3])], ids=["sq4", "sq1"])
def test_gqa_contiguous_capacity_guard(sq, over):
    """A request whose new rows run past the cache's S rows: rows >= S are not written (they are sentinel rows of the
    same allocation here), and the other requests' rows and outputs are those of the reference."""
    B, Hq, Hkv, S, extra = 3, 32, 8, 512, 16
    for o in over:
        lens = [100, S + o, 37]
        ok = [0, 2]
        c = make_case(B, sq, Hq, Hkv, S, [min(L, S) for L in lens], True, seed=11 + sq)
        c["cache_seqlens"].copy_(torch.tensor(lens, dtype=torch.int32))
        sentinel = -3.0
        kbuf = torch.full((B, S + extra, Hkv, D), sentinel, dtype=torch.bfloat16, device="cuda")
        vbuf = torch.full_like(kbuf, sentinel)
        kbuf[:, :S], vbuf[:, :S] = c["k_cache"], c["v_cache"]
        want_k, want_v = kbuf.clone(), vbuf.clone()
        for b in ok:
            want_k[b, lens[b]:lens[b] + sq] = c["k"][b]
            want_v[b, lens[b]:lens[b] + sq] = c["v"][b]
        bad = lens[1]
        for i in range(sq):
            if bad + i < S:                                   # in-capacity rows of the overflowing request
                want_k[1, bad + i], want_v[1, bad + i] = c["k"][1, i], c["v"][1, i]
        pad, osent = 2 * Hq, 5.0
        obuf = torch.full((B * sq * Hq + 2 * pad, D), osent, dtype=torch.bfloat16, device="cuda")
        out = obuf[pad:pad + B * sq * Hq]
        ref_lens = c["cache_seqlens"].clone()
        ref_lens[1] = 0                                       # the overflowing request's output is unspecified
        ref, _, _ = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], ref_lens, True, 1.0 / math.sqrt(D))
        from chitu_b200 import _lib
        ws, wsn = _backend()._ws(B, Hq, D, c["q"].device)
        _c_call(_lib.load(), c, out, ws=ws, wsn=wsn, kc=kbuf[:, :S], vc=vbuf[:, :S])
        torch.cuda.synchronize()
        assert _same_bits(kbuf, want_k) and _same_bits(vbuf, want_v), f"length S{o:+d}: rows outside the cache changed"
        assert torch.all(obuf[:pad] == osent) and torch.all(obuf[pad + B * sq * Hq:] == osent)
        check_rows(out.view(B, sq, Hq, D), ref, c["cache_seqlens"], sq, True, True, f"capacity S{o:+d}", requests=ok)


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [1, 4, 512])
def test_gqa_contiguous_bit_identical_to_paged(sq):
    """The same data stored in 256-token pages (identity block table over the same memory), S = 4096, the same hint and
    so the same split count: outputs and caches are bit-identical to the paged kernels'."""
    B, Hq, Hkv, S, page = 3, 32, 8, 4096, 256
    lens = [0, 1000, S - sq - 300]
    c = make_case(B, sq, Hq, Hkv, S, lens, True, seed=20 + sq)
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    be = _backend()
    contig = _call(c)
    ck, cv = c["k_cache"].clone(), c["v_cache"].clone()
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    kp = c["k_cache"].view(B * (S // page), page, Hkv, D)
    vp = c["v_cache"].view(B * (S // page), page, Hkv, D)
    table = torch.arange(B * (S // page), dtype=torch.int32, device="cuda").view(B, S // page)
    paged = be.attn_with_kvcache(c["q"], kp, vp, c["k"], c["v"], c["cache_seqlens"], block_table=table, causal=True)
    torch.cuda.synchronize()
    assert _same_bits(contig, paged)
    assert _same_bits(ck, c["k_cache"]) and _same_bits(cv, c["v_cache"])


@pytest.mark.gpu
@pytest.mark.parametrize("sq,launches", [(4, 3), (1, 2)])
def test_gqa_contiguous_split_path(sq, launches):
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    c = make_case(1, sq, 32, 8, 16384, [16384 - sq - 5], True, seed=5)
    ref, _, _ = reference(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"], True,
                          1.0 / math.sqrt(D))
    args = (c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"])
    before = _lib.launch_count()
    a = be.attn_with_kvcache(*args, causal=True)
    assert _lib.launch_count() == before + launches           # (append,) split attention, merge
    b = be.attn_with_kvcache(*args, causal=True)
    nosplit = torch.empty_like(c["q"])
    before = _lib.launch_count()
    _c_call(lib, c, nosplit)                                  # workspace NULL: one split
    assert _lib.launch_count() == before + launches - 1
    torch.cuda.synchronize()
    assert _same_bits(a, b), "the split path is not deterministic"
    check_rows(a, ref, c["cache_seqlens"], sq, True, True, "split")
    check_rows(nosplit, ref, c["cache_seqlens"], sq, True, True, "no split")
    cd, mr = cos_diff(a.float(), nosplit.float()), max_rel(a.float(), nosplit.float())
    assert cd < 1e-5 and mr < 1e-2, (cd, mr)


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [1, 6])
def test_gqa_contiguous_cuda_graph_with_changed_lengths(sq):
    be = _backend()
    lens_a, lens_b = [100, 3000], [700, 40]
    c = make_case(2, sq, 32, 8, 4096, [max(x, y) for x, y in zip(lens_a, lens_b)], True, seed=6)
    c["cache_seqlens"].copy_(torch.tensor(lens_a, dtype=torch.int32))
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    args = (c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"])
    be.attn_with_kvcache(*args, causal=True)                  # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = be.attn_with_kvcache(*args, causal=True)
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    c["cache_seqlens"].copy_(torch.tensor(lens_b, dtype=torch.int32))
    g.replay()
    torch.cuda.synchronize()
    replay_k, replay_v = c["k_cache"].clone(), c["v_cache"].clone()
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    eager = be.attn_with_kvcache(*args, causal=True)
    torch.cuda.synchronize()
    assert _same_bits(out, eager)
    assert _same_bits(replay_k, c["k_cache"]) and _same_bits(replay_v, c["v_cache"])
    ref, _, _ = reference(c["q"], snap_k, snap_v, c["k"], c["v"], c["cache_seqlens"], True, 1.0 / math.sqrt(D))
    check_rows(out, ref, c["cache_seqlens"], sq, True, True, "graph replay")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [2, 4, 8])
def test_speculative_verification_equals_autoregressive_decode(sq):
    be = _backend()
    c = make_case(4, sq, 32, 8, 4100, [0, 255, 1024, 4000], True, seed=8 + sq)
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    verify = _call(c)
    ver_k, ver_v = c["k_cache"].clone(), c["v_cache"].clone()
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    steps = [be.attn_with_kvcache(c["q"][:, i:i + 1].contiguous(), c["k_cache"], c["v_cache"], c["k"][:, i:i + 1],
                                  c["v"][:, i:i + 1], c["cache_seqlens"] + i, causal=True)
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
def test_attn_with_kvcache_contiguous_dispatch():
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    for sq in (1, 3):
        c = make_case(2, sq, 32, 8, 5100, [100, 5000], True, seed=9 + sq)
        contig = _entries(lib, lambda: _call(c))
        assert contig and all("gqa_contiguous" in n for n in contig), contig
        kp = torch.zeros(2 * 20, 256, 8, D, dtype=torch.bfloat16, device="cuda")
        vp = torch.zeros_like(kp)
        table = torch.arange(40, dtype=torch.int32, device="cuda").view(2, 20)
        paged = _entries(lib, lambda: be.attn_with_kvcache(c["q"], kp, vp, c["k"], c["v"], c["cache_seqlens"],
                                                           block_table=table, causal=True))
        name = "gqa_paged_decode" if sq == 1 else "gqa_paged_prefill"
        assert paged and all(name in n for n in paged), paged
