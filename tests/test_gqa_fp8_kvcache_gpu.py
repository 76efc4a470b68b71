"""GQA attention over an fp8 (e4m3fn) paged KV cache (chitu_b200_gqa_paged_attn_fp8kv behind
B200AttnBackend.attn_with_kvcache): argument checks, the Python refusals and the fp32 reference pinned to the oracle
without a GPU; on the H100 parity over NaN-poisoned caches and -1 block-table tails for sq = 1 and sq > 1, the stored
bytes (with and without fused rotary), bit-identity with the bf16 / fp16 kernels on a cache holding the decoded values,
the split path, CUDA-graph replay, verification against successive decodes, dispatch and the LLaMA engine."""
import math

import pytest
import torch

from conftest import cos_diff, max_rel
from test_gqa_paged_prefill_gpu import check_rows, reference

D, PAGE = 128, 256
E4M3 = torch.float8_e4m3fn
NAN8 = 0x7F                      # e4m3fn NaN


def _backend():
    from chitu_b200.attn_backend import B200AttnBackend
    return B200AttnBackend()


def quant(x):
    """The stored form of a new k / v row."""
    return x.float().clamp(-448.0, 448.0).to(E4M3)


def reference_fp8(q, k_cache, v_cache, k, v, cache_seqlens, block_table, causal, scale):
    """The fp32 reference over e4m3 caches: decode the caches, append the stored form of the new rows, then the
    arithmetic of the io-dtype reference.  Returns (out, k_cache, v_cache) with the caches as e4m3."""
    kq = None if k is None else quant(k).float()
    vq = None if v is None else quant(v).float()
    out, kc, vc = reference(q.float(), k_cache.float(), v_cache.float(), kq, vq, cache_seqlens, block_table, causal,
                            scale)
    return out, kc.to(E4M3), vc.to(E4M3)


def make_case(B, sq, Hq, Hkv, lens, append, dtype=torch.bfloat16, seed=0, device="cuda", spare=3, page=PAGE,
              big=False):
    """e4m3 caches whose unused slots and pages are NaN, a permuted block table whose entries past each request's
    pages are -1, q scaled so the running-max rescale is exercised, new k / v rows in the io dtype (or None).  The
    cached values span e4m3's subnormals to its largest normals; `big` puts values beyond +-448 into the new rows."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    need = [-(-(L + (sq if append else 0)) // page) for L in lens]
    nb = sum(need) + spare
    kc = torch.full((nb, page, Hkv, D), NAN8, dtype=torch.uint8).view(E4M3)
    vc = torch.full((nb, page, Hkv, D), NAN8, dtype=torch.uint8).view(E4M3)
    perm = torch.randperm(nb, generator=g)
    bt = torch.full((B, max(need + [1]) + 2), -1, dtype=torch.int32)

    def draw(*shape):
        x = torch.randn(*shape, generator=g)
        return x * torch.exp2(torch.randint(-10, 3, shape, generator=g).float())     # subnormals .. large normals

    o = 0
    for b, (L, n) in enumerate(zip(lens, need)):
        bt[b, :n] = perm[o:o + n].int()
        o += n
        pos = torch.arange(L)
        blk = bt[b, pos // page].long()
        kc[blk, pos % page] = quant(draw(L, Hkv, D))
        vc[blk, pos % page] = quant(draw(L, Hkv, D))
    q = (torch.randn(B, sq, Hq, D, generator=g) * 0.5).to(dtype)
    k = v = None
    if append:
        k, v = draw(B, sq, Hkv, D), draw(B, sq, Hkv, D)
        if big:
            k[..., :4] = torch.tensor([500.0, -1000.0, 449.0, 3e4])
            v[..., :4] = torch.tensor([-500.0, 1000.0, -449.0, 464.0])
        k, v = k.to(dtype), v.to(dtype)
    to = (lambda t: None if t is None else t.to(device))
    return dict(q=to(q), k_cache=to(kc), v_cache=to(vc), k=to(k), v=to(v),
                cache_seqlens=torch.tensor(lens, dtype=torch.int32, device=device), block_table=to(bt))


def _bytes(t):
    return t.view(torch.uint8)


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---------------------------------------------------------------- no GPU needed

def test_gqa_paged_attn_fp8kv_bad_arguments_return_status():
    from chitu_b200 import _lib
    lib = _lib.load()
    A = 16          # a non-null, 16-byte aligned address: every case below is refused before anything is touched

    def call(q=A, q_sb=None, kn=None, vn=None, ksb=0, kst=0, cos=None, sin=None, B=1, sq=4, Hq=32, Hkv=8, d=D,
             page=PAGE, dtype=_lib.CB_BF16):
        q_sb = sq * Hq * d if q_sb is None else q_sb
        return lib.chitu_b200_gqa_paged_attn_fp8kv(q, q_sb, A, A, kn, vn, ksb, kst, 0, 0, cos, sin, A, A, 4, B, sq, Hq,
                                                   Hkv, d, page, 8, 0, 1, 0.08, A, None, 0, dtype, None)

    bad = [dict(q=None), dict(sq=0), dict(Hq=30), dict(Hq=24, Hkv=8),              # null, no query, Hq % Hkv, G = 3
           dict(Hq=32, Hkv=2),                                                     # G = 16
           dict(d=64), dict(d=64, sq=1), dict(page=32), dict(page=100), dict(page=192),
           dict(dtype=_lib.CB_F32), dict(dtype=_lib.CB_FP8_E4M3),                  # fp32 io, fp8 io
           dict(q=A + 8), dict(kn=A),                                              # misaligned base, k without v
           dict(kn=A, vn=A, ksb=100), dict(kn=A, vn=A, kst=4),                     # strides not 16-byte multiples
           dict(cos=A, sin=A),                                                     # rotary with sq > 1
           dict(cos=A, sq=1),                                                      # cos without sin
           dict(q_sb=4 * 32 * D + 8),                                              # q not dense for sq > 1
           dict(sq=1, q_sb=32 * D - 8)]                                            # q rows overlap
    for kw in bad:
        assert call(**kw) < 0, kw
        assert b"gqa_paged_attn_fp8kv" in lib.chitu_b200_last_error(), kw
    before = _lib.launch_count()
    assert call(B=0) == 0                                                          # an empty batch launches nothing
    assert _lib.launch_count() == before


def test_attn_with_kvcache_fp8_refusals():
    be = _backend()
    c = make_case(1, 4, 8, 2, [10], True, device="cpu")
    with pytest.raises(RuntimeError):                          # CPU tensors
        be.attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                             block_table=c["block_table"], causal=True)
    with pytest.raises(RuntimeError, match="same dtype"):      # mixed cache dtypes
        be.attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"].to(torch.bfloat16), c["k"], c["v"],
                             c["cache_seqlens"], block_table=c["block_table"], causal=True)
    nonpaged = torch.zeros(1, 64, 2, D, dtype=E4M3)
    with pytest.raises(RuntimeError, match="paged cache only"):   # the non-paged fp8 cache is not built
        be.attn_with_kvcache(c["q"], nonpaged, nonpaged, c["k"], c["v"], c["cache_seqlens"], causal=True)


@pytest.mark.parametrize("append", [True, False])
def test_reference_equals_oracle_decode(append):
    """On e4m3 caches the reference is the oracle's decode over the decoded values, with the stored form appended."""
    from oracle.chitu_oracle import gqa_paged_decode
    c = make_case(3, 1, 8, 2, [5, 300, 256], append, seed=1, device="cpu")
    got, kc, vc = reference_fp8(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                c["block_table"], True, 1.0 / math.sqrt(D))
    ko, vo = c["k_cache"].to(torch.bfloat16), c["v_cache"].to(torch.bfloat16)
    kn = None if c["k"] is None else quant(c["k"]).to(torch.bfloat16)
    vn = None if c["v"] is None else quant(c["v"]).to(torch.bfloat16)
    want = gqa_paged_decode(c["q"], ko, vo, kn, vn, c["cache_seqlens"], c["block_table"])
    torch.testing.assert_close(got.to(want.dtype), want)         # equal up to the one rounding to bf16
    assert torch.equal(_bytes(kc), _bytes(ko.to(E4M3))) and torch.equal(_bytes(vc), _bytes(vo.to(E4M3)))


def test_reference_causal_append_equals_successive_decodes():
    from oracle.chitu_oracle import gqa_paged_decode
    sq = 5
    c = make_case(2, sq, 8, 2, [3, 254], True, seed=2, device="cpu")
    got, kc, _ = reference_fp8(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                               c["block_table"], True, 1.0 / math.sqrt(D))
    ko, vo = c["k_cache"].to(torch.bfloat16), c["v_cache"].to(torch.bfloat16)
    kn, vn = quant(c["k"]).to(torch.bfloat16), quant(c["v"]).to(torch.bfloat16)
    for i in range(sq):
        step = gqa_paged_decode(c["q"][:, i:i + 1], ko, vo, kn[:, i:i + 1], vn[:, i:i + 1], c["cache_seqlens"] + i,
                                c["block_table"])
        torch.testing.assert_close(got[:, i:i + 1].to(step.dtype), step)
    assert torch.equal(_bytes(kc), _bytes(ko.to(E4M3)))


# ---------------------------------------------------------------- H100

def _run(c, causal):
    return _backend().attn_with_kvcache(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                        block_table=c["block_table"], causal=causal)


def _run_and_check(Hq, Hkv, sq, prefix, causal, append, dtype, seed):
    lens = [prefix, prefix + 77] if sq <= 8 else [prefix]
    c = make_case(len(lens), sq, Hq, Hkv, lens, append, dtype=dtype, seed=seed)
    ref, kc, vc = reference_fp8(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                c["block_table"], causal, 1.0 / math.sqrt(D))
    seqlens = c["cache_seqlens"].clone()
    got = _run(c, causal)
    torch.cuda.synchronize()
    assert got.shape == c["q"].shape and got.dtype == dtype
    assert torch.equal(c["cache_seqlens"], seqlens)
    assert torch.equal(_bytes(c["k_cache"]), _bytes(kc)) and torch.equal(_bytes(c["v_cache"]), _bytes(vc)), \
        "the cache differs from the reference scatter"
    check_rows(got, ref, seqlens, sq, append, causal, f"{Hq}/{Hkv} sq={sq} prefix={prefix} causal={causal} "
                                                      f"append={append} {dtype}")


HEADS = [(8, 8), (16, 8), (32, 8), (32, 4)]          # G = 1, 2, 4, 8


@pytest.mark.gpu
@pytest.mark.parametrize("heads", HEADS, ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("sq", [1, 2, 8, 512, 2048])
@pytest.mark.parametrize("prefix", [0, 4096])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("append", [True, False])
def test_fp8_kvcache_parity_bf16(heads, sq, prefix, causal, append):
    if sq == 1 and not causal:
        pytest.skip("one query token: causal and non-causal are the same call")
    _run_and_check(*heads, sq, prefix, causal, append, torch.bfloat16,
                   seed=7 * heads[0] + heads[1] + 13 * sq + prefix + causal + 2 * append)


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [(32, 8), (16, 2)], ids=lambda h: f"{h[0]}x{h[1]}")
@pytest.mark.parametrize("sq", [1, 8, 512])
@pytest.mark.parametrize("causal", [True, False])
def test_fp8_kvcache_parity_fp16(heads, sq, causal):
    _run_and_check(*heads, sq, 4096, causal, True, torch.float16, seed=11 * sq + causal)


@pytest.mark.gpu
@pytest.mark.parametrize("page", [64, 128])
@pytest.mark.parametrize("sq", [1, 70])
def test_fp8_kvcache_small_pages(page, sq):
    lens = [63, 64, 200, 1000]                           # page and tile boundaries fall inside the new rows
    c = make_case(len(lens), sq, 16, 8, lens, True, seed=page + sq, page=page)
    ref, kc, vc = reference_fp8(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                                c["block_table"], True, 1.0 / math.sqrt(D))
    got = _run(c, True)
    torch.cuda.synchronize()
    assert torch.equal(_bytes(c["k_cache"]), _bytes(kc)) and torch.equal(_bytes(c["v_cache"]), _bytes(vc))
    check_rows(got, ref, c["cache_seqlens"], sq, True, True, f"page {page} sq {sq}")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [1, 3])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_fp8_kvcache_appended_bytes_saturate(sq, dtype):
    """The new rows are stored exactly as x.float().clamp(-448, 448).to(float8_e4m3fn), values past 448 included."""
    c = make_case(2, sq, 32, 8, [100, 700], True, dtype=dtype, seed=20 + sq, big=True)
    _run(c, True)
    torch.cuda.synchronize()
    page = c["k_cache"].shape[1]
    for b, L in enumerate(c["cache_seqlens"].tolist()):
        pos = torch.arange(L, L + sq, device="cuda")
        blk = c["block_table"][b, pos // page].long()
        assert torch.equal(_bytes(c["k_cache"][blk, pos % page]), _bytes(quant(c["k"][b])))
        assert torch.equal(_bytes(c["v_cache"][blk, pos % page]), _bytes(quant(c["v"][b])))
    assert (c["k"].float().abs() > 448).any()


def _rope_tables(B, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    ang = torch.rand(B, D // 2, generator=g) * 6.0
    return ang.cos().cuda(), ang.sin().cuda()


def _fp8_call(lib, c, out, q=None, q_sb=None, cos=None, sin=None, ws=None, wsn=0, causal=True, k=None, v=None):
    from chitu_b200 import _lib
    q = c["q"] if q is None else q
    kc = c["k_cache"]
    B, sq, Hq = c["q"].shape[:3]
    k = c["k"] if k is None else k
    v = c["v"] if v is None else v
    st = (k.stride(0), k.stride(1), v.stride(0), v.stride(1)) if k is not None else (0, 0, 0, 0)
    bt = c["block_table"]
    _lib.check(lib.chitu_b200_gqa_paged_attn_fp8kv(
        q.data_ptr(), sq * Hq * D if q_sb is None else q_sb, kc.data_ptr(), c["v_cache"].data_ptr(),
        None if k is None else k.data_ptr(), None if v is None else v.data_ptr(), *st,
        None if cos is None else cos.data_ptr(), None if sin is None else sin.data_ptr(), c["cache_seqlens"].data_ptr(),
        bt.data_ptr(), bt.stride(0), B, sq, Hq, kc.shape[2], D, kc.shape[1], kc.shape[0], bt.shape[1] * kc.shape[1],
        int(causal), 1.0 / math.sqrt(D), out.data_ptr(), None if ws is None else ws.data_ptr(),
        0 if ws is None else wsn, _lib.dtype_code(c["q"].dtype), _lib.current_stream()), "gqa_paged_attn_fp8kv")


@pytest.mark.gpu
def test_fp8_kvcache_fused_rope_matches_rotary_then_append():
    """sq == 1 with fused rotary on views of a fused qkv row: the stored k is the unfused rotary op's output (rounded to
    the io dtype) stored as e4m3, and the output is the reference's over the rotated q and k."""
    from chitu_b200 import _lib
    lib = _lib.load()
    B, Hq, Hkv = 3, 32, 8
    c = make_case(B, 1, Hq, Hkv, [0, 300, 5000], True, seed=30, big=True)
    W = (Hq + 2 * Hkv) * D
    qkv = torch.full((B, W), float("nan"), dtype=torch.bfloat16, device="cuda")
    qkv[:, :Hq * D] = c["q"].reshape(B, -1)
    qkv[:, Hq * D:(Hq + Hkv) * D] = c["k"].reshape(B, -1)
    qkv[:, (Hq + Hkv) * D:] = c["v"].reshape(B, -1)
    qv, kv, vv = qkv[:, :Hq * D], qkv[:, Hq * D:(Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:]
    cos, sin = _rope_tables(B, 31)
    q_rot = torch.empty(B, Hq, D, dtype=torch.bfloat16, device="cuda")              # the unfused rotary op
    k_rot = torch.empty(B, Hkv, D, dtype=torch.bfloat16, device="cuda")
    _lib.check(lib.chitu_b200_rotary_interleaved(qv.data_ptr(), kv.data_ptr(), q_rot.data_ptr(), k_rot.data_ptr(),
                                                 cos.data_ptr(), sin.data_ptr(), B, Hq, Hkv, D, W, D, W, D,
                                                 _lib.CB_BF16, _lib.current_stream()), "rotary")
    ref, kc, vc = reference_fp8(q_rot.view(B, 1, Hq, D), c["k_cache"], c["v_cache"], k_rot.view(B, 1, Hkv, D),
                                c["v"], c["cache_seqlens"], c["block_table"], True, 1.0 / math.sqrt(D))
    out = torch.empty(B, 1, Hq, D, dtype=torch.bfloat16, device="cuda")
    _fp8_call(lib, c, out, q=qv, q_sb=W, cos=cos, sin=sin, k=kv.view(B, 1, Hkv, D), v=vv.view(B, 1, Hkv, D))
    torch.cuda.synchronize()
    assert (k_rot.float().abs() > 448).any()
    assert torch.equal(_bytes(c["k_cache"]), _bytes(kc)) and torch.equal(_bytes(c["v_cache"]), _bytes(vc))
    check_rows(out, ref, c["cache_seqlens"], 1, True, True, "fused rotary")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [1, 2, 8, 512])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("heads", [(32, 8), (8, 8), (32, 4)], ids=lambda h: f"{h[0]}x{h[1]}")
def test_fp8_kvcache_bit_identical_to_io_cache(sq, dtype, heads):
    """Same tiles, splits and arithmetic: over an io-dtype cache holding the decoded values, with e4m3-representable new
    rows, the io-dtype kernels give the same bits."""
    Hq, Hkv = heads
    c = make_case(3, sq, Hq, Hkv, [0, 1000, 4100], True, dtype=dtype, seed=40 + sq)
    c["k"], c["v"] = quant(c["k"]).to(dtype), quant(c["v"]).to(dtype)
    io = dict(c, k_cache=c["k_cache"].to(dtype), v_cache=c["v_cache"].to(dtype))
    got = _run(c, True)
    want = _run(io, True)
    torch.cuda.synchronize()
    assert _same_bits(got, want)
    assert torch.equal(_bytes(c["k_cache"]), _bytes(io["k_cache"].to(E4M3)))
    assert torch.equal(_bytes(c["v_cache"]), _bytes(io["v_cache"].to(E4M3)))


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [1, 4])
def test_fp8_kvcache_split_path(sq):
    from chitu_b200 import _lib
    lib = _lib.load()
    c = make_case(1, sq, 32, 8, [16384], True, seed=5)
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    ref, _, _ = reference_fp8(c["q"], c["k_cache"], c["v_cache"], c["k"], c["v"], c["cache_seqlens"],
                              c["block_table"], True, 1.0 / math.sqrt(D))
    before = _lib.launch_count()
    a = _run(c, True)
    assert _lib.launch_count() == before + (2 if sq == 1 else 3)     # (append,) split attention, merge
    b = _run(c, True)
    nosplit = torch.empty_like(c["q"])
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    before = _lib.launch_count()
    _fp8_call(lib, c, nosplit)                                        # workspace NULL: one split
    assert _lib.launch_count() == before + (1 if sq == 1 else 2)
    torch.cuda.synchronize()
    assert _same_bits(a, b), "the split path is not deterministic"
    check_rows(a, ref, c["cache_seqlens"], sq, True, True, "split")
    check_rows(nosplit, ref, c["cache_seqlens"], sq, True, True, "no split")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [1, 6])
def test_fp8_kvcache_cuda_graph_with_changed_lengths(sq):
    be = _backend()
    lens_a, lens_b = [100, 3000], [700, 40]
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
    assert torch.equal(_bytes(replay_k), _bytes(c["k_cache"])) and torch.equal(_bytes(replay_v), _bytes(c["v_cache"]))
    ref, _, _ = reference_fp8(c["q"], snap_k, snap_v, c["k"], c["v"], c["cache_seqlens"], c["block_table"], True,
                              1.0 / math.sqrt(D))
    check_rows(out, ref, c["cache_seqlens"], sq, True, True, "graph replay")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [2, 4, 8])
def test_fp8_verification_equals_successive_decodes(sq):
    be = _backend()
    c = make_case(4, sq, 32, 8, [0, 255, 1024, 4000], True, seed=8 + sq)
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    verify = _run(c, True)
    ver_k, ver_v = c["k_cache"].clone(), c["v_cache"].clone()
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    steps = [be.attn_with_kvcache(c["q"][:, i:i + 1].contiguous(), c["k_cache"], c["v_cache"], c["k"][:, i:i + 1],
                                  c["v"][:, i:i + 1], c["cache_seqlens"] + i, block_table=c["block_table"], causal=True)
             for i in range(sq)]
    torch.cuda.synchronize()
    auto = torch.cat(steps, dim=1)
    assert torch.equal(_bytes(ver_k), _bytes(c["k_cache"])) and torch.equal(_bytes(ver_v), _bytes(c["v_cache"]))
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
@pytest.mark.parametrize("sq", [1, 3])
def test_fp8_kvcache_dispatch(sq):
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    c = make_case(2, sq, 32, 8, [100, 5000], True, seed=9 + sq)
    ws, wsn = be._ws(2, 32, D, c["q"].device)
    direct_out = torch.empty_like(c["q"])
    snap_k, snap_v = c["k_cache"].clone(), c["v_cache"].clone()
    holder = {}
    via_backend = _entries(lib, lambda: holder.setdefault("o", _run(c, True)))
    c["k_cache"].copy_(snap_k)
    c["v_cache"].copy_(snap_v)
    via_c = _entries(lib, lambda: _fp8_call(lib, c, direct_out, ws=ws, wsn=wsn))
    assert via_backend == via_c and len(via_c) == (2 if sq == 1 else 3)      # (append,) split attention, merge
    assert set(via_c) == ({"chitu_b200_gqa_paged_attn_fp8kv"} if sq == 1 else {"gqa_paged_prefill_e4m3"})
    assert _same_bits(holder["o"], direct_out)


@pytest.mark.gpu
def test_llama_engine_fp8_kvcache_matches_bf16_engine_on_decoded_cache():
    """kv_dtype=float8_e4m3fn: after set_synthetic_context, a bf16 engine whose caches hold the decoded values gives
    the same greedy tokens over several steps, and logits within the engine tests' tolerance (the two engines differ
    only in the rounding of the rows each step appends)."""
    from chitu_b200.engine import LlamaConfig, LlamaDecodeEngine
    cfg = LlamaConfig(dim=1024, n_layers=2, n_heads=8, n_kv_heads=2, vocab_size=4096, multiple_of=256)
    kw = dict(max_reqs=4, max_seq_len=1024, seed=3)
    e8 = LlamaDecodeEngine(cfg, kv_dtype=E4M3, **kw)
    eb = LlamaDecodeEngine(cfg, **kw)
    assert e8.k_cache.dtype == E4M3 and eb.k_cache.dtype == torch.bfloat16
    e8.set_synthetic_context(500)
    eb.set_synthetic_context(500)
    eb.k_cache.copy_(e8.k_cache.to(torch.bfloat16))
    eb.v_cache.copy_(e8.v_cache.to(torch.bfloat16))
    assert torch.equal(eb.block_table, e8.block_table)
    assert e8.k_cache.float().abs().max() <= 448 and not torch.isnan(e8.k_cache.float()).any()
    e8.capture()
    eb.capture()
    tokens = torch.tensor([1, 17, 300, 4000], dtype=torch.int64)
    for step in range(4):
        t8, tb = e8.decode(tokens), eb.decode(tokens)
        torch.cuda.synchronize()
        cd, mr = cos_diff(e8.logits.float(), eb.logits.float()), max_rel(e8.logits.float(), eb.logits.float())
        assert cd < 1e-2 and mr < 0.15, (step, cd, mr)
        assert torch.equal(t8, tb), (step, t8, tb)
        tokens = t8
    # layer 0's new rows depend on the token and the position only: the fp8 engine stored e4m3 of the bf16 engine's
    for b in range(4):
        for pos in range(500, 504):
            blk, off = int(e8.block_table[b, pos // e8.page]), pos % e8.page
            assert torch.equal(_bytes(e8.k_cache[0, blk, off]), _bytes(quant(eb.k_cache[0, blk, off])))
            assert torch.equal(_bytes(e8.v_cache[0, blk, off]), _bytes(quant(eb.v_cache[0, blk, off])))
