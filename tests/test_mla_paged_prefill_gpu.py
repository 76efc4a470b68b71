"""Absorbed-MLA attention over the paged latent cache with more than one query token per request
(chitu_b200_mla_paged_prefill behind B200AttnBackend.mla_attn_with_kvcache with a 4-D q_nope): argument checks, CPU
refusal and the fp32 reference pinned to the oracle without a GPU; on the H100 per-request parity over NaN-poisoned
caches and garbage block-table tails, the bit-exact append, rows that see no key, output sentinels, the sq = 1 routing,
the split path, CUDA-graph replay, multi-token-prediction verification against step-by-step decode, and dispatch."""
import math

import pytest
import torch

from conftest import cos_diff, max_rel

C, R, PAGE = 512, 64, 64
ROW = C + R
SCALE = 1.0 / math.sqrt(128 + 64)         # the backend's default: 1 / sqrt(qk_nope_head_dim + qk_rope_head_dim)


def _backend():
    from chitu_b200.attn_backend import B200AttnBackend
    return B200AttnBackend()


def reference(q_nope, q_pe, kv_cache, kv, seq_excl, block_table, causal, scale):
    """fp32 on a copy of the cache: scatter the sq new rows at seq_excl[b] + i (64-token pages), then attention over Lk
    keys with the bottom-right causal mask; a row that sees no key is 0.  Returns (out [B, sq, H, C] fp32, cache)."""
    kc = kv_cache.clone()
    B, sq, H, _ = q_nope.shape
    out = torch.zeros(B, sq, H, C, dtype=torch.float32, device=q_nope.device)
    for b in range(B):
        L = int(seq_excl[b])
        if kv is not None:
            pos = torch.arange(L, L + sq, device=kc.device)
            kc[block_table[b, pos // PAGE].long(), pos % PAGE] = kv.reshape(B, sq, ROW)[b]
            L += sq
        if L == 0:
            continue
        pos = torch.arange(L, device=kc.device)
        rows = kc[block_table[b, pos // PAGE].long(), pos % PAGE].float()            # [L, 576]
        q = torch.cat([q_nope[b], q_pe[b]], dim=-1).float()                           # [sq, H, 576]
        hc = max(1, min(H, (1 << 27) // (sq * L)))                                    # bounded score memory
        for h0 in range(0, H, hc):
            s = torch.einsum("ihd,jd->hij", q[:, h0:h0 + hc], rows) * scale
            if causal:
                mask = torch.ones(sq, L, dtype=torch.bool, device=kc.device).tril(diagonal=L - sq)
                s = s.masked_fill(~mask, float("-inf"))
            p = torch.softmax(s, dim=-1).nan_to_num(0.0)
            out[b, :, h0:h0 + hc] = torch.einsum("hij,jd->ihd", p, rows[:, :C])
    return out, kc


def make_case(B, sq, H, lens, append, seed=0, device="cuda", spare=3):
    """A cache whose unused slots and pages are NaN, a permuted block table whose entries past each request's pages are
    -1, q scaled so the running-max rescale is exercised, and the new latent rows [B, sq, 576] (or None)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    need = [-(-(L + (sq if append else 0)) // PAGE) for L in lens]
    nb = sum(need) + spare
    kc = torch.full((nb, PAGE, ROW), float("nan"), dtype=torch.bfloat16)
    perm = torch.randperm(nb, generator=g)
    bt = torch.full((B, max(need + [1]) + 2), -1, dtype=torch.int32)
    o = 0
    for b, (L, n) in enumerate(zip(lens, need)):
        bt[b, :n] = perm[o:o + n].int()
        o += n
        pos = torch.arange(L)
        kc[bt[b, pos // PAGE].long(), pos % PAGE] = torch.randn(L, ROW, generator=g).bfloat16()
    q_nope = (torch.randn(B, sq, H, C, generator=g) * 2.0).bfloat16()
    q_pe = (torch.randn(B, sq, H, R, generator=g) * 2.0).bfloat16()
    kv = torch.randn(B, sq, ROW, generator=g).bfloat16() if append else None
    to = (lambda t: None if t is None else t.to(device))
    return dict(q_nope=to(q_nope), q_pe=to(q_pe), kv_cache=to(kc), kv=to(kv),
                seq_excl=torch.tensor(lens, dtype=torch.int32, device=device), block_table=to(bt))


def _call(be, c, causal=True, **kw):
    return be.mla_attn_with_kvcache(c["q_nope"], c["q_pe"], c["kv_cache"], c["kv"], c["seq_excl"], None,
                                    c["block_table"], causal=causal, **kw)


def _ref(c, causal, seq_excl=None, kv_cache=None):
    return reference(c["q_nope"], c["q_pe"], c["kv_cache"] if kv_cache is None else kv_cache, c["kv"],
                     c["seq_excl"] if seq_excl is None else seq_excl, c["block_table"], causal, SCALE)


def check_rows(got, ref, seq_excl, sq, appended, causal, what):
    for b in range(got.shape[0]):
        g, r = got[b].float(), ref[b]
        assert not torch.isnan(g).any(), f"{what}: NaN in request {b}"
        Lk = int(seq_excl[b]) + (sq if appended else 0)
        blind = min(sq, max(0, sq - Lk)) if causal else (sq if Lk == 0 else 0)   # leading rows that see no key
        assert torch.equal(g[:blind], torch.zeros_like(g[:blind])), f"{what}: request {b} rows without keys must be 0"
        if blind < sq:
            cd, mr = cos_diff(g[blind:], r[blind:]), max_rel(g[blind:], r[blind:])
            assert cd < 1e-5 and mr < 1e-2, f"{what}: request {b} cos_diff {cd:.2e} max_rel {mr:.2e}"


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---------------------------------------------------------------- no GPU needed

def test_mla_paged_prefill_bad_arguments_return_status():
    from chitu_b200 import _lib
    lib = _lib.load()
    A = 16          # a non-null, 16-byte aligned address: every case below is refused before anything is touched

    def call(qn=A, qpe=A, bt=A, new_kv=None, out=A, ws=None, B=1, sq=2, H=16, c=C, r=R, page=PAGE, nb=8):
        return lib.chitu_b200_mla_paged_prefill(qn, qpe, A, new_kv, A, bt, 4, B, sq, H, c, r, page, nb, 256, 1, SCALE,
                                                out, ws, 0 if ws is None else 1 << 20, None)

    bad = [dict(qn=None), dict(qpe=None), dict(bt=None), dict(out=None),    # null pointers (out: no deferred merge)
           dict(sq=0), dict(H=0), dict(B=-1),
           dict(c=256), dict(r=32), dict(page=128),                         # only C 512, R 64, 64-token pages
           dict(qn=A + 8), dict(new_kv=A + 2), dict(out=A + 4), dict(ws=A + 8),   # bases not 16-byte aligned
           dict(B=1 << 20, sq=64, H=128),                                   # B * sq * H beyond int32 row coordinates
           dict(nb=1 << 26)]                                                # num_blocks * 64 beyond int32 rows
    for kw in bad:
        assert call(**kw) < 0, kw
        assert b"mla_paged_prefill" in lib.chitu_b200_last_error(), kw
    before = _lib.launch_count()
    assert call(B=0) == 0                                                   # an empty batch launches nothing
    assert _lib.launch_count() == before


def test_mla_attn_with_kvcache_multi_token_refuses_cpu_tensors():
    c = make_case(1, 4, 16, [10], True, device="cpu")
    with pytest.raises(RuntimeError):
        _call(_backend(), c)


def test_mla_attn_with_kvcache_bf16_python_refusals():
    be = _backend()
    one = make_case(1, 1, 16, [10], True, device="cpu")
    one = dict(one, q_nope=one["q_nope"][:, 0], q_pe=one["q_pe"][:, 0])        # the 3-D single-token q
    cases = (one, make_case(1, 4, 16, [10], True, device="cpu"))
    for c in cases:
        with pytest.raises(RuntimeError):
            _call(be, c)                                                        # CPU tensors
    if not torch.cuda.is_available():
        return
    for c in cases:
        g = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()}
        for kw in (dict(window_size=(16, 0)), dict(softcap=30.0)):
            with pytest.raises(RuntimeError):
                _call(be, g, **kw)


def test_reference_equals_oracle_decode_at_one_token():
    from oracle.chitu_oracle import mla_attn_with_kvcache, mla_decode
    c = make_case(3, 1, 16, [5, 300, 64], True, seed=1, device="cpu")
    got, kc = _ref(c, True)
    ko = c["kv_cache"].clone()
    want = mla_attn_with_kvcache(c["q_nope"][:, 0], c["q_pe"][:, 0], ko, c["kv"], c["seq_excl"], c["block_table"], SCALE)
    torch.testing.assert_close(got[:, 0].to(want.dtype), want)              # equal up to the one rounding to bf16
    assert _same_bits(kc, ko)
    c["kv"] = None
    got, _ = _ref(c, False)
    want = mla_decode(c["q_nope"][:, 0], c["q_pe"][:, 0], c["kv_cache"], c["seq_excl"], c["block_table"], SCALE)
    torch.testing.assert_close(got[:, 0].to(want.dtype), want)


def test_reference_causal_append_equals_successive_decodes():
    from oracle.chitu_oracle import mla_attn_with_kvcache
    sq = 5
    c = make_case(2, sq, 8, [3, 62], True, seed=2, device="cpu")             # request 1 crosses a page inside the rows
    got, kc = _ref(c, True)
    ko = c["kv_cache"].clone()
    for i in range(sq):
        step = mla_attn_with_kvcache(c["q_nope"][:, i], c["q_pe"][:, i], ko, c["kv"][:, i], c["seq_excl"] + i,
                                     c["block_table"], SCALE)
        torch.testing.assert_close(got[:, i].to(step.dtype), step)
    assert _same_bits(kc, ko), "the reference scatter differs from sq oracle appends"


# ---------------------------------------------------------------- H100

CASES = {
    "mtp2": (2, [4095, 0, 17, 64]),
    "mtp7_ragged": (7, [1, 300, 64, 5000]),
    "pages70": (70, [63, 64, 200]),                                         # page edges inside the new rows
    "prefix512": (512, [8192]),
    "prefill1024": (1024, [0]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("H", [8, 16, 32, 128])
@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("append", [True, False])
def test_mla_paged_prefill_parity(H, case, causal, append):
    sq, lens = CASES[case]
    c = make_case(len(lens), sq, H, lens, append, seed=H + 101 * list(CASES).index(case) + causal + 2 * append)
    ref, kc = _ref(c, causal)
    seq_excl = c["seq_excl"].clone()
    got = _call(_backend(), c, causal)
    torch.cuda.synchronize()
    assert got.shape == c["q_nope"].shape and got.dtype == torch.bfloat16
    assert torch.equal(c["seq_excl"], seq_excl)
    assert _same_bits(c["kv_cache"], kc), "the cache differs from the reference scatter"
    check_rows(got, ref, seq_excl, sq, append, causal, f"H={H} {case} causal={causal} append={append}")


def _c_call(lib, c, out, ws=None, wsn=0, causal=True):
    from chitu_b200 import _lib
    qn, kc, bt = c["q_nope"], c["kv_cache"], c["block_table"]
    B, sq, H, _ = qn.shape
    _lib.check(lib.chitu_b200_mla_paged_prefill(
        qn.data_ptr(), c["q_pe"].data_ptr(), kc.data_ptr(), None if c["kv"] is None else c["kv"].data_ptr(),
        c["seq_excl"].data_ptr(), bt.data_ptr(), bt.stride(0), B, sq, H, C, R, PAGE, kc.shape[0], bt.shape[1] * PAGE,
        int(causal), SCALE, out.data_ptr(), None if ws is None else ws.data_ptr(), 0 if ws is None else wsn,
        _lib.current_stream()), "mla_paged_prefill")


@pytest.mark.gpu
def test_mla_paged_prefill_output_sentinels():
    from chitu_b200 import _lib
    lib = _lib.load()
    B, sq, H, lens = 3, 9, 16, [0, 250, 700]
    c = make_case(B, sq, H, lens, True, seed=4)
    pad, sentinel = 3 * H, -7.0
    obuf = torch.full((B * sq * H + 2 * pad, C), sentinel, dtype=torch.bfloat16, device="cuda")
    out = obuf[pad:pad + B * sq * H]
    ref, kc = _ref(c, True)
    _c_call(lib, c, out)
    torch.cuda.synchronize()
    assert torch.all(obuf[:pad] == sentinel) and torch.all(obuf[pad + B * sq * H:] == sentinel)
    assert _same_bits(c["kv_cache"], kc)
    check_rows(out.view(B, sq, H, C), ref, c["seq_excl"], sq, True, True, "output view")


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
def test_one_token_4d_call_is_the_decode_call():
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    c = make_case(3, 1, 16, [100, 5000, 64], True, seed=12)
    snap = c["kv_cache"].clone()
    c3 = dict(c, q_nope=c["q_nope"][:, 0], q_pe=c["q_pe"][:, 0])
    h3, h4 = {}, {}
    e3 = _entries(lib, lambda: h3.setdefault("o", _call(be, c3)))
    c["kv_cache"].copy_(snap)
    e4 = _entries(lib, lambda: h4.setdefault("o", _call(be, c)))
    assert e3 == e4 and e3 and all("mla_decode" in n for n in e3)
    assert h4["o"].shape == (3, 1, 16, C) and _same_bits(h3["o"], h4["o"])
    c["kv_cache"].copy_(snap)
    out = torch.empty_like(c["q_nope"])
    _c_call(lib, c, out)                                                    # the C entry at sq = 1
    torch.cuda.synchronize()
    for b in range(3):
        cd, mr = cos_diff(out[b].float(), h3["o"][b].float()), max_rel(out[b].float(), h3["o"][b].float())
        assert cd < 1e-5 and mr < 1e-2, (b, cd, mr)


@pytest.mark.gpu
def test_mla_paged_prefill_split_path():
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    c = make_case(1, 2, 16, [16384 - 2], True, seed=5)                      # Lk = 16384
    ref, _ = _ref(c, True)
    before = _lib.launch_count()
    a = _call(be, c)
    assert _lib.launch_count() == before + 3                                # append, split attention, merge
    b = _call(be, c)
    nosplit = torch.empty_like(c["q_nope"])
    before = _lib.launch_count()
    _c_call(lib, c, nosplit)                                                # workspace NULL: one split
    assert _lib.launch_count() == before + 2
    torch.cuda.synchronize()
    assert _same_bits(a, b), "the split path is not deterministic"
    check_rows(a, ref, c["seq_excl"], 2, True, True, "split")
    check_rows(nosplit, ref, c["seq_excl"], 2, True, True, "no split")
    cd, mr = cos_diff(a.float(), nosplit.float()), max_rel(a.float(), nosplit.float())
    assert cd < 1e-5 and mr < 1e-2, (cd, mr)


@pytest.mark.gpu
def test_mla_paged_prefill_cuda_graph_with_changed_lengths():
    be = _backend()
    sq, lens_a, lens_b = 4, [100, 3000], [700, 40]
    c = make_case(2, sq, 16, [max(x, y) for x, y in zip(lens_a, lens_b)], True, seed=6)
    c["seq_excl"].copy_(torch.tensor(lens_a, dtype=torch.int32))
    snap = c["kv_cache"].clone()
    _call(be, c)                                                            # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = _call(be, c)
    c["kv_cache"].copy_(snap)
    c["seq_excl"].copy_(torch.tensor(lens_b, dtype=torch.int32))
    g.replay()
    torch.cuda.synchronize()
    replayed = c["kv_cache"].clone()
    c["kv_cache"].copy_(snap)
    eager = _call(be, c)
    torch.cuda.synchronize()
    assert _same_bits(out, eager)
    assert _same_bits(replayed, c["kv_cache"])
    ref, _ = _ref(c, True, kv_cache=snap)
    check_rows(out, ref, c["seq_excl"], sq, True, True, "graph replay")


@pytest.mark.gpu
@pytest.mark.parametrize("sq", [2, 4])
def test_mtp_verification_equals_successive_decodes(sq):
    be = _backend()
    c = make_case(4, sq, 16, [0, 63, 1024, 4000], True, seed=8 + sq)
    snap = c["kv_cache"].clone()
    verify = _call(be, c)
    ver_cache = c["kv_cache"].clone()
    c["kv_cache"].copy_(snap)
    steps = [be.mla_attn_with_kvcache(c["q_nope"][:, i].contiguous(), c["q_pe"][:, i].contiguous(), c["kv_cache"],
                                      c["kv"][:, i].contiguous(), c["seq_excl"] + i, None, c["block_table"])
             for i in range(sq)]
    torch.cuda.synchronize()
    auto = torch.cat(steps, dim=1)
    assert _same_bits(ver_cache, c["kv_cache"])
    for b in range(4):
        cd, mr = cos_diff(verify[b].float(), auto[b].float()), max_rel(verify[b].float(), auto[b].float())
        assert cd < 1e-5 and mr < 1e-2, (b, cd, mr)


@pytest.mark.gpu
def test_mla_attn_with_kvcache_dispatch():
    from chitu_b200 import _lib
    lib = _lib.load()
    be = _backend()
    c = make_case(2, 1, 16, [100, 5000], True, seed=9)
    qn, qp, kc, kv, se, bt = (c[n] for n in ("q_nope", "q_pe", "kv_cache", "kv", "seq_excl", "block_table"))
    qn, qp = qn[:, 0], qp[:, 0]
    ws, wsn = be._ws(2, 16, C, qn.device)
    direct_out = torch.empty_like(qn)

    def direct():
        _lib.check(lib.chitu_b200_mla_decode(
            qn.data_ptr(), qp.data_ptr(), kc.data_ptr(), kv.data_ptr(), se.data_ptr(), bt.data_ptr(), bt.stride(0), 2, 16,
            C, R, PAGE, kc.shape[0], bt.shape[1] * PAGE, SCALE, direct_out.data_ptr(), ws.data_ptr(), wsn,
            _lib.current_stream()), "mla_decode")

    holder = {}
    via_backend = _entries(lib, lambda: holder.setdefault("o", be.mla_attn_with_kvcache(qn, qp, kc, kv, se, None, bt)))
    via_c = _entries(lib, direct)
    assert via_backend == via_c and len(via_c) >= 1
    assert _same_bits(holder["o"][:, 0], direct_out)
    m = make_case(2, 3, 16, [100, 5000], True, seed=10)
    multi = _entries(lib, lambda: _call(be, m))
    assert multi and all("mla_paged_prefill" in n for n in multi)
