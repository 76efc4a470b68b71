"""Absorbed-MLA prefill attention (chitu_b200_mla_prefill behind B200AttnBackend.attn_varlen_func): argument checks and
CPU refusal without a GPU; on the H100 parity with an fp32 flash_attn_varlen_func reference per sequence, NaN-poisoned
strided views, rows that see no key, determinism, CUDA-graph capture with a changed split, and dispatch."""
import math

import pytest
import torch

from conftest import cos_diff, max_rel

QK, DV = 576, 512


def _backend():
    from chitu_b200.attn_backend import B200AttnBackend
    return B200AttnBackend()


def _cu(lens, device):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return torch.tensor(cu, dtype=torch.int32, device=device)


def _inputs(lens_q, lens_k, H, seed=0, device="cuda"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    tq, tk = sum(lens_q), sum(lens_k)
    # q scaled so that the score range (and hence the running-max rescale) is exercised, not only flat softmaxes
    q = (torch.randn(tq, H, QK, generator=g) * 2.0).bfloat16().to(device)
    kv = torch.randn(tk, 1, QK, generator=g).bfloat16().to(device)
    k = kv
    v = kv[..., :DV]                           # v = kv_norm(kv): the first 512 columns of the same rows, as in DeepSeek
    return q, k, v


def reference(q, k, v, lens_q, lens_k, causal, scale):
    """fp32 flash_attn_varlen_func on the GPU, chunked over heads (<= ~1 GB of scores); a row that sees no key is 0."""
    H = q.shape[1]
    out = torch.zeros(q.shape[0], H, v.shape[-1], dtype=torch.float32, device=q.device)
    oq = ok = 0
    for lq, lk in zip(lens_q, lens_k):
        if lq > 0:
            qs, ks, vs = q[oq:oq + lq].float(), k[ok:ok + lk, 0].float(), v[ok:ok + lk, 0].float()
            mask = torch.ones(lq, lk, dtype=torch.bool, device=q.device)
            if causal:
                mask = mask.tril(diagonal=lk - lq)
            hc = max(1, min(H, (1 << 28) // max(1, lq * lk)))
            for h0 in range(0, H, hc):
                s = torch.einsum("qhd,kd->hqk", qs[:, h0:h0 + hc], ks) * scale
                s = s.masked_fill(~mask, float("-inf"))
                p = torch.softmax(s, dim=-1).nan_to_num(0.0)
                out[oq:oq + lq, h0:h0 + hc] = torch.einsum("hqk,kd->qhd", p, vs)
        oq += lq
        ok += lk
    return out


def _check_per_sequence(got, ref, lens_q, what):
    o = 0
    for i, n in enumerate(lens_q):
        if n:
            g, r = got[o:o + n].float(), ref[o:o + n]
            assert not torch.isnan(g).any(), f"{what}: NaN in sequence {i}"
            if r.abs().max() > 0:
                cd, mr = cos_diff(g, r), max_rel(g, r)
                assert cd < 1e-5 and mr < 1e-2, f"{what}: sequence {i} (len {n}) cos_diff {cd:.2e} max_rel {mr:.2e}"
            else:
                assert torch.equal(g, torch.zeros_like(g)), f"{what}: sequence {i} must be zeros"
        o += n


# ---------------------------------------------------------------- no GPU needed

def test_mla_prefill_bad_arguments_return_status():
    from chitu_b200 import _lib
    lib = _lib.load()
    A = 16          # a non-null, 16-byte aligned address: every case below is refused before anything is touched

    def call(q=A, k_sb=QK, v_sb=DV, B=1, H=4, total_q=8, max_q=8):
        return lib.chitu_b200_mla_prefill(q, A, k_sb, A, v_sb, A, A, B, H, total_q, 8, max_q, 1, 0.04, A, None)

    bad = [dict(q=None), dict(H=0), dict(B=-1), dict(max_q=-1),
           dict(k_sb=520), dict(k_sb=580), dict(v_sb=504),           # shorter than a row / not a 16-byte multiple
           dict(q=A + 8),                                            # base not 16-byte aligned
           dict(H=128, total_q=1 << 24)]                             # total_q * H beyond int32 row coordinates
    for kw in bad:
        assert call(**kw) < 0, kw
        assert b"mla_prefill" in lib.chitu_b200_last_error(), kw
    assert call(B=0) == 0                                            # an empty batch launches nothing


def test_attn_varlen_mla_shape_refuses_cpu_tensors():
    be = _backend()
    q = torch.zeros(4, 2, QK, dtype=torch.bfloat16)
    kv = torch.zeros(4, 1, QK, dtype=torch.bfloat16)
    cu = torch.tensor([0, 4], dtype=torch.int32)
    with pytest.raises(RuntimeError):
        be.attn_varlen_func(q, kv, kv[..., :DV], cu, cu, 4, 4, causal=True)


# ---------------------------------------------------------------- H100

PARITY_CASES = [
    ([1], [1]),
    ([64], [64]),
    ([4096], [4096]),
    ([1, 63, 0, 64, 65, 130, 700], [1, 63, 0, 64, 65, 130, 700]),     # ragged, with a zero-length sequence
    ([300, 57], [500, 257]),                                          # Lk = Lq + 200: chunked prefill
]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [8, 16, 128])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("lens", PARITY_CASES, ids=["len1", "len64", "len4096", "ragged", "lk_plus_200"])
def test_mla_prefill_parity(H, causal, lens):
    lens_q, lens_k = lens
    q, k, v = _inputs(lens_q, lens_k, H, seed=H + 7 * causal)
    cq, ck = _cu(lens_q, "cuda"), _cu(lens_k, "cuda")
    got = _backend().attn_varlen_func(q, k, v, cq, ck, max(lens_q), max(lens_k), causal=causal)
    assert got.shape == (q.shape[0], H, DV) and got.dtype == torch.bfloat16
    ref = reference(q, k, v, lens_q, lens_k, causal, 1.0 / math.sqrt(QK))
    _check_per_sequence(got, ref, lens_q, f"H={H} causal={causal}")


@pytest.mark.gpu
def test_mla_prefill_nan_poisoned_views_and_empty_rows():
    from chitu_b200 import _lib
    lib = _lib.load()
    H = 16
    lens_q, lens_k = [100, 70, 33], [40, 90, 33]          # Lq > Lk under causal: rows 0..59 of sequence 0 see no key
    q, k, v = _inputs(lens_q, lens_k, H, seed=3)
    tq, tk, pad = q.shape[0], k.shape[0], 5
    qbuf = torch.full((tq + 2 * pad, H, QK), float("nan"), dtype=torch.bfloat16, device="cuda")
    kbuf = torch.full((tk + 2 * pad, 1, 640), float("nan"), dtype=torch.bfloat16, device="cuda")
    vbuf = torch.full((tk + 2 * pad, 1, 520), float("nan"), dtype=torch.bfloat16, device="cuda")
    qbuf[pad:pad + tq] = q
    kbuf[pad:pad + tk, :, :QK] = k
    vbuf[pad:pad + tk, :, :DV] = v
    qv, kv_, vv = qbuf[pad:pad + tq], kbuf[pad:pad + tk, :, :QK], vbuf[pad:pad + tk, :, :DV]
    sentinel = -7.0
    obuf = torch.full((tq + 2 * pad, H, DV), sentinel, dtype=torch.bfloat16, device="cuda")
    out = obuf[pad:pad + tq]
    cq, ck = _cu(lens_q, "cuda"), _cu(lens_k, "cuda")
    scale = 1.0 / math.sqrt(QK)
    _lib.check(lib.chitu_b200_mla_prefill(qv.data_ptr(), kv_.data_ptr(), kv_.stride(0), vv.data_ptr(), vv.stride(0),
                                          cq.data_ptr(), ck.data_ptr(), len(lens_q), H, tq, tk, max(lens_q), 1, scale,
                                          out.data_ptr(), _lib.current_stream()), "mla_prefill")
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    assert torch.all(obuf[:pad] == sentinel) and torch.all(obuf[pad + tq:] == sentinel)
    assert torch.equal(out[:60], torch.zeros_like(out[:60]))                  # rows that see no key: exact zeros
    ref = reference(q, k, v, lens_q, lens_k, True, scale)
    _check_per_sequence(out, ref, lens_q, "strided NaN-poisoned views")


@pytest.mark.gpu
def test_mla_prefill_deterministic():
    H, lens = 16, [1000, 777, 64]
    q, k, v = _inputs(lens, lens, H, seed=11)
    cu = _cu(lens, "cuda")
    be = _backend()
    a = be.attn_varlen_func(q, k, v, cu, cu, max(lens), max(lens), causal=True)
    b = be.attn_varlen_func(q, k, v, cu, cu, max(lens), max(lens), causal=True)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.gpu
def test_mla_prefill_cuda_graph_with_changed_split():
    H = 16
    lens_a, lens_b = [200, 56, 256], [256, 100, 156]        # same totals, every length <= max_seqlen_q = 256
    q, k, v = _inputs(lens_a, lens_a, H, seed=5)
    cq, ck = _cu(lens_a, "cuda"), _cu(lens_a, "cuda")
    be = _backend()
    be.attn_varlen_func(q, k, v, cq, ck, 256, 256, causal=True)               # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = be.attn_varlen_func(q, k, v, cq, ck, 256, 256, causal=True)
    cq.copy_(_cu(lens_b, "cuda"))
    ck.copy_(_cu(lens_b, "cuda"))
    g.replay()
    torch.cuda.synchronize()
    eager = be.attn_varlen_func(q, k, v, _cu(lens_b, "cuda"), _cu(lens_b, "cuda"), 256, 256, causal=True)
    assert torch.equal(out.view(torch.int16), eager.view(torch.int16))
    ref = reference(q, k, v, lens_b, lens_b, True, 1.0 / math.sqrt(QK))
    _check_per_sequence(out, ref, lens_b, "graph replay")


@pytest.mark.gpu
def test_attn_varlen_dispatch():
    from chitu_b200 import _lib
    be = _backend()
    lens = [48, 80]
    q, k, v = _inputs(lens, lens, 8, seed=2)
    cu = _cu(lens, "cuda")
    before = _lib.launch_count()
    be.attn_varlen_func(q, k, v, cu, cu, 80, 80, causal=True)
    assert _lib.launch_count() == before + 1
    # GQA, head dim 128: the library path, no launch of ours
    qg = torch.randn(128, 8, 128, device="cuda").bfloat16()
    kg = torch.randn(128, 2, 128, device="cuda").bfloat16()
    vg = torch.randn(128, 2, 128, device="cuda").bfloat16()
    before = _lib.launch_count()
    og = be.attn_varlen_func(qg, kg, vg, cu, cu, 80, 80, causal=True)
    assert _lib.launch_count() == before and og.shape == (128, 8, 128)
