"""4-bit MoE experts without a GPU: `quantize.w4a16.pack_experts` from GPTQ and AWQ per-expert tensors against each
format's own dequantisation, every refusal of `fused_experts(use_int4_w4a16=True)` and of
chitu_b200_fused_experts_w4a16 (negative status, nothing launched), and the decode step of
`MixtralDecodeEngine(weight_format="w4a16")` traced with the recording library of tests/test_engine_calls_cpu.py."""
import pytest
import torch

import test_engine_calls_cpu as EC
from chitu_b200.quantize import W4A16Linear
from chitu_b200.quantize import w4a16 as W
from test_w4a16_cpu import _awq_dequant, _awq_tensors, _gptq_dequant, _gptq_tensors

BF, F16, U8 = torch.bfloat16, torch.float16, torch.uint8


# ---------------------------------------------------------------------------------------------------- pack_experts
def _experts(fmt, E, K1, F, seed):
    """E experts' (gate, up, down) W4A16Linear from `fmt` checkpoint tensors, and each module's format dequantisation
    [N, K] in fp16."""
    tensors, build, deq = {"gptq": (_gptq_tensors, W4A16Linear.from_gptq, _gptq_dequant),
                           "awq": (_awq_tensors, W4A16Linear.from_awq, _awq_dequant)}[fmt]
    mods, refs = ([], [], []), ([], [], [])
    for e in range(E):
        for i, (K, N) in enumerate(((K1, F), (K1, F), (F, K1))):
            _, _, s, qw, qz = tensors(K, N, seed=seed + 10 * e + i)
            mods[i].append(build(qw, qz, s))
            refs[i].append(deq(qw, qz, s))
    return mods, refs


@pytest.mark.parametrize("fmt", ["gptq", "awq"])
def test_pack_experts_equals_the_format_dequant_with_bf16_scales(fmt):
    """w1 = [gate ; up] and w2 = down of every expert, in the layout fused_experts takes; the dequantised stacks equal
    each format's own dequantisation with the scales rounded to bf16 (the one rounding the MoE path adds)."""
    E, K1, F = 3, 256, 384
    (gate, up, down), (rg, ru, rd) = _experts(fmt, E, K1, F, seed=7 if fmt == "gptq" else 11)
    w1, w1_s, w1_z, w2, w2_s, w2_z = W.pack_experts(gate, up, down)
    assert (w1.shape, w1_s.shape, w1_z.shape) == ((E, 2 * F, K1 // 2), (E, 2 * F, K1 // 128), (E, 2 * F, K1 // 128))
    assert (w2.shape, w2_s.shape, w2_z.shape) == ((E, K1, F // 2), (E, K1, F // 128), (E, K1, F // 128))
    assert (w1.dtype, w1_s.dtype, w1_z.dtype, w2.dtype, w2_s.dtype, w2_z.dtype) == (U8, BF, U8, U8, BF, U8)
    assert all(t.is_contiguous() for t in (w1, w1_s, w1_z, w2, w2_s, w2_z))
    for e in range(E):
        for got_q, got_s, got_z, mods, refs, rows in ((w1, w1_s, w1_z, (gate[e], up[e]), (rg[e], ru[e]), F),
                                                      (w2, w2_s, w2_z, (down[e],), (rd[e],), K1)):
            for j, (m, ref) in enumerate(zip(mods, refs)):
                sl = slice(j * rows, (j + 1) * rows)
                assert torch.equal(got_q[e, sl], m.qweight) and torch.equal(got_z[e, sl], m.zeros)
                assert torch.equal(got_s[e, sl], m.scales.to(BF))
                # the format's own values fp16((q - z) * s) give back the integers q - z (|q - z| <= 15, one fp16
                # rounding); with s rounded to bf16 the element is bf16((q - z) * bf16(s))
                s16 = m.scales.float().repeat_interleave(128, dim=1)
                qz = torch.round(ref.float() / s16)
                assert torch.equal((qz * s16).to(F16), ref)
                want = (qz * m.scales.to(BF).float().repeat_interleave(128, dim=1)).to(BF)
                got = W.dequantize(got_q[e, sl], got_s[e, sl], got_z[e, sl])
                assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (fmt, e, j)
    # the stacked dequantisation is the per-expert one
    assert torch.equal(W.dequantize(w1, w1_s, w1_z)[1].view(torch.int16),
                       W.dequantize(w1[1], w1_s[1], w1_z[1]).view(torch.int16))


def test_dequantize_without_zeros_means_zeros_of_eight():
    g = torch.Generator().manual_seed(3)
    q = W.pack_rows(torch.randint(0, 16, (2, 8, 256), generator=g).view(16, 256)).view(2, 8, 128)
    s = (torch.rand(2, 8, 2, generator=g) * 0.01).to(BF)
    assert torch.equal(W.dequantize(q, s, None), W.dequantize(q, s, torch.full((2, 8, 2), 8, dtype=U8)))


def test_pack_experts_refusals():
    (gate, up, down), _ = _experts("gptq", 2, 128, 256, seed=1)
    with pytest.raises(ValueError, match="same number"):
        W.pack_experts(gate, up, down[:1])
    with pytest.raises(ValueError, match="chain"):
        W.pack_experts(gate, up, gate)
    biased = W4A16Linear._from_layout(down[0].qweight, down[0].scales, down[0].zeros, torch.zeros(128))
    with pytest.raises(ValueError, match="bias"):
        W.pack_experts(gate, up, [biased, down[1]])


# ------------------------------------------------------------------------------------------------ Python refusals
def _w4_args(E=2, T=3, topk=2, K1=256, N1=512):
    return dict(hidden_states=torch.zeros(T, K1, dtype=BF), w1=torch.zeros(E, N1, K1 // 2, dtype=U8),
                w2=torch.zeros(E, K1, N1 // 4, dtype=U8), topk_weights=torch.ones(T, topk, dtype=BF),
                topk_ids=torch.zeros(T, topk, dtype=torch.int64), use_int4_w4a16=True,
                w1_scale=torch.ones(E, N1, K1 // 128, dtype=BF), w2_scale=torch.ones(E, K1, N1 // 256, dtype=BF),
                w1_zp=torch.zeros(E, N1, K1 // 128, dtype=U8), w2_zp=torch.zeros(E, K1, N1 // 256, dtype=U8))


def _with(**over):
    a = _w4_args()
    a.update(over)
    return a


REFUSALS = {
    "fp16 hidden states": (_with(hidden_states=torch.zeros(3, 256, dtype=F16)), "bf16"),
    "group 64": (_with(block_shape=[0, 64]), "groups of 128"),
    "block 128x128": (_with(block_shape=[128, 128]), "groups of 128"),
    "w1 int32": (_with(w1=torch.zeros(2, 512, 32, dtype=torch.int32)), "w1 must be"),
    "w1 shape": (_with(w1=torch.zeros(2, 512, 64, dtype=U8)), "w1 must be"),
    "w2 shape": (_with(w2=torch.zeros(2, 256, 256, dtype=U8)), "w2 must be"),
    "w1 scale fp16": (_with(w1_scale=torch.ones(2, 512, 2, dtype=F16)), "w1_scale must be"),
    "w2 scale shape": (_with(w2_scale=torch.ones(2, 256, 4, dtype=BF)), "w2_scale must be"),
    "no w1 scale": (_with(w1_scale=None), "needs w1_scale"),
    "w1 zp packed": (_with(w1_zp=torch.zeros(2, 256, 2, dtype=U8)), "pack_experts"),
    "w2 zp packed": (_with(w2_zp=torch.zeros(2, 128, 2, dtype=U8)), "pack_experts"),
    "w2 zp int32": (_with(w2_zp=torch.zeros(2, 256, 2, dtype=torch.int32)), "w2_zp must be"),
    "activation scales": (_with(a1_scale=torch.ones(1)), "activation scales"),
    "K1 % 128": (_with(hidden_states=torch.zeros(3, 192, dtype=BF)), "K1 % 128"),
    "N1 % 256": (_with(w1=torch.zeros(2, 384, 128, dtype=U8)), "N1 % 256"),
    "topk shapes": (_with(topk_ids=torch.zeros(3, 3, dtype=torch.int64)), "topk"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_wrapper_refusals(name):
    from chitu_b200 import fused_moe
    kw, match = REFUSALS[name]
    with pytest.raises(ValueError, match=match):
        fused_moe.fused_experts(**kw)


def test_wrapper_keeps_int8_and_invoke_refusals():
    from chitu_b200 import fused_moe
    a = _w4_args()
    with pytest.raises(NotImplementedError):
        fused_moe.fused_experts(a["hidden_states"], a["w1"], a["w2"], a["topk_weights"], a["topk_ids"],
                                use_int8_w8a16=True)
    with pytest.raises(NotImplementedError):
        fused_moe.invoke_fused_moe_kernel(None, None, None, None, None, None, None, None, None, None, None, False, 2, {},
                                          use_int4_w4a16=True)


def test_wrapper_refuses_cpu_tensors_after_its_checks():
    from chitu_b200 import fused_moe
    with pytest.raises(RuntimeError, match="CUDA"):
        fused_moe.fused_experts(**_w4_args())
    with pytest.raises(RuntimeError, match="CUDA"):
        fused_moe.fused_experts(**_with(w1_zp=None, w2_zp=None, block_shape=[0, 128]))


# ------------------------------------------------------------------------------------------------- C entry refusals
def test_c_entry_refuses_bad_arguments_and_launches_nothing():
    """Every argument check of chitu_b200_fused_experts_w4a16 comes before a launch: null operands, dtypes, a short
    workspace (-1), shapes the grouped path cannot take (-2, no 4-bit fallback); T = 0 does nothing.  Weight mode 3
    is not reachable through chitu_b200_fused_experts."""
    from chitu_b200 import _lib as L
    lib = L.load()
    A = 1 << 20                               # stand-in addresses: every case is refused before a dereference
    T, topk, E, N1, K1 = 4, 2, 8, 512, 256

    def call(**kw):
        a = dict(x=A, w1=2 * A, s1=3 * A, z1=4 * A, w2=5 * A, s2=6 * A, z2=7 * A, tw=8 * A, twd=L.CB_BF16, ids=9 * A,
                 idd=L.CB_I64, T=T, topk=topk, E=E, N1=N1, K1=K1, out=10 * A, res=None, ws=11 * A, nbytes=None)
        a.update(kw)
        nbytes = a["nbytes"] if a["nbytes"] is not None else lib.chitu_b200_moe_workspace_bytes(a["T"], a["topk"], a["E"],
                                                                                                 a["N1"], a["K1"])
        rc = lib.chitu_b200_fused_experts_w4a16(a["x"], a["w1"], a["s1"], a["z1"], a["w2"], a["s2"], a["z2"], a["tw"],
                                                a["twd"], a["ids"], a["idd"], a["T"], a["topk"], a["E"], a["N1"], a["K1"],
                                                a["out"], a["res"], a["ws"], nbytes, None)
        return rc, lib.chitu_b200_last_error().decode(errors="replace")

    before = L.launch_count()
    for kw in (dict(x=None), dict(w1=None), dict(w2=None), dict(s1=None), dict(s2=None), dict(tw=None), dict(ids=None),
               dict(out=None), dict(ws=None), dict(twd=L.CB_F16), dict(idd=L.CB_I16), dict(T=-1), dict(topk=0),
               dict(E=0), dict(N1=0), dict(K1=0), dict(N1=513), dict(nbytes=1024)):
        rc, msg = call(**kw)
        assert rc == -1 and "fused_experts" in msg, (kw, rc, msg)
    for kw in (dict(N1=384), dict(K1=192), dict(N1=384, T=0), dict(T=4097, topk=2)):
        rc, msg = call(**kw)
        assert rc == -2 and "fused_experts_w4a16" in msg, (kw, rc, msg)
    assert call(T=0) == (0, call(T=0)[1])
    assert call(T=0, z1=None, z2=None)[0] == 0
    rc = lib.chitu_b200_fused_experts(A, 2 * A, 5 * A, None, None, 8 * A, L.CB_BF16, 9 * A, L.CB_I64, 0, topk, E, N1, K1,
                                      3, 10 * A, None, 11 * A, 1 << 30, None)
    assert rc == -1 and "wmode" in lib.chitu_b200_last_error().decode()
    assert L.launch_count() == before


# --------------------------------------------------------------------------------------------------------- engine
def _trace(**kw):
    rec = EC.Recorder()
    with EC._patched(rec):
        eng = EC._mixtral(**kw)
        rec.watch(eng)
        eng._step_body()
    return eng, rec


W4_NAMES = {"chitu_b200_linear_bf16": "chitu_b200_w4a16_gemm",
            "chitu_b200_fused_experts": "chitu_b200_fused_experts_w4a16"}


@pytest.mark.parametrize("tp_size", [1, 2])
def test_mixtral_w4a16_step_calls(tp_size):
    """The W4 engine runs qkv and o through chitu_b200_w4a16_gemm and the experts through chitu_b200_fused_experts_w4a16
    on the layers' own 4-bit tensors; every other call is the bf16 engine's, and the step has as many launches."""
    from chitu_b200._lib import CB_BF16
    bf, rec_bf = _trace(tp_size=tp_size)
    w4, rec = _trace(tp_size=tp_size, weight_format="w4a16")
    names_bf = [c[0] for c in rec_bf.calls]
    names = [c[0] for c in rec.calls]
    assert len(names) == len(names_bf)
    n_layers, head = len(w4.layers), 1
    assert names.count("chitu_b200_w4a16_gemm") == 2 * n_layers
    assert names.count("chitu_b200_fused_experts_w4a16") == n_layers
    assert names.count("chitu_b200_linear_bf16") == head and names_bf.count("chitu_b200_linear_bf16") == 2 * n_layers + head
    for a, b in zip(names, names_bf):
        assert a in (b, W4_NAMES.get(b)), (a, b)
    ptr = lambda t: rec.pointer(t.data_ptr())                                  # noqa: E731
    gemms = [c for c in rec.calls if c[0] == "chitu_b200_w4a16_gemm"]
    experts = [c for c in rec.calls if c[0] == "chitu_b200_fused_experts_w4a16"]
    D = w4.D
    for li, lw in enumerate(w4.layers):
        for c, name, N, K in ((gemms[2 * li], "wqkv", (w4.Hq + 2 * w4.Hkv) * D, w4.cfg.dim),
                              (gemms[2 * li + 1], "wo", w4.cfg.dim, w4.Hq * D)):
            q, s, z = lw[name]
            assert c[2:5] == [ptr(q), ptr(s), ptr(z)] and c[8:11] == [N, K, CB_BF16], (li, name)
        (q1, s1, z1), (q2, s2, z2) = lw["w1"], lw["w2"]
        c = experts[li]
        assert c[2:8] == [ptr(q1), ptr(s1), ptr(z1), ptr(q2), ptr(s2), ptr(z2)]
        assert c[12:17] == [w4.B, w4.topk, w4.E, 2 * w4.F, w4.cfg.dim]
        assert tuple(q1.shape) == (w4.E, 2 * w4.F, w4.cfg.dim // 2) and q1.dtype == U8
        assert tuple(s2.shape) == (w4.E, w4.cfg.dim, w4.F // 128) and s2.dtype == BF


def test_mixtral_w4a16_refuses_a_process_group():
    with pytest.raises(ValueError, match="w4a16"):
        EC._mixtral(tp_size=2, process_group=EC.PG, weight_format="w4a16")
    with pytest.raises(ValueError, match="weight_format"):
        EC._mixtral(tp_size=1, weight_format="int3")


def test_mixtral_w4a16_weights_and_bytes():
    """Each 4-bit weight is quantize_rtn of the bf16 engine's weight (same seed); ref_layers() gives their dequantised
    values; the algorithmic bytes count packed weights, scales and zeros."""
    bf = EC._mixtral(tp_size=1)
    w4 = EC._mixtral(tp_size=1, weight_format="w4a16")
    for lb, lq, lr in zip(bf.layers, w4.layers, w4.ref_layers()):
        for name in ("wqkv", "wo"):
            assert all(torch.equal(a, b) for a, b in zip(lq[name], W.quantize_rtn(lb[name], BF)))
            assert torch.equal(lr[name], W.dequantize(*lq[name]))
        for name in ("w1", "w2"):
            want = W.quantize_rtn(lb[name][1], BF)
            assert all(torch.equal(a[1], b) for a, b in zip(lq[name], want))
            assert lr[name].shape == lb[name].shape and lr[name].dtype == BF
        assert torch.equal(lq["gate_w"], lb["gate_w"])
    assert torch.equal(bf.embed, w4.embed) and torch.equal(bf.head, w4.head)
    c = w4.cfg
    n_attn = ((w4.Hq + 2 * w4.Hkv) * w4.D + w4.Hq * w4.D) * c.dim
    n_exp = 3 * w4.F * c.dim
    rest = bf.algorithmic_bytes(100, 2.0) - c.n_layers * (2 * n_attn + 2.0 * 2 * n_exp)
    w4b = lambda n: n // 2 + n // 128 * 3                                      # noqa: E731
    attn_w4 = w4b((w4.Hq + 2 * w4.Hkv) * w4.D * c.dim) + w4b(c.dim * w4.Hq * w4.D)
    assert w4.algorithmic_bytes(100, 2.0) == int(rest + c.n_layers * (attn_w4 + 2.0 * w4b(n_exp)))
