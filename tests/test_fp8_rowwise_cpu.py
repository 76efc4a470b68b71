"""FP8 rowwise (e4m3 W8A8, per-channel weight and per-token activation scales) without a GPU: the quantisation rule
against vLLM's, the module's constructors and refusals, every C-entry refusal, and the LLaMA engine's FP8 step traced
with the recording library of tests/test_engine_calls_cpu.py."""
import pytest
import torch

import test_engine_calls_cpu as EC
from chitu_b200.quantize import Fp8Linear
from chitu_b200.quantize import fp8 as Q

BF, E4M3 = torch.bfloat16, torch.float8_e4m3fn


def quant_rowwise(x, scale=None, scale_ub=None):
    """The per-token rule of chitu_b200_quant_fp8_rowwise restated in torch: (q e4m3, s fp32 [rows])."""
    xf = x.float().reshape(-1, x.shape[-1])
    if scale is None:
        amax = xf.abs().amax(dim=-1)
        if scale_ub is not None:
            amax = amax.clamp(max=float(scale_ub))
        # a tensor divisor: torch divides a CUDA tensor by a Python scalar as a multiply by its reciprocal
        s = (amax / torch.full_like(amax, 448.0)).clamp(min=Q.MIN_SCALE)
    else:
        s = torch.full((xf.shape[0],), float(scale), dtype=torch.float32, device=x.device)
    q = (xf * s.reciprocal()[:, None]).clamp(-448.0, 448.0).to(E4M3)
    return q.view(x.shape), s


def _rows(seed, M=24, K=512):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, K, generator=g) * 2.0 ** (torch.arange(M) % 7 - 3).float()[:, None]).to(BF)
    x[0] = 0                                          # the min-scale floor
    x[1, 5] = 3e4                                     # a large outlier (saturates under an upper bound)
    return x


def _vllm_quant(static):
    """vLLM's QuantFP8(static, PER_TOKEN / PER_TENSOR).forward_native, called on a stand-in for the module: building the
    CustomOp itself needs a vLLM config and a device platform, which forward_native does not use."""
    import types
    vq = pytest.importorskip("vllm.model_executor.layers.quantization.input_quant_fp8")
    from vllm.model_executor.layers.quantization.utils.quant_utils import GroupShape
    assert vq._FP8_DTYPE == E4M3 and vq._FP8_MAX == 448.0
    this = types.SimpleNamespace(static=static, group_shape=GroupShape.PER_TENSOR if static else GroupShape.PER_TOKEN,
                                 is_group_quant=False, num_token_padding=None)
    return lambda x, **kw: vq.QuantFP8.forward_native(this, x, **kw)


@pytest.mark.parametrize("mode", ["dynamic", "dynamic_ub", "static"])
def test_rule_equals_vllm_quant_fp8_forward_native(mode):
    x = _rows(1)
    if mode == "static":
        op, kw = _vllm_quant(True), dict(scale=torch.tensor([0.0173], dtype=torch.float32))
    else:
        op = _vllm_quant(False)
        kw = dict(scale_ub=torch.tensor([1.5], dtype=torch.float32)) if mode == "dynamic_ub" else {}
    want_q, want_s = op(x, **kw)
    q, s = quant_rowwise(x, scale=kw.get("scale"), scale_ub=kw.get("scale_ub"))
    assert torch.equal(q.view(torch.uint8), want_q.view(torch.uint8)), mode
    assert torch.equal(s, want_s.float().expand(x.shape[0], 1).reshape(-1)), mode


def test_rule_edges():
    q, s = quant_rowwise(_rows(2))
    assert float(s[0]) == torch.tensor(1.0 / (448 * 512), dtype=torch.float32).item() and not q[0].float().any()
    assert float(q[1, 5].float()) == 448.0                           # the row's amax lands on the largest e4m3
    q, s = quant_rowwise(_rows(2), scale_ub=1.0)                    # the bound clamps row 1's amax: its outlier saturates
    assert float(q[1, 5].float()) == 448.0 and float(s[1]) == (torch.tensor(1.0) / 448).item()


def test_quantize_weight_layout_and_rule():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(48, 256, generator=g) * 0.05
    w[7] = 0
    q, s = Q.quantize_weight(w)
    assert q.dtype == E4M3 and tuple(q.shape) == (48, 256) and s.dtype == torch.float32 and tuple(s.shape) == (48,)
    want = w.abs().amax(dim=-1) / 448
    assert torch.equal(s[torch.arange(48) != 7], want[torch.arange(48) != 7]) and float(s[7]) == 1.0
    assert torch.equal(q.view(torch.uint8), (w / s[:, None]).clamp(-448, 448).to(E4M3).view(torch.uint8))
    assert torch.equal(q.float().abs().amax(dim=-1)[torch.arange(48) != 7], torch.full((47,), 448.0))
    assert torch.equal(Q.dequantize(q, s), q.float() * s[:, None])


def test_from_float_and_checkpoint_layouts():
    lin = torch.nn.Linear(256, 64, bias=True)
    m = Fp8Linear.from_float(lin)
    q, s = Q.quantize_weight(lin.weight.detach())
    assert torch.equal(m.weight.view(torch.uint8), q.view(torch.uint8)) and torch.equal(m.weight_scale, s)
    assert m.bias.dtype == BF and m.input_scale is None and m.input_scale_ub is None
    N, K = 64, 256
    for ws in (s[:, None], s, torch.tensor(0.02), 0.02):
        m = Fp8Linear.from_compressed_tensors(q, ws)
        assert tuple(m.weight_scale.shape) == (N,) and m.weight_scale.dtype == torch.float32
        assert torch.equal(m.weight_scale, torch.as_tensor(ws, dtype=torch.float32).reshape(-1).expand(N))
    m = Fp8Linear.from_compressed_tensors(q, s[:, None], input_scale=torch.tensor([0.5]))
    assert tuple(m.input_scale.shape) == (1,) and float(m.input_scale) == 0.5 and m.input_scale_ub is None
    m = Fp8Linear.from_fbgemm(q, s[:, None], input_scale_ub=torch.tensor(1200.0), bias=torch.ones(N))
    assert float(m.input_scale_ub) == 1200.0 and m.input_scale is None and m.bias.dtype == BF
    assert (m.in_features, m.out_features) == (K, N)


def test_module_refusals():
    q, s = Q.quantize_weight(torch.randn(32, 128))
    with pytest.raises(ValueError, match="e4m3"):
        Fp8Linear.from_compressed_tensors(q.to(torch.float8_e5m2), s)
    with pytest.raises(ValueError, match="e4m3"):
        Fp8Linear.from_fbgemm(q.float(), s[:, None])
    with pytest.raises(ValueError, match="weight_scale"):
        Fp8Linear.from_compressed_tensors(q, s[:16])
    with pytest.raises(ValueError, match="16"):
        Fp8Linear(200, 32)
    with pytest.raises(ValueError, match="16"):
        Q.quantize_weight(torch.randn(8, 72))
    m = Fp8Linear.from_compressed_tensors(q, s)
    for dt in (torch.float16, torch.float32):
        with pytest.raises(ValueError, match="bf16"):
            m(torch.zeros(2, 128, dtype=dt))
    with pytest.raises(ValueError, match="CUDA"):
        m(torch.zeros(2, 128, dtype=BF))
    with pytest.raises(ValueError, match="CUDA"):
        Q.quant_act_fp8(torch.zeros(2, 128, dtype=BF))
    with pytest.raises(ValueError, match="bf16"):
        Q.quant_act_fp8(torch.zeros(2, 128, dtype=torch.float16))


def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def test_c_entries_refuse_bad_arguments_and_launch_nothing():
    from chitu_b200._lib import launch_count
    lib = _lib()
    A = 1 << 20                                  # 16-byte aligned stand-ins: every case is refused before a dereference
    a, a_s, b, b_s, y, ws, bias, res = (i * A for i in range(1, 9))

    def plain(**kw):
        v = dict(a=a, a_s=a_s, b=b, b_s=b_s, bias=None, res=None, y=y, M=4, N=64, K=256, ws_bytes=1 << 20)
        v.update(kw)
        return lib.chitu_b200_fp8_rowwise_gemm(v["a"], v["a_s"], v["b"], v["b_s"], v["bias"], v["res"], v["y"], v["M"],
                                               v["N"], v["K"], ws, v["ws_bytes"], None), "chitu_b200_fp8_rowwise_gemm"

    def pairs(**kw):
        v = dict(a=a, a_s=a_s, b=b, b_s=b_s, y=y, M=4, N=64, K=256, ws_bytes=1 << 20)
        v.update(kw)
        return (lib.chitu_b200_fp8_rowwise_gemm_silu_pairs(v["a"], v["a_s"], v["b"], v["b_s"], v["y"], v["M"], v["N"],
                                                           v["K"], ws, v["ws_bytes"], None),
                "chitu_b200_fp8_rowwise_gemm_silu_pairs")

    before = launch_count()
    bad = [dict(a=None), dict(a_s=None), dict(b=None), dict(b_s=None), dict(y=None), dict(a=a + 8), dict(a_s=a_s + 4),
           dict(b=b + 8), dict(b_s=b_s + 4), dict(y=y + 2), dict(K=200), dict(K=8), dict(K=0), dict(M=-1), dict(N=0),
           dict(ws_bytes=16)]
    for call in (plain, pairs):
        for kw in bad:
            rc, name = call(**kw)
            assert rc < 0, (name, kw)
            assert name in lib.chitu_b200_last_error().decode(), (name, kw)
    for kw in (dict(res=res + 8), dict(bias=bias + 2)):
        rc, name = plain(**kw)
        assert rc < 0 and name in lib.chitu_b200_last_error().decode(), kw
    rc, name = pairs(N=65)
    assert rc < 0 and name in lib.chitu_b200_last_error().decode()
    for call in (plain, pairs):                  # M = 0: nothing to do
        assert call(M=0)[0] == 0

    x, q, qs, w, sc = a, b, a_s, bias, b_s
    quant = lambda **kw: lib.chitu_b200_quant_fp8_rowwise(                      # noqa: E731
        kw.get("x", x), kw.get("q", q), kw.get("qs", qs), kw.get("rows", 4), kw.get("K", 256), kw.get("scale"),
        kw.get("ub"), None)
    for kw in (dict(x=None), dict(q=None), dict(qs=None), dict(x=x + 8), dict(q=q + 4), dict(K=200), dict(K=0),
               dict(rows=-1), dict(scale=sc, ub=sc + 16)):
        assert quant(**kw) < 0, kw
        assert "chitu_b200_quant_fp8_rowwise" in lib.chitu_b200_last_error().decode(), kw
    assert quant(rows=0) == 0
    norm = lambda **kw: lib.chitu_b200_rmsnorm_quant_fp8_rowwise(                # noqa: E731
        kw.get("x", x), kw.get("w", w), kw.get("y"), kw.get("q", q), kw.get("qs", qs), kw.get("rows", 4),
        kw.get("dim", 512), 1e-5, None)
    for kw in (dict(x=None), dict(w=None), dict(q=None), dict(qs=None), dict(dim=0), dict(dim=16384),
               dict(x=x + 1), dict(w=w + 3), dict(rows=-1)):
        assert norm(**kw) < 0, kw
        assert "chitu_b200_rmsnorm_quant_fp8_rowwise" in lib.chitu_b200_last_error().decode(), kw
    assert norm(rows=0) == 0
    assert launch_count() == before


# --------------------------------------------------------------------------------------------------------- engine
def test_engine_refusals():
    with pytest.raises(ValueError, match="fp8"):
        EC._llama(128, tp_size=2, process_group=EC.PG, weight_format="fp8")
    with pytest.raises(ValueError, match="fp8"):
        EC._llama(128, linear_impl=1, weight_format="fp8")
    with pytest.raises(ValueError, match="weight_format"):
        EC._mixtral(tp_size=1, weight_format="fp8")       # the Mixtral engine has no FP8 experts


def _trace(**kw):
    rec = EC.Recorder()
    with EC._patched(rec):
        eng = EC._llama(128, **kw)
        rec.watch(eng)
        eng._step_body()
    return eng, rec


FP8_NAMES = {"chitu_b200_linear_bf16": "chitu_b200_fp8_rowwise_gemm",
             "chitu_b200_linear_bf16_silu_pairs": "chitu_b200_fp8_rowwise_gemm_silu_pairs",
             "chitu_b200_rmsnorm": "chitu_b200_rmsnorm_quant_fp8_rowwise"}


@pytest.mark.parametrize("tp_size", [1, 2])
def test_llama_fp8_step_calls(tp_size):
    """The FP8 step is the bf16 step's calls with the layer GEMMs and the norms that feed them swapped for their FP8
    entries, plus a per-token quantiser before wo and before w2; the final norm (read by the bf16 head) stays bf16."""
    from chitu_b200._lib import CB_BF16
    bf, rec_bf = _trace(tp_size=tp_size)
    f8, rec = _trace(tp_size=tp_size, weight_format="fp8")
    names_bf = [c[0] for c in rec_bf.calls]
    names = [c[0] for c in rec.calls]
    L = len(f8.layers)
    assert len(names) == len(names_bf) + 2 * L
    assert names.count("chitu_b200_quant_fp8_rowwise") == 2 * L
    rest = [n for n in names if n != "chitu_b200_quant_fp8_rowwise"]
    # the final norm and the head keep their bf16 calls
    keep = {max(j for j, n in enumerate(names_bf) if n == k) for k in ("chitu_b200_rmsnorm", "chitu_b200_linear_bf16")}
    for i, (a, b) in enumerate(zip(rest, names_bf)):
        assert a == (b if i in keep else FP8_NAMES.get(b, b)), (i, a, b)
    # each quantiser sits directly before wo / w2 and writes what they read
    ptr = lambda t: rec.pointer(t.data_ptr())                                  # noqa: E731
    xq, xs = ptr(f8.xq), ptr(f8.xs)
    gemms = [c for c in rec.calls if c[0] == "chitu_b200_fp8_rowwise_gemm"]
    D = f8.D
    for i, c in enumerate(rec.calls):
        if c[0] == "chitu_b200_quant_fp8_rowwise":
            nxt = rec.calls[i + 1]
            assert nxt[0] == "chitu_b200_fp8_rowwise_gemm" and c[2:4] == [xq, xs] and nxt[1:3] == [xq, xs]
            assert c[5] == nxt[10] and c[6:8] == [None, None]
        if c[0] == "chitu_b200_rmsnorm_quant_fp8_rowwise":
            assert c[4:6] == [xq, xs] and c[6:8] == [f8.B, f8.cfg.dim] and c[3] is None
    for li, lw in enumerate(f8.layers):
        for c, name, N, K, has_res in ((gemms[3 * li], "wqkv", (f8.Hq + 2 * f8.Hkv) * D, f8.cfg.dim, False),
                                       (gemms[3 * li + 1], "wo", f8.cfg.dim, f8.Hq * D, True),
                                       (gemms[3 * li + 2], "w2", f8.cfg.dim, f8.F, True)):
            q, s = lw[name]
            assert c[1:5] == [xq, xs, ptr(q), ptr(s)] and c[5] is None and c[8:11] == [f8.B, N, K], (li, name)
            assert (c[6] is not None) == has_res
            assert q.dtype == E4M3 and tuple(q.shape) == (N, K) and s.dtype == torch.float32
    assert sum(1 for n in names if n == "chitu_b200_linear_bf16") == 1 and CB_BF16 == 0     # the head


def test_llama_fp8_weights_are_the_bf16_weights_quantised():
    bf = EC._llama(128)
    f8 = EC._llama(128, weight_format="fp8")
    for lb, lq, lr in zip(bf.layers, f8.layers, f8.ref_layers()):
        for name in ("wqkv", "wo", "w13", "w2"):
            q, s = Q.quantize_weight(lb[name])
            assert torch.equal(lq[name][0].view(torch.uint8), q.view(torch.uint8)) and torch.equal(lq[name][1], s)
        assert lr["wqkv"].dtype == torch.float32
        F = f8.F
        w13 = Q.dequantize(*lq["w13"])                     # interleaved rows -> the reference's [w1 ; w3]
        assert torch.equal(lr["w13"][:F], w13[0::2]) and torch.equal(lr["w13"][F:], w13[1::2])
    assert torch.equal(bf.embed, f8.embed) and torch.equal(bf.head, f8.head)
