"""FP8 rowwise (`tc_gemm_kernel<KIND_FP8R, BN, EPI>`, csrc/gemm_tc.cu, behind chitu_b200_fp8_rowwise_gemm[_silu_pairs]),
its per-token quantisers, and the module and LLaMA engine built on them.

The GEMM is checked against an fp64 reference over the exact operand values, sum_k qx qw * a_s * b_s (+ bias), on the
shapes the schedule model of tests/test_gemm_dispatch_gpu.py picks (a stage is 128 K-elements, as for W4, so W4's case
table serves), with the bound |y - ref| <= u_out |ref| + tau rss and tau the one the block-scaled fp8 kind meets."""
import pytest
import torch
import torch.nn.functional as F

import test_gemm_dispatch_gpu as G
import torch_ref as R
from conftest import cos_diff, max_rel
from test_fp8_rowwise_cpu import quant_rowwise
from test_gemm_dispatch_gpu import (DEV, N_TAILS, NAN_BYTE, SENTINEL, TICKET_BYTES, U_OUT, Padded, _ratio,
                                    _written_slots)
from test_w4a16_gpu import _case_table, _schedule, _split_case

BF, E4M3 = torch.bfloat16, torch.float8_e4m3fn
TAU = G._tau("fp8", 2)


# ---------------------------------------------------------------------------------------------------- operands
def _operands(M, N, K, seed, bias=False):
    """x quantised per token from rows whose scale doubles between neighbours, W quantised per channel, and the fp64
    values the reference multiplies (the scales folded in: a64 = qx a_s, w64 = qw b_s)."""
    from chitu_b200.quantize import fp8 as Q
    g = torch.Generator().manual_seed(seed)
    tok = 2.0 ** (torch.arange(M) % 4 - 1).float()[:, None]
    x, a_s = quant_rowwise((torch.randn(M, K, generator=g) * tok).to(BF))
    w, b_s = Q.quantize_weight(torch.randn(N, K, generator=g) * 0.05 * (1 + torch.rand(N, 1, generator=g)))
    op = dict(M=M, N=N, K=K, x=x, a_s=a_s, w=w, b_s=b_s)
    op["bias"] = (torch.randn(N, generator=g) * 0.5).to(BF) if bias else None
    op["a64"], op["w64"] = x.double() * a_s.double()[:, None], w.double() * b_s.double()[:, None]
    return op


def _reference(op):
    a, w = op["a64"].to(DEV), op["w64"].to(DEV)
    ref = a @ w.T
    if op["bias"] is not None:
        ref = ref + op["bias"].to(DEV).double()
    return ref, ((a * a) @ (w * w).T).sqrt()


class Call:
    """One chitu_b200_fp8_rowwise_gemm[_silu_pairs] with every operand a view inside a NaN-padded buffer (y: sentinel
    pads)."""

    def __init__(self, op, residual=None, pairs=False):
        self.op, self.M, self.N, self.K, self.pairs = op, op["M"], op["N"], op["K"], pairs
        self.x, self.a_s, self.w, self.b_s = (Padded(op[k]) for k in ("x", "a_s", "w", "b_s"))
        self.bias = None if op["bias"] is None else Padded(op["bias"])
        self.residual = None if residual is None else Padded(residual)
        self.y = Padded(torch.empty(self.M, self.N // 2 if pairs else self.N, dtype=BF), pad=SENTINEL, fill=NAN_BYTE)

    def __call__(self, ws):
        from chitu_b200._lib import current_stream, ptr
        lib = G._lib()
        args = (ptr(self.x.view), ptr(self.a_s.view), ptr(self.w.view), ptr(self.b_s.view))
        if self.pairs:
            return lib.chitu_b200_fp8_rowwise_gemm_silu_pairs(*args, ptr(self.y.view), self.M, self.N, self.K, ptr(ws),
                                                              ws.numel(), current_stream())
        return lib.chitu_b200_fp8_rowwise_gemm(*args, None if self.bias is None else ptr(self.bias.view),
                                               None if self.residual is None else ptr(self.residual.view),
                                               ptr(self.y.view), self.M, self.N, self.K, ptr(ws), ws.numel(),
                                               current_stream())

    def run(self, ws):
        from chitu_b200._lib import check
        check(self(ws), f"fp8 rowwise M={self.M} N={self.N} K={self.K}")
        return self.y.view

    def pads_intact(self):
        bufs = [self.x, self.a_s, self.w, self.b_s, self.y, self.bias, self.residual]
        return all(b.pads_intact() for b in bufs if b is not None)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _workspace(M, N):
    ws = torch.full((G._lib().chitu_b200_linear_workspace_bytes(M, N),), 0xFF, dtype=torch.uint8, device=DEV)
    ws[:TICKET_BYTES].zero_()
    return ws


def _partials_match(op, ws, sc):
    """Each split contributor's fp32 partial slot against the fp64 unscaled sum over its own stages: the split
    reduction adds unscaled partials and scales once."""
    BN, n_tiles = sc["BN"], sc["n_tiles"]
    slots = ws[TICKET_BYTES:].view(torch.float32).view(-1, 2, BN, 128)
    qa, qw = op["x"].double().to(DEV), op["w"].double().to(DEV)
    worst = 0.0
    for t, contributors in sc["split"].items():
        m0, n0 = (t // n_tiles) * BN, (t % n_tiles) * 128
        rows, cols = min(BN, op["M"] - m0), min(128, op["N"] - n0)
        for c, slot, s_lo, s_hi in contributors:
            a, w = qa[m0:m0 + rows, s_lo * 128:s_hi * 128], qw[n0:n0 + cols, s_lo * 128:s_hi * 128]
            ref, rss = a @ w.T, ((a * a) @ (w * w).T).sqrt()
            got = slots[c, slot, :rows, :cols].double()
            worst = max(worst, _ratio(got, ref, rss, 2.0 ** -24, TAU))
    return worst


def _check(call, ws, sc, ref, rss):
    y = call.run(ws)
    torch.cuda.synchronize()
    what = (call.M, call.N, call.K)
    assert call.pads_intact(), ("a pad was overwritten",) + what
    assert bool(torch.isfinite(y).all()), ("non-finite output",) + what
    assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0, ("tickets left non-zero",) + what
    assert _written_slots(ws, sc["BN"]) == sc["slots"], ("partial slots differ from the schedule model",) + what
    assert _partials_match(call.op, ws, sc) <= 1.0, ("a split partial is outside the bound",) + what
    r = _ratio(y, ref, rss, U_OUT[BF], TAU)
    assert r <= 1.0, ("outside the bound", r) + what
    return r


# ------------------------------------------------------------------------- injected-error self-test of the bound
def test_bound_rejects_injected_errors():
    """The bound catches a token scale off by one row, a channel scale off by one row, and one dropped stage."""
    for M, N, K, _ in _case_table(132):
        op = _operands(M, N, K, seed=M * 7919 + N + K)
        a, w = op["a64"], op["w64"]
        ref, rss = a @ w.T, ((a * a) @ (w * w).T).sqrt()
        assert _ratio(ref.to(BF), ref, rss, U_OUT[BF], TAU) <= 1.0
        qa, qw = op["x"].double(), op["w"].double()
        bad = []
        if M > 1:
            bad.append((qa * op["a_s"].double().roll(1)[:, None]) @ w.T)
        bad.append(a @ (qw * op["b_s"].double().roll(1)[:, None]).T)
        k0 = (K // 128) // 2 * 128
        bad.append(ref - a[:, k0:k0 + 128] @ w[:, k0:k0 + 128].T)
        for y in bad:
            assert _ratio(y.to(BF), ref, rss, U_OUT[BF], TAU) > 1.0, (M, N, K)


# ---------------------------------------------------------------------------------------------------- GPU calls
@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True])
def test_case_table_parity(bias):
    """Every (BN x regime) cell: inside the bound, pads untouched, and the workspace shows the model's split with each
    contributor's unscaled partial inside its own bound."""
    sms = _sms()
    worst = 0.0
    for M, N, K, _ in _case_table(sms):
        op = _operands(M, N, K, seed=M * 7919 + N + K, bias=bias)
        ref, rss = _reference(op)
        worst = max(worst, _check(Call(op), _workspace(M, N), _schedule(M, N, K, sms), ref, rss))
    print(f"[fp8 rowwise bound] bias={bias} cases={len(_case_table(sms))} max|y-ref|/bound={worst:.3f}")


@pytest.mark.gpu
def test_tails():
    """N that leaves a partial weight tile, K down to one TMA pitch (16) and K that leaves a partial stage (80, 1040),
    M across the token tiles and m_chunks (129, 256).  Every operand sits between NaN pads."""
    sms = _sms()
    worst = 0.0
    for N in N_TAILS:
        for K in (16, 80, 1040):
            for M in (1, 7, 16, 33, 64, 129, 256):
                op = _operands(M, N, K, seed=3 * M + 5 * N + K, bias=N % 2 == 0)
                ref, rss = _reference(op)
                worst = max(worst, _check(Call(op), _workspace(M, N), _schedule(M, N, K, sms), ref, rss))
    print(f"[fp8 rowwise bound] tails max|y-ref|/bound={worst:.3f}")


@pytest.mark.gpu
def test_k14336_down_projection():
    """LLaMA-3-8B's w2 shape at bs 1 and 16: the per-stage promotion keeps K = 14336 inside the fp32 bound."""
    sms = _sms()
    for M in (1, 16):
        op = _operands(M, 4096, 14336, seed=M)
        ref, rss = _reference(op)
        _check(Call(op), _workspace(M, 4096), _schedule(M, 4096, 14336, sms), ref, rss)


@pytest.mark.gpu
def test_residual_is_one_more_rounding():
    """y(residual) == bf16(float(y) + float(residual)) bit for bit, whole-tile and split (the last contributor adds)."""
    for M, N, K in (_split_case("whole", 64), _split_case("slot1", 128), _split_case("count_gt_cb", 16)):
        op = _operands(M, N, K, seed=M + N + K, bias=True)
        res = torch.randn(M, N, generator=torch.Generator().manual_seed(N)).to(BF)
        plain = Call(op).run(_workspace(M, N)).cpu()
        c = Call(op, residual=res)
        got = c.run(_workspace(M, N)).cpu()
        assert c.pads_intact()
        want = (plain.float() + res.float()).to(BF)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (M, N, K)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(17, 256, 256), (32, 768, 512), (100, 256, 256), (128, 384, 1024),
                                   (1, 28672, 4096), (16, 28672, 4096)])
def test_silu_pairs_equal_plain_gemm_then_silu_and_mul(M, N, K):
    """The pairs epilogue == the plain GEMM (same schedule, so the same fp32 sums) followed by chitu_b200_silu_and_mul
    over its de-interleaved output, bit for bit."""
    from chitu_b200._lib import CB_BF16, check, current_stream, ptr
    op = _operands(M, N, K, seed=M * N + K)
    c = Call(op, pairs=True)
    got = c.run(_workspace(M, N)).clone()
    assert c.pads_intact()
    plain = Call(op).run(_workspace(M, N))
    gu = torch.cat([plain[:, 0::2], plain[:, 1::2]], dim=1).contiguous()
    want = torch.empty(M, N // 2, dtype=BF, device=DEV)
    check(G._lib().chitu_b200_silu_and_mul(ptr(gu), ptr(want), M, N // 2, CB_BF16, current_stream()), "silu")
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (M, N, K)


@pytest.mark.gpu
def test_deterministic_shared_workspace_and_graph_replay():
    """Split shapes of three BN alternating on one workspace reproduce their first results; a captured call replayed
    with new inputs copied in == the eager calls, bit for bit."""
    shapes = [_split_case("slot1", bn) for bn in (16, 64, 128)]
    calls = [Call(_operands(M, N, K, seed=M + N, bias=True)) for M, N, K in shapes]
    ws = torch.zeros(max(G._lib().chitu_b200_linear_workspace_bytes(M, N) for M, N, _ in shapes), dtype=torch.uint8,
                     device=DEV)
    first = [c.run(ws).clone() for c in calls]
    for _ in range(2):
        for c, f in zip(calls, first):
            assert torch.equal(c.run(ws).view(torch.int16), f.view(torch.int16)), (c.M, c.N, c.K)
    assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0

    M, N, K = _split_case("slot1")
    ops = [_operands(M, N, K, seed=100 + i) for i in range(4)]
    call = Call(ops[0])
    ws = torch.zeros(G._lib().chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)

    def load(op):
        for buf, name in ((call.x, "x"), (call.a_s, "a_s"), (call.w, "w"), (call.b_s, "b_s")):
            buf.view.copy_(op[name].to(DEV))

    eager = []
    for op in ops[1:]:
        load(op)
        eager.append(call.run(ws).clone())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call.run(ws)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call.run(ws)
    for op, want in zip(ops[1:], eager):
        load(op)
        call.y.view.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(call.y.view.view(torch.int16), want.view(torch.int16))
    assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0


@pytest.mark.gpu
def test_workspace_short_refused_launch_nothing():
    from chitu_b200._lib import launch_count
    M, N, K = 16, 256, 512
    op = _operands(M, N, K, seed=4)
    ws = _workspace(M, N)
    before = launch_count()
    for pairs, name in ((False, "chitu_b200_fp8_rowwise_gemm"), (True, "chitu_b200_fp8_rowwise_gemm_silu_pairs")):
        assert Call(op, pairs=pairs)(ws[:-1]) == -2 and name in G._lib().chitu_b200_last_error().decode()
    torch.cuda.synchronize()
    assert launch_count() == before and bool((ws[TICKET_BYTES:] == 0xFF).all())


# ------------------------------------------------------------------------------------------------- quantisers
def _quant(x, scale=None, scale_ub=None):
    from chitu_b200._lib import check, current_stream, ptr
    rows, K = x.shape
    q = torch.full((rows, K), 0x7F, dtype=torch.uint8, device=DEV).view(E4M3)
    s = torch.full((rows,), float("nan"), device=DEV)
    check(G._lib().chitu_b200_quant_fp8_rowwise(ptr(x), ptr(q), ptr(s), rows, K, ptr(scale), ptr(scale_ub),
                                                current_stream()), "quant_fp8_rowwise")
    return q, s


def _rows(M, K, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g) * 2.0 ** (torch.arange(M) % 9 - 4).float()[:, None]
    x[0] = 0                                                # all-zero row: the min-scale floor
    if M > 2:
        x[2, K // 3] = 3e4                                  # an outlier that saturates under a bound
    return x.to(BF).to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [16, 80, 4096, 6144, 14336])
def test_quantiser_bit_exact_against_the_torch_rule(K):
    """Dynamic, dynamic with an upper bound, and static (a scale small enough to saturate most rows)."""
    x = _rows(37, K, seed=K)
    for kw in ({}, dict(scale_ub=torch.tensor([0.75], device=DEV)), dict(scale=torch.tensor([1e-3], device=DEV))):
        q, s = _quant(x, kw.get("scale"), kw.get("scale_ub"))
        wq, ws = quant_rowwise(x, kw.get("scale"), kw.get("scale_ub"))
        torch.cuda.synchronize()
        assert torch.equal(q.view(torch.uint8), wq.view(torch.uint8)), (K, list(kw))
        assert torch.equal(s, ws), (K, list(kw))
    assert float(s[0]) == torch.tensor(1e-3).item() and int((q.float().abs() == 448).sum()) > 0
    q, s = _quant(x)
    assert float(s[0]) == quant_rowwise(torch.zeros(1, 16, dtype=BF))[1].item() and not q[0].float().any()


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [128, 4096, 8192])
def test_fused_rmsnorm_quant_equals_norm_then_quant(dim):
    from chitu_b200._lib import CB_BF16, check, current_stream, ptr
    rows = 19
    x = _rows(rows, dim, seed=dim)
    w = (torch.rand(dim, generator=torch.Generator().manual_seed(1)) + 0.5).to(BF).to(DEV)
    lib = G._lib()
    y = torch.empty(rows, dim, dtype=BF, device=DEV)
    check(lib.chitu_b200_rmsnorm(ptr(x), ptr(w), ptr(y), rows, dim, 1e-5, CB_BF16, current_stream()), "rmsnorm")
    want_q, want_s = _quant(y)
    for with_y in (True, False):
        fy = torch.full((rows, dim), float("nan"), dtype=BF, device=DEV)
        q = torch.zeros(rows, dim, dtype=E4M3, device=DEV)
        s = torch.zeros(rows, device=DEV)
        check(lib.chitu_b200_rmsnorm_quant_fp8_rowwise(ptr(x), ptr(w), ptr(fy) if with_y else None, ptr(q), ptr(s),
                                                       rows, dim, 1e-5, current_stream()), "rmsnorm_quant_rowwise")
        torch.cuda.synchronize()
        assert torch.equal(q.view(torch.uint8), want_q.view(torch.uint8)) and torch.equal(s, want_s), (dim, with_y)
        if with_y:
            assert torch.equal(fy.view(torch.int16), y.view(torch.int16))
        else:
            assert bool(fy.isnan().all())


@pytest.mark.gpu
def test_gemm_directly_after_its_quantiser():
    """The GEMM launched right behind the quantiser that writes its activations and scales (PDL: the GEMM streams its
    weights early but reads x and a_s after griddepcontrol.wait) gives the bits of a run with a device synchronise
    between the two."""
    from chitu_b200._lib import check, current_stream, ptr
    lib = G._lib()
    for M, N, K in ((16, 4096, 14336), (1, 6144, 4096), (64, 1024, 4096)):
        op = _operands(M, N, K, seed=M + K)
        x = _rows(M, K, seed=N)
        w, b_s = op["w"].to(DEV), op["b_s"].to(DEV)
        ws = torch.zeros(lib.chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
        outs = []
        for sync in (True, False):
            q = torch.full((M, K), 0x7F, dtype=torch.uint8, device=DEV).view(E4M3)    # NaN until the quantiser runs
            s = torch.full((M,), float("nan"), device=DEV)
            y = torch.empty(M, N, dtype=BF, device=DEV)
            torch.cuda.synchronize()
            check(lib.chitu_b200_quant_fp8_rowwise(ptr(x), ptr(q), ptr(s), M, K, None, None, current_stream()), "q")
            if sync:
                torch.cuda.synchronize()
            check(lib.chitu_b200_fp8_rowwise_gemm(ptr(q), ptr(s), ptr(w), ptr(b_s), None, None, ptr(y), M, N, K,
                                                  ptr(ws), ws.numel(), current_stream()), "gemm")
            torch.cuda.synchronize()
            outs.append(y)
        assert bool(torch.isfinite(outs[0]).all())
        assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)), (M, N, K)


# ------------------------------------------------------------------------------------------------------- module
@pytest.mark.gpu
def test_module_forward_matches_scaled_mm():
    """Fp8Linear.forward against torch._scaled_mm(qx, qw^T, scale_a [M, 1], scale_b [1, N], bias, out_dtype=bf16) on the
    same operands: both inside the fp64 bound, for from_float, compressed-tensors (static and dynamic) and fbgemm."""
    from chitu_b200.quantize import Fp8Linear
    from chitu_b200.quantize import fp8 as Q
    K, N = 512, 384
    lin = torch.nn.Linear(K, N, bias=True)
    with torch.no_grad():
        lin.weight.normal_(0, 0.05, generator=torch.Generator().manual_seed(3))
    q, s = Q.quantize_weight(lin.weight.detach())
    mods = {"float": Fp8Linear.from_float(lin),
            "ct_dynamic": Fp8Linear.from_compressed_tensors(q, s[:, None]),
            "ct_static": Fp8Linear.from_compressed_tensors(q, s[:, None], input_scale=torch.tensor(0.01)),
            "fbgemm": Fp8Linear.from_fbgemm(q, s[:, None], input_scale_ub=torch.tensor(2.0),
                                            bias=lin.bias.detach())}
    for name, m in mods.items():
        m = m.to(DEV)
        for shape in ((32, K), (2, 8, K), (64, K), (5, K)):
            x = (torch.randn(*shape, generator=torch.Generator().manual_seed(len(shape))) * 0.5).to(BF).to(DEV)
            y = m(x)
            assert y.shape == (*shape[:-1], N) and y.dtype == BF
            qx, sx = Q.quant_act_fp8(x.reshape(-1, K), m.input_scale, m.input_scale_ub)
            wq, ws = quant_rowwise(x.reshape(-1, K), m.input_scale, m.input_scale_ub)
            assert torch.equal(qx.view(torch.uint8), wq.view(torch.uint8)) and torch.equal(sx, ws)
            a64, w64 = qx.double() * sx.double()[:, None], m.weight.double() * m.weight_scale.double()[:, None]
            ref = a64 @ w64.T + (0 if m.bias is None else m.bias.double())
            rss = ((a64 * a64) @ (w64 * w64).T).sqrt()
            u = U_OUT[BF]
            bound = 2 * u * ref.abs() + TAU * rss
            M = qx.shape[0]
            outs = [(y.reshape(M, N), "Fp8Linear")]
            if M % 16 == 0:                                 # _scaled_mm's shape rule for e4m3 operands
                outs.append((torch._scaled_mm(qx, m.weight.T, scale_a=sx[:, None].contiguous(),
                                              scale_b=m.weight_scale[None, :].contiguous(), bias=m.bias,
                                              out_dtype=BF), "_scaled_mm"))
            for got, who in outs:
                err = (got.double() - ref).abs()
                assert bool((err <= bound).all()), (name, shape, who, float((err / bound).max()))


# ------------------------------------------------------------------------------------------------------- engine
def _llama(B, S, n_layers=2, weight_format="fp8", kv_dtype=BF):
    import dataclasses

    from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
    cfg = dataclasses.replace(LLAMA3_8B, n_layers=n_layers)
    eng = LlamaDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, device=DEV, page_size=256,
                            weight_format=weight_format, kv_dtype=kv_dtype)
    eng.set_synthetic_context(S)
    return cfg, eng


def _fp8_lin(x, w):
    """An FP8 engine linear in fp32: x quantised per token (the engine's rule), times the dequantised weight."""
    q, s = quant_rowwise(x)
    return ((q.float() * s[:, None]) @ w.T).to(BF)


def _fp8_llama_step(layers, eng, cfg, tokens, kc, vc, lens, cos, sin):
    """tests/torch_ref.llama_layer with each linear's input quantised per token, composed from torch_ref's pieces."""
    Hq, Hkv, eps = cfg.n_heads, cfg.n_kv_heads, cfg.norm_eps
    h = eng.embed[tokens]
    B = h.shape[0]
    for li, lw in enumerate(layers):
        D = lw["wqkv"].shape[0] // (Hq + 2 * Hkv)
        qkv = _fp8_lin(R.rms_norm(h, lw["attn_norm"], eps), lw["wqkv"])
        q = qkv[:, : Hq * D].reshape(B, Hq, D)
        k = qkv[:, Hq * D: (Hq + Hkv) * D].reshape(B, Hkv, D)
        v = qkv[:, (Hq + Hkv) * D:].reshape(B, Hkv, D)
        q, k = R.rotary_interleaved(q, k, cos, sin)
        o = R.gqa_paged_decode(q.view(B, 1, Hq, D), kc[li], vc[li], k.view(B, 1, Hkv, D), v.view(B, 1, Hkv, D), lens,
                               eng.block_table)
        h = h + _fp8_lin(o.reshape(B, Hq * D), lw["wo"])
        Fd = lw["w13"].shape[0] // 2
        gu = _fp8_lin(R.rms_norm(h, lw["ffn_norm"], eps), lw["w13"])
        h = h + _fp8_lin(F.silu(gu[:, :Fd]) * gu[:, Fd:], lw["w2"])
    return R.final_logits(h, eng.norm, eng.head, eps)


@pytest.mark.gpu
def test_llama3_8b_fp8_two_layer_step_vs_torch_ref():
    """Full-width LLaMA-3-8B, 2 layers, bs 16: the FP8 engine's logits against an fp32 reference over ref_layers()
    (the dequantised weights) with the same per-token activation quantisation, at the W4 engine test's tolerance."""
    from test_fullwidth_gpu import _ulp_perturb
    B, S = 16, 1024
    cfg, eng = _llama(B, S)
    lens = torch.full((B,), S, dtype=torch.int32)
    lens[1], lens[2] = 255, 256
    eng.seq_lens.copy_(lens)
    tokens = torch.randint(100, 1000, (B,), generator=torch.Generator().manual_seed(0)).to(DEV)
    kc = [eng.k_cache[l].clone() for l in range(cfg.n_layers)]
    vc = [eng.v_cache[l].clone() for l in range(cfg.n_layers)]
    ln = eng.seq_lens.clone()
    cos, sin = eng.cos_table[ln.long()], eng.sin_table[ln.long()]
    layers = eng.ref_layers()
    for lw in layers:
        assert all(lw[n].dtype == torch.float32 for n in ("wqkv", "wo", "w13", "w2"))
    ref = _fp8_llama_step(layers, eng, cfg, tokens, [c.clone() for c in kc], [c.clone() for c in vc], ln, cos, sin)
    pert = _ulp_perturb(eng.embed, torch.Generator(device=DEV).manual_seed(1))
    saved, eng.embed = eng.embed, pert
    ref2 = _fp8_llama_step(layers, eng, cfg, tokens, kc, vc, ln, cos, sin)
    eng.embed = saved
    floor_mr, floor_cd = max_rel(ref2, ref), cos_diff(ref2, ref)
    eng.decode(tokens.cpu().pin_memory())
    torch.cuda.synchronize()
    got = eng.logits.float()
    mr, cd = max_rel(got, ref), cos_diff(got, ref)
    print(f"llama-3-8b fp8 2 layers: logits max_rel {mr:.3e} (floor {floor_mr:.3e}) cos_diff {cd:.3e} "
          f"(floor {floor_cd:.3e})")
    assert mr < max(1e-2, 3 * floor_mr) and mr < 0.1
    assert cd < max(1e-4, 3 * floor_cd) and cd < 5e-3


@pytest.mark.gpu
@pytest.mark.parametrize("kv_dtype", [BF, E4M3])
def test_llama3_8b_fp8_graph_replay_equals_eager(kv_dtype):
    """A run of decode steps: graph replay bit-identical to eager (logits, next tokens, KV caches, lengths); the captured
    step launches the bf16 step's kernels plus two quantisers per layer."""
    B, S, steps = 4, 600, 4
    cfg, eager = _llama(B, S, kv_dtype=kv_dtype)
    _, graph = _llama(B, S, kv_dtype=kv_dtype)
    graph.capture()
    tokens = torch.randint(100, 1000, (B,), generator=torch.Generator().manual_seed(5))
    for _ in range(steps):
        a, b = eager.decode(tokens.pin_memory()), graph.decode(tokens.pin_memory())
        torch.cuda.synchronize()
        assert torch.equal(a, b)
        assert torch.equal(eager.logits.view(torch.int16), graph.logits.view(torch.int16))
        tokens = a
    assert torch.equal(eager.seq_lens, graph.seq_lens) and int(eager.seq_lens[0]) == S + steps
    for c_e, c_g in zip(eager.caches, graph.caches):
        assert torch.equal(c_e.view(torch.uint8), c_g.view(torch.uint8))
    del eager
    _, bf = _llama(B, S, weight_format="bf16", kv_dtype=kv_dtype)
    bf.capture()
    assert graph.launches_per_step == bf.launches_per_step + 2 * cfg.n_layers
