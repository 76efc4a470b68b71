"""W4A16 (`tc_gemm_kernel<KIND_W4, BN, EPI>`, csrc/gemm_tc.cu, behind chitu_b200_w4a16_gemm[_silu_pairs]) against an
fp64 reference over the exact dequantised element values io((q - z) * s), on shapes picked by the schedule model of
tests/test_gemm_dispatch_gpu.py with a W4 stage of 128 K-elements (S = K / 128), and the module and LLaMA engine
built on it.

The bound is that file's: |y - ref| <= u_out |ref| + 2^-13 rss (fp32 accumulation, one output rounding)."""
import functools

import pytest
import torch
import torch.nn.functional as F

import test_gemm_dispatch_gpu as G
import torch_ref as R
from conftest import cos_diff, max_rel
from test_gemm_dispatch_gpu import (BNS, DEV, M_EDGES, NAN_BYTE, REGIMES, SENTINEL, TAU_FP32, TICKET_BYTES, U_OUT,
                                    Padded, _pick_bn, _ratio, _written_slots)

BF, F16 = torch.bfloat16, torch.float16
KIND = "w4"                                   # _schedule: any kind but "16" has 128 K-elements per stage
MAX_STAGES, MAX_N_TILES = 32, 17
UNREACHABLE = tuple((bn, "m_chunks") for bn in (16, 32, 64))


def _schedule(M, N, K, sms):
    return G._schedule(KIND, M, N, K, sms)


@functools.lru_cache(maxsize=None)
def _case_table(sms):
    """One (M, N, K) per reachable (BN, regime) cell: test_gemm_dispatch_gpu._case_table's search with W4 stages."""
    best = {}
    for M in sorted({m for ms in M_EDGES.values() for m in ms}):
        for nt in range(1, MAX_N_TILES + 1):
            for S in range(1, MAX_STAGES + 1):
                N, K = nt * 128, S * 128
                sc = _schedule(M, N, K, sms)
                cost = (sc["grid"] < 2, N * K, N, K)
                for r in sc["regimes"]:
                    key = (sc["BN"], r, M)
                    if key not in best or cost < best[key]:
                        best[key] = cost
    cases = {}
    for BN in BNS:
        for ri, r in enumerate(REGIMES):
            hits = {M: best[(BN, r, M)] for M in M_EDGES[BN] if (BN, r, M) in best}
            if not hits:
                continue
            want = M_EDGES[BN][ri % len(M_EDGES[BN])]
            M = want if want in hits else min(hits, key=lambda m: hits[m])
            _, _, N, K = hits[M]
            cases.setdefault((M, N, K), set()).add((BN, r))
    return tuple((M, N, K, frozenset(c)) for (M, N, K), c in cases.items())


@pytest.mark.parametrize("sms", [132, 114])
def test_case_table_covers_every_reachable_cell(sms):
    table = _case_table(sms)
    cells = {c for *_, cs in table for c in cs}
    assert cells == {(bn, r) for bn in BNS for r in REGIMES} - set(UNREACHABLE)
    for M, N, K, cs in table:
        sc = _schedule(M, N, K, sms)
        assert {(sc["BN"], r) for r in sc["regimes"]} >= cs and K % 128 == 0


# ---------------------------------------------------------------------------------------------------- operands
def _operands(M, N, K, seed, dtype=BF):
    """x [M, K] (neighbouring tokens differ in scale by 2x), q / z uniform over 0..15 with both extremes present,
    scales around 0.01, and the fp64 values the reference multiplies."""
    from chitu_b200.quantize import w4a16 as W
    g = torch.Generator().manual_seed(seed)
    tok = 2.0 ** (torch.arange(M) % 4 - 1).float()[:, None]
    q = torch.randint(0, 16, (N, K), generator=g)
    q[0, 0], q[-1, -1] = 0, 15
    z = torch.randint(0, 16, (N, K // 128), generator=g).to(torch.uint8)
    z[0, 0], z[-1, -1] = 0, 15
    s = ((torch.rand(N, K // 128, generator=g) + 0.5) * 0.01).to(dtype)
    op = dict(M=M, N=N, K=K, dtype=dtype, x=(torch.randn(M, K, generator=g) * tok).to(dtype), qweight=W.pack_rows(q),
              scales=s, zeros=z)
    op["w"] = W.dequantize(op["qweight"], s, z)
    op["a64"], op["w64"] = op["x"].double(), op["w"].double()
    return op


def _reference(op, device=DEV):
    a, w = op["a64"].to(device), op["w64"].to(device)
    return a @ w.T, ((a * a) @ (w * w).T).sqrt()


class Call:
    """One chitu_b200_w4a16_gemm[_silu_pairs] with every operand a view inside a NaN-padded buffer (y: sentinel pads)."""

    def __init__(self, op, residual=None, pairs=False):
        self.op, self.M, self.N, self.K, self.dtype, self.pairs = op, op["M"], op["N"], op["K"], op["dtype"], pairs
        self.x, self.qw = Padded(op["x"]), Padded(op["qweight"])
        self.s, self.z = Padded(op["scales"]), Padded(op["zeros"])
        self.residual = None if residual is None else Padded(residual)
        ncol = self.N // 2 if pairs else self.N
        self.y = Padded(torch.empty(self.M, ncol, dtype=self.dtype), pad=SENTINEL, fill=NAN_BYTE)

    def __call__(self, ws):
        from chitu_b200._lib import current_stream, dtype_code, ptr
        lib = G._lib()
        args = (ptr(self.x.view), ptr(self.qw.view), ptr(self.s.view), ptr(self.z.view))
        if self.pairs:
            return lib.chitu_b200_w4a16_gemm_silu_pairs(*args, ptr(self.y.view), self.M, self.N, self.K,
                                                        dtype_code(self.dtype), ptr(ws), ws.numel(), current_stream())
        res = None if self.residual is None else ptr(self.residual.view)
        return lib.chitu_b200_w4a16_gemm(*args, res, ptr(self.y.view), self.M, self.N, self.K, dtype_code(self.dtype),
                                         ptr(ws), ws.numel(), current_stream())

    def run(self, ws):
        from chitu_b200._lib import check
        check(self(ws), f"w4a16 M={self.M} N={self.N} K={self.K}")
        return self.y.view

    def pads_intact(self):
        bufs = [self.x, self.qw, self.s, self.z, self.y] + ([self.residual] if self.residual else [])
        return all(b.pads_intact() for b in bufs)


def _check(call, ws, sc, ref, rss):
    y = call.run(ws)
    torch.cuda.synchronize()
    what = (call.M, call.N, call.K, str(call.dtype))
    assert call.pads_intact(), ("a pad was overwritten",) + what
    assert bool(torch.isfinite(y).all()), ("non-finite output",) + what
    assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0, ("tickets left non-zero",) + what
    assert _written_slots(ws, sc["BN"]) == sc["slots"], ("partial slots differ from the schedule model",) + what
    r = _ratio(y, ref, rss, U_OUT[call.dtype], TAU_FP32)
    assert r <= 1.0, ("outside the bound", r) + what
    return r


# ------------------------------------------------------------------------- injected-error self-test of the bound
def _injections(op, sc):
    """Outputs of kernels with one error each: a wrong zero in one group of the first tile, the scales of the next
    group used for one group, a dropped stage."""
    from chitu_b200.quantize import w4a16 as W
    M, N, K, out = op["M"], op["N"], op["K"], op["dtype"]
    a = op["a64"]
    g0 = (K // 128) // 2

    def with_w(w):
        return (a @ w.double().T).to(out)

    z = op["zeros"].clone()
    zi = z[: min(N, 128), g0].int()
    z[: min(N, 128), g0] = torch.where(zi == 15, zi - 1, zi + 1).to(torch.uint8)
    yield "a wrong zero", with_w(W.dequantize(op["qweight"], op["scales"], z))
    if K >= 256:
        s = op["scales"].clone()
        s[:, g0] = op["scales"][:, (g0 + 1) % (K // 128)]
        yield "a wrong scale group", with_w(W.dequantize(op["qweight"], s, op["zeros"]))
    w = op["w"].clone()
    w[:, g0 * 128:(g0 + 1) * 128] = 0
    yield "a stage dropped", with_w(w)


def test_bound_rejects_injected_errors():
    names = set()
    for M, N, K, _ in _case_table(132):
        op = _operands(M, N, K, seed=M * 7919 + N + K)
        ref, rss = _reference(op, "cpu")
        assert _ratio(ref.to(BF), ref, rss, U_OUT[BF], TAU_FP32) <= 1.0
        for name, y in _injections(op, _schedule(M, N, K, 132)):
            names.add(name)
            assert _ratio(y, ref, rss, U_OUT[BF], TAU_FP32) > 1.0, (name, M, N, K)
    assert names == {"a wrong zero", "a wrong scale group", "a stage dropped"}


# ---------------------------------------------------------------------------------------------------- GPU calls
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _workspace(M, N):
    ws = torch.full((G._lib().chitu_b200_linear_workspace_bytes(M, N),), 0xFF, dtype=torch.uint8, device=DEV)
    ws[:TICKET_BYTES].zero_()
    return ws


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF, F16])
def test_case_table_parity(dtype):
    """Every (BN x regime) cell: inside the bound, pads untouched, and the workspace shows the model's split."""
    sms = _sms()
    worst = 0.0
    for M, N, K, _ in _case_table(sms):
        op = _operands(M, N, K, seed=M * 7919 + N + K, dtype=dtype)
        ref, rss = _reference(op)
        worst = max(worst, _check(Call(op), _workspace(M, N), _schedule(M, N, K, sms), ref, rss))
    print(f"[w4a16 bound] dtype={str(dtype).split('.')[-1]} cases={len(_case_table(sms))} max|y-ref|/bound={worst:.3f}")


def _linear16(op, w, M, N, K, pairs=False):
    """chitu_b200_linear_bf16 (or _silu_pairs) on the dequantised weight w."""
    from chitu_b200._lib import check, current_stream, dtype_code, ptr
    lib = G._lib()
    x, wd = op["x"].to(DEV), w.to(DEV).contiguous()
    ws = torch.zeros(lib.chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
    if pairs:
        y = torch.empty(M, N // 2, dtype=BF, device=DEV)
        check(lib.chitu_b200_linear_bf16_silu_pairs(ptr(x), ptr(wd), ptr(y), M, N, K, ptr(ws), ws.numel(),
                                                    current_stream()), "pairs")
    else:
        y = torch.empty(M, N, dtype=op["dtype"], device=DEV)
        check(lib.chitu_b200_linear_bf16(ptr(x), ptr(wd), None, None, ptr(y), M, N, K, dtype_code(op["dtype"]), ptr(ws),
                                         ws.numel(), 2, current_stream()), "linear_bf16")
    torch.cuda.synchronize()
    return y


def _both_whole(M, N, K, sms):
    return not _schedule(M, N, K, sms)["split"] and not G._schedule("16", M, N, K, sms)["split"]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF, F16])
def test_whole_tiles_equal_linear16_on_the_dequantised_weight(dtype):
    """Where both schedules give every tile one whole-tile work item, W4 and the 16-bit kernel issue the same wgmma
    sequence (k = 16 steps in K order into one fp32 accumulator) over the same operand values: bit-identical."""
    sms = _sms()
    shapes = [(M, N, K) for M, N, K, _ in _case_table(sms) if _both_whole(M, N, K, sms)]
    shapes += [(M, N, K) for M in (1, 16, 40, 128) for N, K in ((256, 256), (1024, 512), (128, 4096))
               if _both_whole(M, N, K, sms)]
    assert len(shapes) >= 8
    for M, N, K in shapes:
        op = _operands(M, N, K, seed=M + 3 * N + K, dtype=dtype)
        got = Call(op).run(_workspace(M, N)).clone()
        want = _linear16(op, op["w"], M, N, K)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (M, N, K, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF, F16])
def test_tails(dtype):
    """N that leaves a partial weight tile, K from one group to 14336, M from 1 to 256.  Every operand sits between NaN
    pads: a read past M rows of x, past N rows of the weights or past the last group would show up in y."""
    sms = _sms()
    worst = 0.0
    for N in (8, 100, 1000):
        for K in (128, 4224, 14336):
            for M in (1, 7, 16, 33, 64, 129, 256):
                op = _operands(M, N, K, seed=3 * M + 5 * N + K, dtype=dtype)
                ref, rss = _reference(op)
                worst = max(worst, _check(Call(op), _workspace(M, N), _schedule(M, N, K, sms), ref, rss))
    print(f"[w4a16 bound] tails dtype={str(dtype).split('.')[-1]} max|y-ref|/bound={worst:.3f}")


def _split_case(regime, bn=None):
    for M, N, K, cells in _case_table(_sms()):
        if any(r == regime and (bn is None or b == bn) for b, r in cells):
            return M, N, K
    raise AssertionError((regime, bn))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [BF, F16])
def test_residual_is_one_more_rounding(dtype):
    """y(residual) == round(float(y) + float(residual)) bit for bit, whole-tile and split (the last contributor adds)."""
    for M, N, K in (_split_case("whole", 64), _split_case("slot1", 128), _split_case("count_gt_cb", 16)):
        op = _operands(M, N, K, seed=M + N + K, dtype=dtype)
        res = torch.randn(M, N, generator=torch.Generator().manual_seed(N)).to(dtype)
        plain = Call(op).run(_workspace(M, N)).cpu()
        c = Call(op, residual=res)
        got = c.run(_workspace(M, N)).cpu()
        assert c.pads_intact()
        want = (plain.float() + res.float()).to(dtype)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (M, N, K, dtype)


PAIR_SHAPES = [(17, 256, 256), (32, 768, 512), (100, 256, 256), (128, 384, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", PAIR_SHAPES)
def test_silu_pairs_equal_linear_bf16_silu_pairs(M, N, K):
    """BN 32 and 128, whole tiles on both schedules: the W4 pairs epilogue == linear_bf16_silu_pairs on the dequantised
    interleaved weight, bit for bit; fp16 == SiluAndMul with fp16 roundings of the plain W4 output (<= 1 ulp, the exp)."""
    sms = _sms()
    assert _pick_bn(M) in (32, 128) and _both_whole(M, N, K, sms)
    op = _operands(M, N, K, seed=M * N + K)
    c = Call(op, pairs=True)
    got = c.run(_workspace(M, N)).clone()
    assert c.pads_intact()
    want = _linear16(op, op["w"], M, N, K, pairs=True)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (M, N, K)
    op16 = _operands(M, N, K, seed=M * N + K + 1, dtype=F16)
    plain = Call(op16).run(_workspace(M, N)).float()
    c16 = Call(op16, pairs=True)
    got16 = c16.run(_workspace(M, N))
    g, u = plain[:, 0::2], plain[:, 1::2]
    want16 = ((g / (1.0 + torch.exp(-g))).to(F16).float() * u).to(F16)
    diff = (got16.view(torch.int16).int() - want16.view(torch.int16).int()).abs()
    assert c16.pads_intact() and int(diff.max()) <= 1 and float((diff > 0).float().mean()) < 0.01


@pytest.mark.gpu
def test_deterministic_shared_workspace_and_graph_replay():
    """Two calls give the same bits; split shapes of three BN alternating on one workspace reproduce their first
    results; a captured call replayed with new inputs copied in == the eager calls, bit for bit."""
    shapes = [_split_case("slot1", bn) for bn in (16, 64, 128)]
    calls = [Call(_operands(M, N, K, seed=M + N)) for M, N, K in shapes]
    ws = torch.zeros(max(G._lib().chitu_b200_linear_workspace_bytes(M, N) for M, N, _ in shapes), dtype=torch.uint8,
                     device=DEV)
    first = [c.run(ws).clone() for c in calls]
    assert torch.equal(calls[0].run(ws).view(torch.int16), first[0].view(torch.int16))
    for _ in range(2):
        for c, f in zip(calls, first):
            assert torch.equal(c.run(ws).view(torch.int16), f.view(torch.int16)), (c.M, c.N, c.K)
    assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0

    M, N, K = _split_case("slot1")
    ops = [_operands(M, N, K, seed=100 + i) for i in range(4)]
    call = Call(ops[0])
    ws = torch.zeros(G._lib().chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)

    def load(op):
        for buf, name in ((call.x, "x"), (call.qw, "qweight"), (call.s, "scales"), (call.z, "zeros")):
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
def test_shape_refusals_launch_nothing():
    """A workspace too small: -2 naming the entry, no launch, the workspace untouched."""
    from chitu_b200._lib import launch_count
    M, N, K = 16, 256, 512
    op = _operands(M, N, K, seed=4)
    ws = _workspace(M, N)
    before = launch_count()
    for pairs, name in ((False, "chitu_b200_w4a16_gemm"), (True, "chitu_b200_w4a16_gemm_silu_pairs")):
        c = Call(op, pairs=pairs)
        assert c(ws[:-1]) == -2 and name in G._lib().chitu_b200_last_error().decode()
    torch.cuda.synchronize()
    assert launch_count() == before and bool((ws[TICKET_BYTES:] == 0xFF).all())


# ------------------------------------------------------------------------------------------------------- module
def _module_cases():
    from chitu_b200.quantize import W4A16Linear
    from test_w4a16_cpu import _awq_tensors, _gptq_tensors
    K, N = 512, 384
    _, _, s, qw, qz = _gptq_tensors(K, N, seed=1)
    yield "gptq", W4A16Linear.from_gptq(qw, qz, s)
    _, _, s, qw, qz = _awq_tensors(K, N, seed=2)
    yield "awq", W4A16Linear.from_awq(qw, qz, s, bias=torch.randn(N) * 0.1)
    lin = torch.nn.Linear(K, N, bias=True)
    with torch.no_grad():
        lin.weight.normal_(0, 0.05, generator=torch.Generator().manual_seed(3))
    yield "float", W4A16Linear.from_float(lin, BF)


@pytest.mark.gpu
def test_module_forward_matches_f_linear_on_the_dequantised_weight():
    for name, m in _module_cases():
        m = m.to(DEV)
        w = m.dequantized_weight()
        for shape in ((5, m.in_features), (2, 3, m.in_features), (70, m.in_features)):
            x = (torch.randn(*shape, generator=torch.Generator().manual_seed(len(shape)), device="cpu") * 0.5)
            x = x.to(m.dtype).to(DEV)
            for bias in (m.bias, None):
                saved, m.bias = m.bias, bias
                y = m(x)
                m.bias = saved
                assert y.shape == (*shape[:-1], m.out_features) and y.dtype == m.dtype
                ref = F.linear(x.double(), w.double(), None if bias is None else bias.double())
                rss = ((x.double() ** 2) @ (w.double() ** 2).T).sqrt()
                u = U_OUT[m.dtype]
                # one rounding of the product, one more for the bias add
                bound = 2 * u * ref.abs() + TAU_FP32 * rss + (0 if bias is None else u * bias.double().abs())
                err = (y.double() - ref).abs()
                assert bool((err <= bound).all()), (name, shape, bias is None, float((err / bound).max()))


# ------------------------------------------------------------------------------------------------------- engine
def _llama(weight_format, B, S, n_layers=2):
    import dataclasses

    from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
    cfg = dataclasses.replace(LLAMA3_8B, n_layers=n_layers)
    eng = LlamaDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, device=DEV, page_size=256,
                            weight_format=weight_format)
    eng.set_synthetic_context(S)
    return cfg, eng


@pytest.mark.gpu
def test_llama3_8b_w4a16_two_layer_step_vs_torch_ref():
    """Full-width LLaMA-3-8B, 2 layers, bs 16: the W4 engine's logits against tests/torch_ref.llama_decode_step over
    ref_layers() (the dequantised weights), with the full-width test's noise-floor tolerance."""
    from test_fullwidth_gpu import _ulp_perturb
    B, S = 16, 1024
    cfg, eng = _llama("w4a16", B, S)
    lens = torch.full((B,), S, dtype=torch.int32)
    lens[1], lens[2] = 255, 256
    eng.seq_lens.copy_(lens)
    tokens = torch.randint(100, 1000, (B,), generator=torch.Generator().manual_seed(0))
    kc = [eng.k_cache[l].clone() for l in range(cfg.n_layers)]
    vc = [eng.v_cache[l].clone() for l in range(cfg.n_layers)]
    ln = eng.seq_lens.clone()
    cos, sin = eng.cos_table[ln.long()], eng.sin_table[ln.long()]
    layers = eng.ref_layers()
    for lw in layers:
        assert all(lw[n].dtype == BF for n in ("wqkv", "wo", "w13", "w2"))
    ref = R.llama_decode_step(layers, eng.embed, eng.norm, eng.head, tokens.to(DEV), [c.clone() for c in kc],
                              [c.clone() for c in vc], ln, eng.block_table, cos, sin, cfg.n_heads, cfg.n_kv_heads,
                              cfg.norm_eps)
    ref2 = R.llama_decode_step(layers, _ulp_perturb(eng.embed, torch.Generator(device=DEV).manual_seed(1)), eng.norm,
                               eng.head, tokens.to(DEV), kc, vc, ln, eng.block_table, cos, sin, cfg.n_heads,
                               cfg.n_kv_heads, cfg.norm_eps)
    floor_mr, floor_cd = max_rel(ref2, ref), cos_diff(ref2, ref)
    eng.decode(tokens.pin_memory())
    torch.cuda.synchronize()
    got = eng.logits.float()
    mr, cd = max_rel(got, ref), cos_diff(got, ref)
    print(f"llama-3-8b w4a16 2 layers: logits max_rel {mr:.3e} (floor {floor_mr:.3e}) cos_diff {cd:.3e} "
          f"(floor {floor_cd:.3e})")
    assert mr < max(1e-2, 3 * floor_mr) and mr < 0.1
    assert cd < max(1e-4, 3 * floor_cd) and cd < 5e-3


@pytest.mark.gpu
def test_llama3_8b_w4a16_graph_replay_equals_eager():
    """A run of decode steps: graph replay bit-identical to eager (logits, next tokens, KV caches, lengths), and the
    captured step has the bf16 engine's launch count."""
    B, S, steps = 4, 600, 4
    _, eager = _llama("w4a16", B, S)
    _, graph = _llama("w4a16", B, S)
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
        assert torch.equal(c_e.view(torch.int16), c_g.view(torch.int16))
    del eager
    _, bf = _llama("bf16", B, S)
    bf.capture()
    assert graph.launches_per_step == bf.launches_per_step > 0
