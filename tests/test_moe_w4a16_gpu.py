"""4-bit MoE experts (chitu_b200_fused_experts_w4a16: the grouped path of csrc/moe.cu with `tc_gemm_kernel<KIND_W4>` in
grouped mode) against fp64 references over the exact dequantised weights, with the host model of
tests/test_moe_dispatch_gpu.py (plan, stream-K split, regimes, workspace layout and read-back) at W4's stages of 128
K-elements, and the Mixtral-8x7B engine built on it.

Every expert and every weight row carries its own scales and zeros, and the experts no token is routed to hold NaN
scales: a kernel that read another expert's or another row's scale row (as a clamp to one expert's width would) fails
the bound or turns the output NaN."""
import functools

import numpy as np
import pytest
import torch

import test_moe_dispatch_gpu as M
import torch_ref as R
from conftest import cos_diff, max_rel
from test_gemm_dispatch_gpu import NAN_BYTE, SENTINEL, TICKET_BYTES, Padded
from test_pdl_ordering_gpu import run_case, slow_row  # noqa: F401  (slow_row is a fixture)

pytestmark = pytest.mark.gpu
BF, F32, U8 = torch.bfloat16, torch.float32, torch.uint8
DEV = "cuda:0"
W4 = "w4"          # the host model's weight mode: any mode but "bf16" has 128 K-elements per stage, "soft" the same shapes


# ------------------------------------------------------------------------------------------------ case table
@functools.lru_cache(maxsize=None)
def _case_table(sms):
    """One routing per reachable grouped (BN x plan x GEMM x regime) cell at W4 stages (the soft-fp8 search: the same
    stage counts and shape domain), then the routing extras (shared expert, E = 1, P = 1, every pair absent,
    duplicates); ids / weight dtypes and the residual rotate."""
    cases = []
    shapes = {}
    for (_, _, *cell), (_, *shape) in sorted(M._search("soft", sms).items()):
        shapes.setdefault(tuple(shape), set()).add((W4, "grouped", *cell))
    for i, ((T, topk, E, N1, K1, na), cells) in enumerate(shapes.items()):
        cases.append(dict(wmode=W4, T=T, topk=topk, E=E, N1=N1, K1=K1, routing="chunks", na=na,
                          ids_dtype=(torch.int32, torch.int64)[i % 2], tw_dtype=(BF, F32)[(i // 2) % 2],
                          residual=(i // 4) % 2 == 1, cell=frozenset(cells)))
    for T, topk, E, N1, K1, routing, idt, twt, res in M.GROUPED_EXTRAS:
        cases.append(dict(wmode=W4, T=T, topk=topk, E=E, N1=N1, K1=K1, routing=routing, na=None, ids_dtype=idt,
                          tw_dtype=twt, residual=res, cell=None))
    for i, c in enumerate(cases):
        c["seed"] = 5000 + i
    return tuple(cases)


def _cells(case, sms):
    return {(W4, *c[1:]) for c in M._case_cells(dict(case, wmode=W4), sms)}


# ---------------------------------------------------------------------------------------------------- operands
def _stack(E, N, K, active, g, zeros=True):
    """(qweight [E, N, K/2], scales [E, N, K/128] bf16, zeros [E, N, K/128] or None, dequantised [E, N, K] bf16) with
    weights for the `active` experts only: q and z uniform over 0..15 with both extremes in every expert, scales
    0.005..0.015 per row and group.  Every other expert has NaN scales (and a NaN reference)."""
    from chitu_b200.quantize import w4a16 as W
    na = active.numel()
    qw = torch.full((E, N, K // 2), 0x88, dtype=U8)
    s = torch.full((E, N, K // 128), float("nan"), dtype=BF)
    z = torch.full((E, N, K // 128), 8, dtype=U8)
    ref = torch.full((E, N, K), float("nan"), dtype=BF)
    if na:
        q = torch.randint(0, 16, (na, N, K), generator=g)
        q[:, 0, 0], q[:, -1, -1] = 0, 15
        za = torch.randint(0, 16, (na, N, K // 128), generator=g).to(U8)
        za[:, 0, 0], za[:, -1, -1] = 0, 15
        qw[active] = W.pack_rows(q.view(na * N, K)).view(na, N, K // 2)
        s[active] = ((torch.rand(na, N, K // 128, generator=g) + 0.5) * 0.01).to(BF)
        if zeros:
            z[active] = za
        ref[active] = W.dequantize(qw[active], s[active], z[active])
    return qw, s, (z if zeros else None), ref


def _operands(case, zeros=True):
    """The host model's routing and activations (M._operands with bf16 weights) and 4-bit expert stacks."""
    T, topk, E, N1, K1 = (case[k] for k in ("T", "topk", "E", "N1", "K1"))
    op = M._operands(dict(case, wmode="bf16", N1=128 * 2, K1=K1, E=1, routing="absent"))   # x, residual
    g = torch.Generator().manual_seed(case["seed"] + 77)
    ids, w = M._routing(case)
    active = torch.tensor(sorted({int(e) for e in ids.reshape(-1) if 0 <= e < E}), dtype=torch.long)
    op.update(case=case, ids=torch.from_numpy(ids).to(case["ids_dtype"]), tw=torch.from_numpy(w).to(case["tw_dtype"]))
    op["tw32"] = op["tw"].float()
    op["w1"], op["w1_sc"], op["w1_z"], op["w1r"] = _stack(E, N1, K1, active, g, zeros)
    op["w2"], op["w2_sc"], op["w2_z"], op["w2r"] = _stack(E, K1, N1 // 2, active, g, zeros)
    op["w1_s"] = op["w2_s"] = None         # the host model's fp8 block scales
    return op


class W4Call:
    """chitu_b200_fused_experts_w4a16 on buffers the test owns; x and out between NaN / sentinel pads."""

    def __init__(self, op):
        c = self.c = op["case"]
        self.op = op
        self.x = Padded(op["x"])
        d = lambda t: None if t is None else t.to(DEV)                       # noqa: E731
        self.w = [d(op[k]) for k in ("w1", "w1_sc", "w1_z", "w2", "w2_sc", "w2_z")]
        self.ids, self.tw = op["ids"].to(DEV), op["tw"].to(DEV)
        self.res = None if op["res"] is None else Padded(op["res"])
        self.out = Padded(torch.empty(c["T"], c["K1"], dtype=BF), pad=SENTINEL, fill=NAN_BYTE)

    def __call__(self, ws, nbytes=None, T=None, res=True):
        from chitu_b200._lib import current_stream, dtype_code, ptr
        c = self.c
        return M._lib().chitu_b200_fused_experts_w4a16(
            ptr(self.x.view), *[ptr(t) for t in self.w], ptr(self.tw), dtype_code(self.tw.dtype), ptr(self.ids),
            dtype_code(self.ids.dtype), c["T"] if T is None else T, c["topk"], c["E"], c["N1"], c["K1"], ptr(self.out.view),
            None if (self.res is None or not res) else ptr(self.res.view), ptr(ws), ws.numel() if nbytes is None else nbytes,
            current_stream())

    def run(self, ws, res=True):
        from chitu_b200._lib import check
        check(self(ws, res=res), f"fused_experts_w4a16 T={self.c['T']} E={self.c['E']}")
        torch.cuda.synchronize()
        return self.out.view


def _ws(c):
    return M._fresh_ws(M._lib().chitu_b200_moe_workspace_bytes(c["T"], c["topk"], c["E"], c["N1"], c["K1"]))


def _run_case(case, sms):
    op = _operands(case)
    c = case
    call = W4Call(op)
    ws = _ws(c)
    out = call.run(ws)
    what = (c["T"], c["topk"], c["E"], c["N1"], c["K1"], c["routing"])
    assert call.x.pads_intact() and call.out.pads_intact() and (call.res is None or call.res.pads_intact()), what
    assert bool(torch.isfinite(out).all()), ("non-finite output",) + what
    assert int(ws[:TICKET_BYTES].count_nonzero()) == 0, ("tickets left non-zero",) + what
    path, got = M._read_ws(ws, c, sms)
    assert path == "grouped"
    got["out"] = out
    BN = M._chunk_rows(c["T"] * c["topk"], c["E"])
    pl = M._moe_plan(op["ids"].numpy(), op["tw32"].numpy(), c["E"], BN, c["N1"], c["K1"])
    stats = M._check_grouped(op, got, pl)
    assert M._written_slots(ws, BN, sms) == M._model_slots(pl, W4, c["N1"], c["K1"], sms), \
        ("partial slots differ from the grouped split model",) + what
    return op, out.clone(), stats


def test_fused_experts_w4a16_stage_by_stage():
    """Every case: plan exact, gathered rows bit-exact, c1 and c3 inside the fp32-accumulation bound over the
    dequantised weights, a2 within one ulp per rounding, the combine bit-exact, pads and tickets intact, the partial
    slots as the split model says.  Every reachable (BN x plan x GEMM x regime) cell is reached."""
    sms = M._sms()
    seen, worst = set(), {}
    for case in _case_table(sms):
        _, _, stats = _run_case(case, sms)
        cells = _cells(case, sms)
        if case["cell"] is not None:
            assert cells >= case["cell"], (case, cells)
        seen |= cells
        for k, v in stats.items():
            worst[k] = max(worst.get(k, 0.0), v)
    want = {(W4, "grouped", bn, pl, g, r) for bn in M.BNS for pl in M.PLANS for g in (1, 2) for r in M.REGIMES}
    want -= {(W4, "grouped", 128, pl, g, r) for pl in M.PLANS for g in (1, 2) for r in ("slot0", "slot1")}
    assert seen == want, sorted(want - seen)
    print(f"[moe w4 bound] cases={len(_case_table(sms))} " + " ".join(f"{k}={v:.3f}" for k, v in sorted(worst.items())))


def _both_whole(c, sms):
    """The host model gives every launch of both kinds whole tiles: W4 (K / 128 stages) and bf16 (K / 64)."""
    if c["routing"] != "chunks":
        return False
    P = c["T"] * c["topk"]
    BN = M._chunk_rows(P, c["E"])
    pl = M._moe_plan(*M._routing(c), c["E"], BN, c["N1"], c["K1"])
    return all(M._regime(nt, M._stages(w, K), BN, sms) == "whole"
               for w in (W4, "bf16") for nt, K in ((pl["num_tiles1"], c["K1"]), (pl["num_tiles2"], c["N1"] // 2)))


def test_whole_tiles_bit_identical_to_bf16_on_the_dequantised_weights():
    """Where both kinds' GEMMs run whole tiles, W4 and bf16 issue the same wgmma sequence over the same operand values
    into one fp32 accumulator: chitu_b200_fused_experts (bf16, on the dequantised stacks) gives the same bits."""
    sms = M._sms()
    cases = [c for c in _case_table(sms) if _both_whole(c, sms)]
    assert len(cases) >= 3, len(cases)
    for case in cases:
        op = _operands(case)
        got = W4Call(op).run(_ws(case)).clone()
        bop = dict(op, case=dict(case, wmode="bf16"), w1=op["w1r"], w2=op["w2r"])
        want = M.FusedCall(bop).run(_ws(case))
        assert M._same_bits(got, want), (case["T"], case["E"], case["N1"], case["K1"])


def test_null_zeros_equal_zeros_of_eight():
    sms = M._sms()
    for case in [c for c in _case_table(sms) if c["routing"] == "chunks"][:4] + [_case_table(sms)[-5]]:
        a = _operands(case, zeros=False)
        b = dict(a, w1_z=torch.full_like(a["w1_sc"], 8, dtype=U8), w2_z=torch.full_like(a["w2_sc"], 8, dtype=U8))
        ca, cb = W4Call(a), W4Call(b)
        assert ca.w[2] is None and ca.w[5] is None
        assert M._same_bits(ca.run(_ws(case)).clone(), cb.run(_ws(case))), case["seed"]


def test_residual_is_one_more_rounding():
    sms = M._sms()
    for case in [c for c in _case_table(sms) if c["residual"]][:4]:
        op = _operands(case)
        call = W4Call(op)
        plain = call.run(_ws(case), res=False).clone()
        got = call.run(_ws(case))
        want = (plain.float() + op["res"].to(DEV).float()).to(BF)
        assert M._same_bits(got, want), case["seed"]


def test_deterministic_shared_workspace_and_graph_replay():
    """Three cases of different P and E alternating on one workspace reproduce their first results; a captured call
    replayed after new routing (other experts, chunk counts, all absent) and new weights are copied in equals the eager
    calls bit for bit."""
    sms = M._sms()
    table = [c for c in _case_table(sms) if c["routing"] == "chunks"]
    picks = [next(c for c in table if any(x[2:4] == key for x in c["cell"])) for key in ((16, "small"), (128, "large"),
                                                                                          (32, "large"))]
    calls = [W4Call(_operands(c)) for c in picks]
    nbytes = max(M._lib().chitu_b200_moe_workspace_bytes(c["T"], c["topk"], c["E"], c["N1"], c["K1"]) for c in picks)
    ws = M._fresh_ws(nbytes)
    first = [call.run(ws).clone() for call in calls]
    for _ in range(2):
        for call, f in zip(calls, first):
            assert M._same_bits(call.run(ws), f), (call.c["T"], call.c["E"])
    assert int(ws[:TICKET_BYTES].count_nonzero()) == 0

    base = dict(wmode=W4, T=40, topk=3, E=8, N1=256, K1=256, routing="shared", na=None, ids_dtype=torch.int32,
                tw_dtype=F32, residual=True, seed=9)
    call = W4Call(_operands(base))
    ws = _ws(base)
    variants = [dict(base, routing="random", seed=10), dict(base, routing="chunks", na=3, seed=11),
                dict(base, routing="absent", seed=12)]
    ops = [_operands(v) for v in variants]

    def load(op):
        call.ids.copy_(op["ids"].to(torch.int32))
        call.tw.copy_(op["tw"])
        for t, k in zip(call.w, ("w1", "w1_sc", "w1_z", "w2", "w2_sc", "w2_z")):
            t.copy_(op[k].nan_to_num(0.01) if t.dtype == BF else op[k])    # every expert finite: routing B may use it

    eager = []
    for op in ops:
        load(op)
        eager.append(call.run(ws).clone())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call(ws)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(ws)
    for op, want in zip(ops, eager):
        load(op)
        call.out.view.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert M._same_bits(call.out.view, want)
    assert int(ws[:TICKET_BYTES].count_nonzero()) == 0


def test_refusals_launch_nothing():
    """More than 8192 pairs (no 4-bit path beyond the grouped one), a workspace one byte short and shapes the grouped
    path cannot take return a status, launch nothing and leave the workspace and the output alone."""
    from chitu_b200._lib import launch_count
    base = dict(wmode=W4, T=6, topk=2, E=4, N1=256, K1=256, routing="random", na=None, ids_dtype=torch.int32,
                tw_dtype=BF, residual=False, seed=3)
    before = launch_count()
    for over in (dict(T=4097, topk=2, K1=128), dict(), dict(N1=384), dict(K1=192)):
        case = dict(base, **over)
        op = _operands(case) if not ({"N1", "K1"} & set(over)) else _operands(base)
        call = W4Call(dict(op, case=case))
        need = M._lib().chitu_b200_moe_workspace_bytes(case["T"], case["topk"], case["E"], case["N1"], case["K1"])
        ws = M._fresh_ws(need)
        rc = call(ws, need - 1 if not over else need)
        torch.cuda.synchronize()
        assert rc != 0 and M._last_error(), over
        assert bool((ws[TICKET_BYTES:] == NAN_BYTE).all()), over
        assert bool((call.out.view.view(torch.int16) == -1).all()), over
    assert launch_count() == before


# ------------------------------------------------------------------------------------------------- launch order
def test_w4_experts_directly_after_the_gate_that_routes_them(slow_row):  # noqa: F811
    """moe_gate writes the routing while the experts' plan kernel is already resident behind it (a slow predecessor
    holds the gate in its wait): back to back on one stream and replayed from a graph, the result equals the same
    launches synchronised one by one (tests/test_pdl_ordering_gpu.py's harness)."""
    from chitu_b200 import _lib
    from chitu_b200._lib import current_stream, ptr
    T, topk, E, N1, K1 = 16, 2, 8, 512, 256
    case = dict(wmode=W4, T=T, topk=topk, E=E, N1=N1, K1=K1, routing="random", na=None, ids_dtype=torch.int64,
                tw_dtype=BF, residual=True, seed=21)
    op = _operands(case)
    op["w1_sc"], op["w2_sc"] = op["w1_sc"].nan_to_num(0.01), op["w2_sc"].nan_to_num(0.01)
    gate_w = (torch.randn(E, K1, generator=torch.Generator().manual_seed(1)) * 0.05).to(BF).to(DEV)
    lib = _lib.load()

    def build():
        s = dict(x=op["x"].to(DEV), res=op["res"].to(DEV), out=torch.full((T, K1), -1, dtype=torch.int16, device=DEV).view(BF),
                 tw=torch.full((T, topk), -1, dtype=torch.int16, device=DEV).view(BF),
                 ids=torch.full((T, topk), -1, dtype=torch.int64, device=DEV),
                 gws=torch.zeros(lib.chitu_b200_moe_gate_workspace_bytes(T, E), dtype=U8, device=DEV),
                 ws=torch.zeros(lib.chitu_b200_moe_workspace_bytes(T, topk, E, N1, K1), dtype=U8, device=DEV))
        s["w"] = [op[k].to(DEV) for k in ("w1", "w1_sc", "w1_z", "w2", "w2_sc", "w2_z")]
        return s

    def gate(s):
        _lib.check(lib.chitu_b200_moe_gate(ptr(s["x"]), ptr(gate_w), None, 0, T, K1, E, 1, 1, topk, 2, 1.0, ptr(s["tw"]),
                                           ptr(s["ids"]), topk, ptr(s["gws"]), s["gws"].numel(), current_stream()), "gate")

    def experts(s):
        _lib.check(lib.chitu_b200_fused_experts_w4a16(
            ptr(s["x"]), *[ptr(t) for t in s["w"]], ptr(s["tw"]), _lib.CB_BF16, ptr(s["ids"]), _lib.CB_I64, T, topk, E,
            N1, K1, ptr(s["out"]), ptr(s["res"]), ptr(s["ws"]), s["ws"].numel(), current_stream()), "experts")

    ref = run_case((build, gate, experts), slow_row)
    assert bool(torch.isfinite(ref["out"].view(BF)).all())


# ------------------------------------------------------------------------------------------------------ engine
def _mixtral(n_layers, B, S):
    from chitu_b200.engine_mixtral import MixtralConfig, MixtralDecodeEngine
    cfg = MixtralConfig(n_layers=n_layers)
    eng = MixtralDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, device=DEV, tp_size=1, weight_format="w4a16")
    eng.set_synthetic_context(S)
    return cfg, eng


def _eager_then_graph(eng, tokens):
    """Logits of one eager step, then of the same step captured and replayed from the same state."""
    saved = eng.seq_lens.clone()
    eng.decode(tokens.pin_memory())
    torch.cuda.synchronize()
    eager = eng.logits.clone()
    eng.seq_lens.copy_(saved)
    eng.capture()
    eng.decode(tokens.pin_memory())
    torch.cuda.synchronize()
    return eager, eng.logits.clone()


def test_mixtral_8x7b_w4a16_two_layers_vs_torch_ref():
    """Full-width Mixtral-8x7B, 2 layers, tp_size=1, bs 16, S 4096: the W4 engine's logits against tests/torch_ref's
    Mixtral layers over ref_layers() (the dequantised weights), within the bound of
    test_fullwidth_gpu.test_mixtral_engine_step_vs_torch_ref; graph replay equals eager bit for bit.  At full width a
    token's top-2 can flip between two experts whose router probabilities tie to rounding noise.  The noise is measured
    in the same test: how far a one-ulp perturbation of the embedding moves the reference's router probabilities in each
    layer (relative to the token's 2nd probability, over tokens the perturbation routed alike in the earlier layers).  A flipped token must have a reference margin between its 2nd and
    3rd probability below three times that, and is left out of the logit comparison (decode rows are independent);
    every other token's routing must be identical."""
    from test_fullwidth_gpu import _ulp_perturb
    B, S = 16, 4096
    cfg, eng = _mixtral(2, B, S)
    lens = torch.full((B,), S, dtype=torch.int32)
    lens[1], lens[2], lens[3] = 255, 256, 1000
    eng.seq_lens.copy_(lens)
    tokens = torch.randint(100, 1000, (B,), generator=torch.Generator().manual_seed(0))
    kc0 = [eng.k_cache[l].clone() for l in range(cfg.n_layers)]
    vc0 = [eng.v_cache[l].clone() for l in range(cfg.n_layers)]
    ln = eng.seq_lens.clone()
    cos, sin = eng.cos_table[ln.long()], eng.sin_table[ln.long()]
    layers = eng.ref_layers()
    assert all(lw[n].dtype == BF and lw[n].dim() == d for lw in layers for n, d in (("wqkv", 2), ("w1", 3), ("w2", 3)))

    def reference(embed):
        h, routes = embed[tokens.to(DEV)], []
        for li, lw in enumerate(layers):
            r = []
            h = R.mixtral_layer(lw, h, kc0[li].clone(), vc0[li].clone(), ln, eng.block_table, cos, sin, eng.Hq, eng.Hkv,
                                eng.topk, cfg.norm_eps, route_out=r)
            routes.append(r[0])
        return R.final_logits(h, eng.norm, eng.head, cfg.norm_eps), routes

    def same_rows(ids, routes):
        """Per token: the same experts in every layer."""
        ok = torch.ones(B, dtype=torch.bool, device=DEV)
        for a, (b, _) in zip(ids, routes):
            ok &= (a.sort(dim=-1)[0] == b.sort(dim=-1)[0]).all(dim=-1)
        return ok

    ref, routes = reference(eng.embed)
    perturbed = [reference(_ulp_perturb(eng.embed, torch.Generator(device=DEV).manual_seed(seed))) for seed in range(1, 7)]
    eager, graph = _eager_then_graph(eng, tokens)
    assert torch.equal(eager.view(torch.int16), graph.view(torch.int16))
    keep = same_rows([eng.gate_i_all[li] for li in range(cfg.n_layers)], routes)
    for li, (ids, probs) in enumerate(routes):
        top = probs.float().sort(dim=-1, descending=True)[0]
        second = top[:, eng.topk - 1]
        # over the tokens whose earlier layers the perturbation routed alike (a flip upstream is not rounding noise)
        noise = max(float(((p2[li][1].float() - probs.float()).abs().amax(dim=-1) / second)[same_rows(
            [r[0] for r in p2[:li]], routes[:li])].max()) for _, p2 in perturbed)
        margin = (second - top[:, eng.topk]) / second
        flipped = ~(eng.gate_i_all[li].sort(dim=-1)[0] == ids.sort(dim=-1)[0]).all(dim=-1)
        print(f"layer {li}: {int(flipped.sum())} tokens routed differently, margins {margin[flipped].tolist()}, "
              f"router noise of a one-ulp perturbation {noise:.3e}")
        assert bool((margin[flipped] < 3 * noise).all()), (li, margin[flipped].tolist(), noise)
    assert int(keep.sum()) >= B - 2, keep.tolist()
    floor = None
    for ref2, routes2 in perturbed:
        if bool((same_rows([r[0] for r in routes2], routes) | ~keep).all()):
            floor = (max_rel(ref2[keep], ref[keep]), cos_diff(ref2[keep], ref[keep]))
            break
    got = eager.float()[keep]
    mr, cd = max_rel(got, ref[keep]), cos_diff(got, ref[keep])
    floor_mr, floor_cd = floor if floor is not None else (1e-2, 1e-4)
    print(f"mixtral-8x7b w4a16 tp1, 2 layers, {int(keep.sum())} of {B} tokens routed alike: logits max_rel {mr:.3e} "
          f"(floor {floor_mr:.3e}) cos_diff {cd:.3e} (floor {floor_cd:.3e})")
    assert mr < max(1e-2, floor_mr) and mr < 0.15
    assert cd < max(1e-4, floor_cd) and cd < 2e-3


def test_mixtral_8x7b_w4a16_full_model_on_one_gpu():
    """All 32 layers of Mixtral-8x7B in W4 at tp_size=1 build on one 80 GB GPU (each layer quantised as it is
    generated) and run a captured step at bs 16, S 4096: finite logits, equal to the eager step."""
    B, S = 16, 4096
    torch.cuda.empty_cache()
    cfg, eng = _mixtral(32, B, S)
    print(f"mixtral-8x7b w4a16 32 layers: {torch.cuda.memory_allocated() / 1e9:.1f} GB allocated, "
          f"peak {torch.cuda.max_memory_allocated() / 1e9:.1f} GB")
    tokens = torch.randint(100, 1000, (B,), generator=torch.Generator().manual_seed(1))
    eager, graph = _eager_then_graph(eng, tokens)
    assert bool(torch.isfinite(eager.float()).all())
    assert torch.equal(eager.view(torch.int16), graph.view(torch.int16))
    assert eng.launches_per_step > 0
    del eng
    torch.cuda.empty_cache()
