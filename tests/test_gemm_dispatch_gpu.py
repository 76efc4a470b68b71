"""The decode GEMM (`tc_gemm_kernel<KIND, BN, EPI>`, csrc/gemm_tc.cu) and its SIMT fallback (csrc/gemv.cu) against an
fp64 reference of the exact operand values, on shapes chosen by a restatement of the host schedule of `run()`.

`_schedule` restates `run()`: the token tile BN, the stream-K split of the stage list over the CTAs, the whole-tile vs
split choice, every split tile's contributors and the partial slot each contributor fills.  The case table holds one
shape per (weight kind x BN x regime) cell the schedule can reach; the GPU tests run it through the C entries with
buffers they own, and read the workspace back to check that the kernel split and reduced exactly as the model says.

The bound: every element satisfies |y - ref| <= u_out |ref| + tau rss, rss = sqrt(sum_k t_k^2) over the scaled products
t_k.  u_out is the output rounding (bf16 2^-8, fp16 2^-11); tau covers the accumulation: 2^-13 for fp32-accumulating
paths, 2^-8 for the fp8 wgmma path (Hopper's fp8 MMA is reported to accumulate with ~14 bits; not measured for this
kernel).  `test_bound_rejects_injected_errors` shows that the bound is tight enough to see a dropped stage, a wrong
activation scale, a dropped bias and a missing split contributor.  int8 results are exact integers scaled in fp32, so
they are compared bit for bit."""
import functools
import math

import pytest
import torch

from oracle import chitu_oracle as O

BF, F16, F8 = torch.bfloat16, torch.float16, torch.float8_e4m3fn
DEV = "cuda:0"

# ---------------------------------------------------------------------------------------------- schedule model
KINDS = ("16", "fp8", "soft", "i8")          # bf16 / fp16 weights, fp8 block-scaled, soft fp8 (W8A16), int8 (W8A8)
BNS = (16, 32, 64, 128)
CB = {16: 8, 32: 4, 64: 2, 128: 1}           # split contributors the last arriver reads per round trip
REGIMES = ("whole", "slot0", "slot1", "count_gt_cb", "m_chunks")
M_EDGES = {16: (1, 16), 32: (17, 32), 64: (33, 64), 128: (65, 128, 129, 256)}
STAGE_K = {"16": 64, "fp8": 128, "soft": 128, "i8": 128}     # K elements per 128-byte pipeline stage
MAX_STAGES = {"16": 65, "fp8": 32, "soft": 32, "i8": 32}     # search domain: K up to 4160 (16-bit) / 4096
MAX_N_TILES = 17                                             # search domain: N up to 2176
TICKET_BYTES = 65536 * 2 * 4                                 # Params::tickets, before the partial slots
# m_chunks > 1 needs M > BN, and only BN = 128 serves more than one token tile's worth of M
UNREACHABLE = tuple((k, bn, "m_chunks") for k in KINDS for bn in (16, 32, 64))


def _cdiv(a, b):
    return -(-a // b)


def _pick_bn(M):
    return 16 if M <= 16 else 32 if M <= 32 else 64 if M <= 64 else 128


@functools.lru_cache(maxsize=None)
def _split(BN, m_chunks, n_tiles, S, sms):
    """The kind-independent part of `run()`: (grid, per, {split tile: ((cta, slot, s_lo, s_hi), ...)})."""
    tiles = n_tiles * m_chunks
    total = tiles * S
    grid = min(sms, total)
    if total // grid < 4:
        grid = max(total // 4, 1)
    per = _cdiv(total, grid)
    if per * 8 < S:
        per = _cdiv(S, 8)
    grid = _cdiv(total, per)
    whole_per = S * _cdiv(tiles, sms)
    if per % S != 0 and 0.15 * whole_per <= 0.15 * per + 3.5:    # a split costs ~3.5 us, a 16 KB stage ~0.15 us
        per = whole_per
        grid = _cdiv(total, per)
    items = {}
    for c in range(grid):
        g, g_end = min(c * per, total), min(c * per + per, total)
        while g < g_end:
            t = g // S
            s_lo = g - t * S
            s_hi = min(S, s_lo + g_end - g)
            # a CTA keeps the partial of its first work item in slot 0 and of any later one in slot 1
            items.setdefault(t, []).append((c, 0 if (c * per) // S == t else 1, s_lo, s_hi))
            g += s_hi - s_lo
    split = {t: tuple(v) for t, v in items.items() if len(v) > 1}
    for t, v in split.items():        # the kernel's contributor range of a tile
        assert len(v) == ((t + 1) * S - 1) // per - (t * S) // per + 1
    return grid, per, split


def _schedule(kind, M, N, K, sms):
    """Host arithmetic of `run()` (csrc/gemm_tc.cu) with a full workspace."""
    BN = _pick_bn(M)
    S = _cdiv(K * (2 if kind == "16" else 1), 128)
    n_tiles, m_chunks = _cdiv(N, 128), _cdiv(M, BN)
    grid, per, split = _split(BN, m_chunks, n_tiles, S, sms)
    slots = {(c, slot) for v in split.values() for c, slot, _, _ in v}
    regimes = set()
    if not split:
        regimes.add("whole")
    else:
        regimes.add("slot1" if any(slot for _, slot in slots) else "slot0")
        if max(len(v) for v in split.values()) > CB[BN]:
            regimes.add("count_gt_cb")
        if m_chunks > 1:
            regimes.add("m_chunks")
    return dict(BN=BN, S=S, n_tiles=n_tiles, m_chunks=m_chunks, grid=grid, per=per, split=split, slots=slots,
                regimes=regimes)


@functools.lru_cache(maxsize=None)
def _case_table(sms):
    """One (kind, M, N, K) per reachable (kind, BN, regime) cell: the smallest weight that keeps more than one CTA
    busy, M rotating over the BN edges."""
    cases = {}
    for kind in KINDS:
        best = {}                                   # (BN, regime, M) -> (one CTA only, weight elements, N, K)
        for M in sorted({m for ms in M_EDGES.values() for m in ms}):
            for nt in range(1, MAX_N_TILES + 1):
                for S in range(1, MAX_STAGES[kind] + 1):
                    N, K = nt * 128, S * STAGE_K[kind]
                    sc = _schedule(kind, M, N, K, sms)
                    cost = (sc["grid"] < 2, N * K, N, K)
                    for r in sc["regimes"]:
                        key = (sc["BN"], r, M)
                        if key not in best or cost < best[key]:
                            best[key] = cost
        for BN in BNS:
            for ri, r in enumerate(REGIMES):
                hits = {M: best[(BN, r, M)] for M in M_EDGES[BN] if (BN, r, M) in best}
                if not hits:
                    continue
                want = M_EDGES[BN][ri % len(M_EDGES[BN])]
                M = want if want in hits else min(hits, key=lambda m: hits[m])
                _, _, N, K = hits[M]
                cases.setdefault((kind, M, N, K), set()).add((BN, r))
    return tuple((kind, M, N, K, frozenset(cells)) for (kind, M, N, K), cells in cases.items())


def _cells(table):
    return {(kind, bn, r) for kind, _, _, _, cells in table for bn, r in cells}


@pytest.mark.parametrize("sms", [132, 114])
def test_case_table_covers_every_reachable_cell(sms):
    """The table has a case for every cell any shape of the search domain reaches (a cell reached anywhere gets a
    case), so equality with everything but UNREACHABLE also says the UNREACHABLE cells are reached nowhere."""
    table = _case_table(sms)
    everything = {(k, bn, r) for k in KINDS for bn in BNS for r in REGIMES}
    assert _cells(table) == everything - set(UNREACHABLE)
    for kind, M, N, K, cells in table:               # every case really is in the cells it stands for
        sc = _schedule(kind, M, N, K, sms)
        assert {(sc["BN"], r) for r in sc["regimes"]} >= cells
        assert M in M_EDGES[sc["BN"]] and N <= MAX_N_TILES * 128 and K <= 4160


def test_schedule_model_invariants():
    """Every stage of a split tile is covered exactly once; a CTA's slot 0 holds its first work item and slot 1 its
    last; a launch never uses more CTAs (partial slot pairs) than the device has SMs."""
    for sms in (132, 114):
        for kind, M, N, K, _ in _case_table(sms):
            sc = _schedule(kind, M, N, K, sms)
            S, per, total = sc["S"], sc["per"], sc["n_tiles"] * sc["m_chunks"] * sc["S"]
            assert sc["grid"] <= sms
            for t, v in sc["split"].items():
                covered = sorted((lo, hi) for _, _, lo, hi in v)
                assert covered[0][0] == 0 and covered[-1][1] == S
                assert all(a[1] == b[0] for a, b in zip(covered, covered[1:]))
                for c, slot, _, _ in v:
                    first, last = (c * per) // S, (min(c * per + per, total) - 1) // S
                    assert t == (first if slot == 0 else last) and (slot == 0 or first != last)


# ------------------------------------------------------------------------------------------- reference and bound
U_OUT = {BF: 2.0 ** -8, F16: 2.0 ** -11}
TAU_FP32 = 2.0 ** -13          # fp32 accumulation: 16-bit and soft-fp8 wgmma, every SIMT kernel
TAU_FP8_MMA = 2.0 ** -8        # fp8 wgmma


def _tau(kind, impl):
    return TAU_FP8_MMA if kind == "fp8" and impl != 1 else TAU_FP32


def _quant_fp8_act(af):
    """per_token_group_quant_fp8 over 128-wide groups; a partial last group is padded with zeros."""
    M, K = af.shape
    kb = _cdiv(K, 128)
    ap = torch.zeros(M, kb * 128)
    ap[:, :K] = af
    q, s = O.per_token_group_quant_fp8(ap, 128)
    return q[:, :K].contiguous(), s.contiguous()


def _fp8_weight(N, K, g):
    w = torch.randn(N, K, generator=g) * 0.05
    nb, kb = _cdiv(N, 128), _cdiv(K, 128)
    wp = torch.zeros(nb * 128, kb * 128)
    wp[:N, :K] = w
    blocks = wp.view(nb, 128, kb, 128)
    s = blocks.abs().amax(dim=(1, 3)).clamp(min=1e-8) / 448.0
    q = (blocks / s[:, None, :, None]).reshape(nb * 128, kb * 128)[:N, :K].to(F8)
    return q.contiguous(), s.float().contiguous()


def _operands(kind, M, N, K, seed, dtype=BF):
    """Host operands of one call plus the fp64 values the reference multiplies (`a` [M, K], `w` [N, K]; fp8: the scales
    a_s [M, K/128] and b_s [N/128, K/128]).  Activations of neighbouring tokens differ in scale by a factor of two."""
    g = torch.Generator().manual_seed(seed)
    tok = 2.0 ** (torch.arange(M) % 4 - 1).float()[:, None]
    op = dict(kind=kind, M=M, N=N, K=K, dtype=dtype)
    if kind == "16":
        op["x"] = (torch.randn(M, K, generator=g) * tok).to(dtype)
        op["w"] = (torch.randn(N, K, generator=g) * 0.05).to(dtype)
        op["bias"] = (torch.randn(N, generator=g) * 0.05 * math.sqrt(K)).to(dtype)
        op["a64"], op["w64"] = op["x"].double(), op["w"].double()
    elif kind == "fp8":
        op["w"], op["b_s"] = _fp8_weight(N, K, g)
        op["x"], op["a_s"] = _quant_fp8_act(torch.randn(M, K, generator=g) * tok)
        op["a64"], op["w64"] = op["x"].double(), op["w"].double()
    elif kind == "soft":
        op["w"], op["b_s"] = _fp8_weight(N, K, g)
        op["x"] = (torch.randn(M, K, generator=g) * tok).to(dtype)
        op["a64"] = op["x"].double()
        op["w64"] = O.weight_dequant_soft_fp8(op["w"], op["b_s"]).double()     # the weight rounded to bf16 first
    else:
        op["x"] = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8)
        op["w"] = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8)
        op["a_s"] = (torch.rand(M, generator=g) + 0.5) / (73.0 * K ** 0.25)
        op["b_s"] = (torch.rand(N, generator=g) + 0.5) / (73.0 * K ** 0.25)
        op["bias"] = torch.randn(N, generator=g).to(F16)
    return op


def _dot(op, k_lo, k_hi, a_s=None):
    """fp64 sum over k in [k_lo, k_hi) of the scaled products t_k, and sum of t_k^2: [M, N] each (fp8: per 128-K
    block, (a_blk . b_blk^T) * a_s * b_s)."""
    a, w = op["a64"], op["w64"]
    if op["kind"] != "fp8":
        x, y = a[:, k_lo:k_hi], w[:, k_lo:k_hi]
        return x @ y.T, (x * x) @ (y * y).T
    a_s = (op["a_s"] if a_s is None else a_s).to(a)
    b_s = op["b_s"].to(a).repeat_interleave(128, dim=0)[: op["N"]]
    ref = torch.zeros(a.shape[0], w.shape[0], dtype=a.dtype, device=a.device)
    ss = torch.zeros_like(ref)
    for kb in range(k_lo // 128, _cdiv(k_hi, 128)):
        lo, hi = max(k_lo, kb * 128), min(k_hi, kb * 128 + 128)
        x, y = a[:, lo:hi], w[:, lo:hi]
        sc = a_s[:, kb:kb + 1] * b_s[None, :, kb]
        ref += (x @ y.T) * sc
        ss += ((x * x) @ (y * y).T) * sc * sc
    return ref, ss


def _reference(op, bias=True):
    ref, ss = _dot(op, 0, op["K"])
    if bias and "bias" in op and op["kind"] == "16":
        ref = ref + op["bias"].to(ref)
    return ref, ss.sqrt()


def _ratio(y, ref, rss, u_out, tau):
    """max over elements of |y - ref| / (u_out |ref| + tau rss); inf when y is not finite."""
    y = y.to(ref.device)
    if not bool(torch.isfinite(y).all()):
        return math.inf
    err = (y.double() - ref).abs()
    bound = u_out * ref.abs() + tau * rss
    r = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max())


def _to_device(op):
    d = dict(op)
    d["a64"], d["w64"] = op["a64"].to(DEV), op["w64"].to(DEV)
    return d


# ------------------------------------------------------------------------- injected-error self-test of the bound
def _injections(op, sc, BN):
    """(name, the output of a kernel with that error: the fp64 reference with the error, rounded to the output dtype)."""
    M, N, K, kind = op["M"], op["N"], op["K"], op["kind"]
    ref, _ = _reference(op)
    out = op["dtype"]
    rows = slice(0, min(N, 128))                  # the first tile
    cols = slice(0, min(M, BN))
    st = STAGE_K[kind]
    yield "a 64-K stage dropped", (ref - _tile_only(_dot(op, (sc["S"] // 2) * st, (sc["S"] // 2) * st + 64)[0],
                                                   cols, rows)).to(out)
    if kind == "fp8" and M >= 2:
        a_s = op["a_s"].clone()
        a_s[1] = op["a_s"][0]                     # token 1 scaled with token 0's a_s
        wrong = ref.clone()
        wrong[1, rows] = _dot(op, 0, K, a_s)[0][1, rows]
        yield "a neighbouring token's a_s", wrong.to(out)
    if kind == "16":
        yield "bias dropped", (ref - op["bias"].to(ref)).to(out)
    if sc["split"]:
        t, v = max(sc["split"].items(), key=lambda tv: len(tv[1]))
        _, _, s_lo, s_hi = v[-1]                  # the last contributor's share
        n0, m0 = (t % sc["n_tiles"]) * 128, (t // sc["n_tiles"]) * BN
        part = _dot(op, s_lo * st, min(s_hi * st, K))[0]
        yield "a split contributor missing", (ref - _tile_only(part, slice(m0, min(m0 + BN, M)),
                                                              slice(n0, min(n0 + 128, N)))).to(out)


def _tile_only(part, cols, rows):
    z = torch.zeros_like(part)
    z[cols, rows] = part[cols, rows]
    return z


@pytest.mark.parametrize("kind", ["16", "fp8", "soft"])
def test_bound_rejects_injected_errors(kind):
    """On the case table's shapes the bound admits the correctly rounded reference and rejects each injected error."""
    names = set()
    for k, M, N, K, _ in _case_table(132):
        if k != kind:
            continue
        sc = _schedule(kind, M, N, K, 132)
        op = _operands(kind, M, N, K, seed=M * 7919 + N + K)
        ref, rss = _reference(op)
        u, tau = U_OUT[op["dtype"]], _tau(kind, 2)
        assert _ratio(ref.to(op["dtype"]), ref, rss, u, tau) <= 1.0
        for name, y in _injections(op, sc, sc["BN"]):
            names.add(name)
            assert _ratio(y, ref, rss, u, tau) > 1.0, (name, M, N, K)
    want = {"a 64-K stage dropped", "a split contributor missing"}
    want |= {"bias dropped"} if kind == "16" else {"a neighbouring token's a_s"} if kind == "fp8" else set()
    assert names == want


# ---------------------------------------------------------------------------------------------------- GPU calls
PAD = 256          # bytes of pad before and after every operand view (keeps the views 16-byte aligned)
NAN_BYTE = 0xFF    # NaN in bf16, fp16, fp8 e4m3 and fp32 (and -1 in int8)
SENTINEL = 0xA5


def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Padded:
    """A contiguous view in the middle of a larger byte buffer; the pads hold `pad` bytes."""

    def __init__(self, t, pad=NAN_BYTE, fill=None):
        nbytes = t.numel() * t.element_size()
        self.buf = torch.full((2 * PAD + nbytes,), pad, dtype=torch.uint8, device=DEV)
        self.pad, self.nbytes = pad, nbytes
        self.view = self.buf[PAD:PAD + nbytes].view(t.dtype).view(t.shape)
        if fill is None:
            self.view.copy_(t.to(DEV))
        else:
            self.buf[PAD:PAD + nbytes].fill_(fill)

    def pads_intact(self):
        return bool((self.buf[:PAD] == self.pad).all()) and bool((self.buf[PAD + self.nbytes:] == self.pad).all())


def _out_dtype(kind, dtype):
    return F16 if kind == "i8" else dtype


class Call:
    """One GEMM through its C entry, with x, W and y as views inside NaN / sentinel padded buffers."""

    def __init__(self, op, bias=None, residual=None):
        self.op = op
        self.kind, self.M, self.N, self.K = op["kind"], op["M"], op["N"], op["K"]
        self.x, self.w = Padded(op["x"]), Padded(op["w"])
        self.a_s = op["a_s"].to(DEV) if "a_s" in op else None
        self.b_s = op["b_s"].to(DEV) if "b_s" in op else None
        self.bias = None if bias is None else bias.to(DEV)
        self.residual = None if residual is None else residual.to(DEV)
        self.out_dtype = _out_dtype(self.kind, op["dtype"])
        self.y = Padded(torch.empty(self.M, self.N, dtype=self.out_dtype), pad=SENTINEL, fill=NAN_BYTE)

    def __call__(self, impl, ws=None, ws_bytes=None):
        from chitu_b200._lib import current_stream, dtype_code, ptr
        lib, st = _lib(), current_stream()
        nb = 0 if ws is None else (ws.numel() if ws_bytes is None else ws_bytes)
        M, N, K, x, w, y = self.M, self.N, self.K, ptr(self.x.view), ptr(self.w.view), ptr(self.y.view)
        if self.kind == "16":
            return lib.chitu_b200_linear_bf16(x, w, ptr(self.bias), ptr(self.residual), y, M, N, K,
                                              dtype_code(self.out_dtype), ptr(ws), nb, impl, st)
        if self.kind == "fp8":
            return lib.chitu_b200_fp8_gemm(x, ptr(self.a_s), w, ptr(self.b_s), y, M, N, K, ptr(self.residual),
                                           ptr(ws), nb, impl, st)
        if self.kind == "soft":
            return lib.chitu_b200_soft_fp8_gemm(x, w, ptr(self.b_s), y, M, N, K, dtype_code(self.out_dtype),
                                                ptr(ws), nb, impl, st)
        return lib.chitu_b200_w8a8_gemm(y, x, w, ptr(self.a_s), ptr(self.b_s), ptr(self.bias), M, N, K, ptr(ws), nb,
                                        impl, st)

    def run(self, impl, ws=None):
        from chitu_b200._lib import check
        check(self(impl, ws), f"{self.kind} gemm M={self.M} N={self.N} K={self.K} impl={impl}")
        return self.y.view


def _workspace(M, N):
    """Tickets zeroed, partial slots filled with 0xFF."""
    ws = torch.full((_lib().chitu_b200_linear_workspace_bytes(M, N),), 0xFF, dtype=torch.uint8, device=DEV)
    ws[:TICKET_BYTES].zero_()
    return ws


def _written_slots(ws, BN):
    slots = ws[TICKET_BYTES:].view(torch.int32).view(-1, 2, BN * 128)
    untouched = (slots == -1).all(dim=-1)
    return {(int(c), int(s)) for c, s in torch.nonzero(~untouched).tolist()}


def _check_call(call, impl, ws, sc, ref, rss, tau, exact=None):
    """Run once and check: finite, pads unchanged, within the bound (or bit-equal to `exact`), tickets back at zero
    and the written partial slots those of the model.  Returns the ratio to the bound."""
    y = call.run(impl, ws)
    torch.cuda.synchronize()
    what = (call.kind, call.M, call.N, call.K, impl, str(call.out_dtype))
    assert call.x.pads_intact() and call.w.pads_intact(), what
    assert call.y.pads_intact(), ("output pad overwritten",) + what
    assert bool(torch.isfinite(y).all()), ("non-finite output",) + what
    if ws is not None:
        assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0, ("tickets left non-zero",) + what
        assert _written_slots(ws, sc["BN"]) == sc["slots"], ("partial slots differ from the schedule model",) + what
    if exact is not None:
        assert torch.equal(y.cpu().view(torch.int16), exact.view(torch.int16)), ("not bit-exact",) + what
        return 0.0
    r = _ratio(y, ref, rss, U_OUT[call.out_dtype], tau)
    assert r <= 1.0, ("outside the bound", r) + what
    return r


def _ratio_report(kind, impl, dtype, worst, n):
    print(f"[gemm bound] kind={kind} impl={impl} dtype={str(dtype).split('.')[-1]} cases={n} max|y-ref|/bound={worst:.3f}")


# ------------------------------------------------------------------------------------- parity over the case table
@pytest.mark.gpu
@pytest.mark.parametrize("impl", [2, 1])
@pytest.mark.parametrize("kind", ["16", "fp8", "soft"])
def test_case_table_parity(kind, impl):
    """Every case of the table on the device's SM count: inside the bound, pads untouched, and (wgmma) the workspace
    shows the model's split.  16-bit runs bf16 and fp16 with a bias."""
    sms = _sms()
    cases = [c for c in _case_table(sms) if c[0] == kind]
    for dtype in ((BF, F16) if kind == "16" else (BF,)):
        worst = 0.0
        for _, M, N, K, _ in cases:
            sc = _schedule(kind, M, N, K, sms)
            op = _operands(kind, M, N, K, seed=M * 7919 + N + K, dtype=dtype)
            ref, rss = _reference(_to_device(op))
            call = Call(op, bias=op.get("bias"))
            ws = _workspace(M, N) if impl == 2 else None
            worst = max(worst, _check_call(call, impl, ws, sc, ref, rss, _tau(kind, impl)))
        _ratio_report(kind, impl, dtype, worst, len(cases))


def _w8a8_exact(op, bias):
    return O.w8a8_mm(op["x"], op["w"], op["a_s"], op["b_s"], bias)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [2, 1])
def test_int8_bit_exact_over_case_table(impl):
    """int8 at every BN and regime == w8a8gemm.mm's semantics (exact int32 dot, fp32 scales, fp16 out, fp16 bias add),
    bit for bit, with and without bias."""
    sms = _sms()
    cases = [c for c in _case_table(sms) if c[0] == "i8"]
    for _, M, N, K, _ in cases:
        sc = _schedule("i8", M, N, K, sms)
        op = _operands("i8", M, N, K, seed=M * 7919 + N + K)
        for bias in (None, op["bias"]):
            ws = _workspace(M, N) if impl == 2 else None
            _check_call(Call(op, bias=bias), impl, ws, sc, None, None, None, exact=_w8a8_exact(op, bias))
    print(f"[gemm bound] kind=i8 impl={impl} cases={len(cases)} bit-exact")


# ---------------------------------------------------------------------------------------------------------- tails
N_TAILS = (8, 100, 1000, 192, 77)
K_TAILS_16 = (8, 72, 1000, 4104)


def _tail_shapes(kind):
    K = {"16": 1024, "fp8": 512, "soft": 512, "i8": 528}[kind]
    shapes = [(M, N, K) for N in N_TAILS for M in (1, 33, 129)]
    if kind == "16":
        shapes += [(M, 1000, K) for K in K_TAILS_16 for M in (16, 65)]
    return shapes


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [2, 1])
@pytest.mark.parametrize("kind", KINDS)
def test_tails(kind, impl):
    """N that leaves a partial weight tile (8, 100, 1000, N % 128 = 64, odd) and 16-bit K whose last TMA box is partly
    out of bounds (8, 72, 1000, 4104); int8 K = 528 likewise."""
    sms = _sms()
    worst = 0.0
    for M, N, K in _tail_shapes(kind):
        sc = _schedule(kind, M, N, K, sms)
        for dtype in ((BF, F16) if kind == "16" else (BF,)):
            op = _operands(kind, M, N, K, seed=3 * M + 5 * N + K, dtype=dtype)
            ws = _workspace(M, N) if impl == 2 else None
            if kind == "i8":
                _check_call(Call(op, bias=op["bias"]), impl, ws, sc, None, None, None, exact=_w8a8_exact(op, op["bias"]))
                continue
            ref, rss = _reference(_to_device(op))
            worst = max(worst, _check_call(Call(op, bias=op.get("bias")), impl, ws, sc, ref, rss, _tau(kind, impl)))
    print(f"[gemm bound] tails kind={kind} impl={impl} max|y-ref|/bound={worst:.3f}")


# ------------------------------------------------------------------------------------------------------ epilogues
def _split_case(kind, sms, regime="slot1", bn=None):
    for k, M, N, K, cells in _case_table(sms):
        if k == kind and any(r == regime and (bn is None or b == bn) for b, r in cells):
            return M, N, K
    raise AssertionError((kind, regime, bn))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [2, 1])
@pytest.mark.parametrize("kind,dtype", [("16", BF), ("16", F16), ("fp8", BF)])
def test_residual_is_one_more_rounding(kind, dtype, impl):
    """y(residual) == round(float(y) + float(residual)) bit for bit, on a whole-tile shape and on a split shape (where
    the last arriving contributor adds the residual)."""
    sms = _sms()
    for M, N, K in (_split_case(kind, sms, "whole", 64), _split_case(kind, sms, "slot1", 128),
                    _split_case(kind, sms, "count_gt_cb", 16)):
        op = _operands(kind, M, N, K, seed=M + N + K, dtype=dtype)
        res = torch.randn(M, N, generator=torch.Generator().manual_seed(N)).to(dtype)
        ws = _workspace(M, N) if impl == 2 else None
        plain = Call(op, bias=op.get("bias")).run(impl, ws).cpu()
        got = Call(op, bias=op.get("bias"), residual=res).run(impl, ws).cpu()
        want = (plain.float() + res.float()).to(dtype)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (kind, dtype, M, N, K, impl)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(17, 384, 1792), (32, 1000, 2048), (129, 640, 1024), (100, 384, 4096)])
def test_silu_pairs_epilogue_at_bn_32_and_128(M, N, K):
    """linear_bf16_silu_pairs at BN 32 / 128 with N % 256 != 0 == SiluAndMul of the plain linear of the same
    interleaved weight (same schedule, so the same fp32 sums): exact up to the fp32 exp (<= 1 bf16 ulp, rarely)."""
    from chitu_b200._lib import check, current_stream, ptr
    assert _pick_bn(M) in (32, 128) and N % 256 != 0
    lib = _lib()
    op = _operands("16", M, N, K, seed=M * N + K)
    plain = Call(op)
    ws = _workspace(M, N)
    sc = _schedule("16", M, N, K, _sms())
    ref, rss = _reference(_to_device(op), bias=False)
    _check_call(plain, 2, ws, sc, ref, rss, TAU_FP32)
    ws[TICKET_BYTES:].fill_(0xFF)
    y = Padded(torch.empty(M, N // 2, dtype=BF), pad=SENTINEL, fill=NAN_BYTE)
    check(lib.chitu_b200_linear_bf16_silu_pairs(ptr(plain.x.view), ptr(plain.w.view), ptr(y.view), M, N, K, ptr(ws),
                                                ws.numel(), current_stream()), "pairs")
    torch.cuda.synchronize()
    assert y.pads_intact() and bool(torch.isfinite(y.view).all())
    assert _written_slots(ws, sc["BN"]) == sc["slots"]
    g, u = plain.y.view[:, 0::2].float(), plain.y.view[:, 1::2].float()
    want = ((g / (1.0 + torch.exp(-g))).to(BF).float() * u).to(BF)
    got = y.view
    diff = (got.view(torch.int16).int() - want.view(torch.int16).int()).abs()
    assert int(diff.max()) <= 1 and float((diff > 0).float().mean()) < 0.01


# -------------------------------------------------------------------------------------- determinism and reuse
@pytest.mark.gpu
def test_split_shapes_are_deterministic_and_share_a_workspace():
    """A split shape called twice gives the same bits; three split shapes of different BN alternating on one workspace
    each reproduce their first result."""
    sms = _sms()
    shapes = [_split_case("16", sms, "slot1", bn) for bn in (16, 64, 128)]
    calls = [Call(_operands("16", M, N, K, seed=M + N)) for M, N, K in shapes]
    nbytes = max(_lib().chitu_b200_linear_workspace_bytes(M, N) for M, N, _ in shapes)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    first = [c.run(2, ws).clone() for c in calls]
    assert torch.equal(calls[0].run(2, ws).view(torch.int16), first[0].view(torch.int16))
    for _ in range(2):
        for c, f in zip(calls, first):
            assert torch.equal(c.run(2, ws).view(torch.int16), f.view(torch.int16)), (c.M, c.N, c.K)
    assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_split_shape_in_a_cuda_graph(kind):
    """One split shape per kind captured once and replayed with new inputs copied in == eager calls, bit for bit."""
    sms = _sms()
    M, N, K = _split_case(kind, sms, "slot1")
    ops = [_operands(kind, M, N, K, seed=100 + i) for i in range(4)]
    call = Call(ops[0], bias=ops[0].get("bias"))
    ws = torch.zeros(_lib().chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)

    def load(op):
        call.x.view.copy_(op["x"].to(DEV))
        call.w.view.copy_(op["w"].to(DEV))
        for name in ("a_s", "b_s", "bias"):
            if getattr(call, name) is not None:
                getattr(call, name).copy_(op[name].to(DEV))

    eager = []
    for op in ops[1:]:
        load(op)
        eager.append(call.run(2, ws).clone())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call.run(2, ws)                           # warm-up off the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call.run(2, ws)
    for op, want in zip(ops[1:], eager):
        load(op)
        call.y.view.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(call.y.view.view(torch.int16), want.view(torch.int16)), kind
    assert int(ws[:TICKET_BYTES].view(torch.int32).count_nonzero()) == 0


# ------------------------------------------------------------------------------------- fallbacks and refusals
def _last_error():
    return _lib().chitu_b200_last_error().decode(errors="replace")


@pytest.mark.gpu
def test_shapes_the_wgmma_path_cannot_take_run_simt_under_auto():
    """fp8 with K % 128 != 0 and soft-fp8 with fp16 activations: impl=2 refuses with a message, impl=0 runs the SIMT
    kernel and lands inside the fp32-accumulation bound."""
    sms = _sms()
    for kind, M, N, K, dtype in (("fp8", 16, 300, 400, BF), ("fp8", 40, 256, 1040, BF), ("soft", 9, 200, 512, F16)):
        op = _operands(kind, M, N, K, seed=M + K, dtype=dtype)
        ws = _workspace(M, N)
        call = Call(op)
        assert call(2, ws) != 0 and "wgmma path unavailable" in _last_error()
        y = call.run(0, ws)
        torch.cuda.synchronize()
        assert call.x.pads_intact() and call.w.pads_intact() and call.y.pads_intact()
        ref, rss = _reference(_to_device(op))
        assert _ratio(y, ref, rss, U_OUT[call.out_dtype], TAU_FP32) <= 1.0, (kind, M, N, K)
        assert int(ws[:TICKET_BYTES].count_nonzero()) == 0 and bool((ws[TICKET_BYTES:] == 0xFF).all())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_workspace_one_byte_short(kind):
    """A workspace one byte short: impl=0 takes the SIMT kernel (and leaves the workspace alone), impl=2 returns a
    non-zero status with a message."""
    M, N, K = 17, 384, 1024
    op = _operands(kind, M, N, K, seed=7)
    call = Call(op, bias=op.get("bias"))
    need = _lib().chitu_b200_linear_workspace_bytes(M, N)
    ws = _workspace(M, N)
    assert call(2, ws, need - 1) != 0 and "wgmma path unavailable" in _last_error()
    from chitu_b200._lib import check
    check(call(0, ws, need - 1), "impl 0")
    torch.cuda.synchronize()
    assert bool((ws[TICKET_BYTES:] == 0xFF).all())
    if kind == "i8":
        assert torch.equal(call.y.view.cpu().view(torch.int16), _w8a8_exact(op, op["bias"]).view(torch.int16))
    else:
        ref, rss = _reference(_to_device(op))
        assert _ratio(call.y.view, ref, rss, U_OUT[call.out_dtype], TAU_FP32) <= 1.0


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """16-bit K % 8 != 0 returns a status on every impl without a launch; M = 0 returns 0 and writes nothing."""
    from chitu_b200._lib import launch_count
    op = _operands("16", 4, 128, 16, seed=1)
    lib = _lib()
    ws = _workspace(4, 128)
    call = Call(op)
    call.K = 12                                   # rows of 24 bytes: neither TMA nor the 16-byte SIMT loads
    before = launch_count()
    for impl in (0, 1, 2):
        assert call(impl, ws) != 0 and _last_error()
    assert launch_count() == before
    for kind in KINDS:
        op = _operands(kind, 4, 128, 256, seed=2)
        c = Call(op, bias=op.get("bias"))
        c.M = 0
        for impl in (0, 1, 2):
            assert c(impl, ws) == 0
    from chitu_b200._lib import current_stream, ptr
    y = torch.full((4, 64), float("nan"), dtype=BF, device=DEV)
    assert lib.chitu_b200_linear_bf16_silu_pairs(ptr(call.x.view), ptr(call.w.view), ptr(y), 0, 128, 16, ptr(ws),
                                                 ws.numel(), current_stream()) == 0
    torch.cuda.synchronize()
    assert launch_count() == before
    assert int(ws[:TICKET_BYTES].count_nonzero()) == 0 and bool((ws[TICKET_BYTES:] == 0xFF).all())


# -------------------------------------------------------------------------- weight written by the preceding call
@pytest.mark.gpu
def test_linear_reads_weight_written_by_the_preceding_dequant():
    """weight_dequant_fp8 into a NaN-filled buffer, then straight away linear_bf16 (wgmma) on that buffer.  The GEMM
    streams its first weight stages before griddepcontrol.wait, so the dequant must not let it start early."""
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib()
    M, N, K = 8, 4096, 4096                       # the dequant runs many waves of CTAs
    g = torch.Generator().manual_seed(10)
    wq, ws_scale = _fp8_weight(N, K, g)
    x = torch.randn(M, K, generator=g).to(BF)
    w = torch.full((N, K), float("nan"), dtype=BF, device=DEV)
    xd, wqd, sd = x.to(DEV), wq.to(DEV), ws_scale.to(DEV)
    y = torch.empty(M, N, dtype=BF, device=DEV)
    ws = torch.zeros(lib.chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    st = current_stream()
    check(lib.chitu_b200_weight_dequant_fp8(ptr(wqd), ptr(sd), ptr(w), 1, N, K, 128, 0, st), "dequant")
    check(lib.chitu_b200_linear_bf16(ptr(xd), ptr(w), None, None, ptr(y), M, N, K, 0, ptr(ws), ws.numel(), 2, st),
          "linear")
    torch.cuda.synchronize()
    w_ref = O.weight_dequant(wq, ws_scale)
    assert torch.equal(w.cpu().view(torch.int16), w_ref.view(torch.int16))
    a64, w64 = x.double().to(DEV), w_ref.double().to(DEV)
    ref, rss = a64 @ w64.T, ((a64 * a64) @ (w64 * w64).T).sqrt()
    assert _ratio(y, ref, rss, U_OUT[BF], TAU_FP32) <= 1.0
