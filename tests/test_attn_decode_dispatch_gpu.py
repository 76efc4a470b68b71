"""Paged decode attention against an fp64 reference, on shapes chosen by a restatement of the host code that splits the
keys: GQA through `chitu_b200_gqa_paged_decode[_rope]` (`gqa_decode_mmaT_kernel`, or `gqa_decode_kernel` for D = 64
and pages that are not a power of two), the same kernels through `chitu_b200_gqa_contiguous_attn` and
`chitu_b200_gqa_paged_attn_fp8kv` (seqlen_q == 1), and absorbed MLA through `chitu_b200_mla_decode` (direct, merged,
or `out = NULL` followed by `chitu_b200_mla_absorb_o_merge_quant`), with and without a split plan.

The host model restates `pick_splits_waves`, `pick_splits`, `splits_that_fit`, `mla_num_splits` (csrc/splitkv.cuh),
the keys-per-split search of `attn_plan_kernel` (csrc/core.cu) and the plan condition of `mla_decode_tc_kernel`
(csrc/mla_tc.cu), plus the key range [s * chunk, min((s + 1) * chunk, L)) each kernel gives split s.  All of them
assume 132 SMs, whatever the device.  The case table holds one case per reachable (entry, kernel, dtype, G, split
regime) and (H, split regime, plan, output) cell; the GPU tests run it with NaN-poisoned caches, a NaN trap page behind
every unused block-table column, sentinel pads around the output and a 0xFF workspace, and read the per-split partials
back to check the split count, every split's key range and its LSE.

The bound: every element satisfies
    |y - ref| <= u_out |ref| + TAU u_p sqrt(sum_j w_j^2 v_j^2) + U_ACC sum_j w_j |v_j| + TAU_S sum_j w_j a_j (|v_j| + |ref|)
with w = softmax(s) in fp64 and a_j = scale sum_i |q_i k_ji| + its maximum over the keys (the size of the fp32 score
and exponent arguments).  u_out is the output rounding (bf16 2^-8, fp16 2^-11, 0 for the fp32 partials), u_p the
rounding of P before the P.V MMA (bf16 2^-8, fp16 2^-11; 0 on the SIMT kernel, which keeps P in fp32).
`test_bound_rejects_injected_errors` shows that the bound sees a key dropped or counted twice at a split boundary, the
appended key dropped, a key read past the end, a tile read through the wrong block-table entry, two heads swapped and a
split LSE taken in the natural-log domain, on data where one "needle" key carries about 40 % of the softmax mass."""
import functools
import math

import pytest
import torch

BF, F16, F8 = torch.bfloat16, torch.float16, torch.float8_e4m3fn
DEV = "cuda:0"

# ---------------------------------------------------------------------------------------------- host model
SMS = 132                  # the split heuristics assume an H100's 132 SMs, whatever the device
GQA_CTAS = 1               # kGqaCtas
GQA_TILE = 16              # kGqaTile: keys per tile of the tensor-core GQA kernel
MLA_TILE = 64              # keys per tile (= page) of the MLA kernel
MAX_SPLITS = 128           # kMaxSplits
MLA_C, MLA_R = 512, 64
PLAN_BYTES, PLAN_MAGIC = 256, 0x504C414E
W_MAGIC, W_KPS, W_MAX, W_TOTAL, W_BATCH, W_PAGE, W_HEADS = range(7)


def _cdiv(a, b):
    return -(-a // b)


def split_kv_bytes(rows, dv, splits):
    return rows * splits * (dv + 1) * 4 + PLAN_BYTES


def splits_that_fit(splits, rows, dv, ws_bytes):
    while splits > 1 and split_kv_bytes(rows, dv, splits) > ws_bytes:
        splits -= 1
    return splits


def pick_splits_waves(ctas, max_len, slots):
    by_len = min(_cdiv(max_len, 128), 64)
    best, best_cost = 1, 1e30
    for s in range(1, by_len + 1):
        waves = _cdiv(ctas * s, slots)
        cost = waves * (max_len / s + 192.0) + (64.0 if s > 1 else 0.0)
        if cost < best_cost - 1e-9:
            best, best_cost = s, cost
    return best


def pick_splits(ctas, max_len, min_keys, max_splits):
    want = _cdiv(SMS * 4, ctas)
    s = min(want, _cdiv(max_len, min_keys), max_splits)
    return max(s, 1)


def mla_num_splits(B, H, max_len, ws_bytes):
    want = SMS // (B * _cdiv(H, 16))
    s = max(min(want, _cdiv(max_len, 64) // 2, MAX_SPLITS), 1)
    return splits_that_fit(s, B * H, MLA_C, ws_bytes)


def gqa_picked(kernel, B, Hkv, max_len):
    """The split count the heuristic picks before the workspace is consulted."""
    if kernel == "tc":
        return pick_splits_waves(B * Hkv, max_len, SMS * GQA_CTAS)
    return pick_splits(B * Hkv, max_len, 256, 64)


def gqa_splits(kernel, B, Hq, Hkv, D, max_len, ws_bytes):
    """ws_bytes None: no workspace."""
    s = gqa_picked(kernel, B, Hkv, max_len)
    return splits_that_fit(s, B * Hq, D, ws_bytes) if ws_bytes is not None else 1


def attn_plan(lens_incl, heads, page, hint, ws_bytes):
    """attn_plan_kernel's plan words for seqlens_incl = lens_incl (chitu_b200_attn_plan)."""
    B = len(lens_incl)
    slots = max(SMS // _cdiv(heads, 16), 1)
    max_splits = mla_num_splits(B, heads, hint, ws_bytes)
    pages = [_cdiv(L, page) for L in lens_incl]
    total_pages, max_pages = sum(pages), max(pages)
    pps = max(2, _cdiv(total_pages, slots), _cdiv(max_pages, max_splits), 1)
    for _ in range(64):
        splits = [_cdiv(p, pps) for p in pages]
        total, mx = sum(splits), max(splits)
        if total <= slots or pps >= max_pages:
            break
        pps += 1
    return {W_MAGIC: PLAN_MAGIC, W_KPS: pps * page, W_MAX: mx, W_TOTAL: total, W_BATCH: B, W_PAGE: page,
            W_HEADS: heads}


def plan_honoured(plan, B, H, L, splits):
    """mla_decode_tc_kernel's condition for request length L (mla_tc.cu): the plan's keys per split or None."""
    per = _cdiv(_cdiv(L, splits), MLA_TILE) * MLA_TILE
    if (plan is None or plan.get(W_MAGIC) != PLAN_MAGIC or plan[W_PAGE] != MLA_TILE or plan[W_BATCH] != B
            or plan[W_HEADS] != H or plan[W_KPS] < per or _cdiv(L, plan[W_KPS]) > splits):
        return None
    return plan[W_KPS]


def chunk_of(kernel, L, splits, kps=None):
    """Keys per split of request length L: split s covers [s * chunk, min((s + 1) * chunk, L))."""
    c = _cdiv(L, splits)
    if kernel == "tc":
        return _cdiv(c, GQA_TILE) * GQA_TILE
    if kernel == "mla":
        return kps if kps is not None else _cdiv(c, MLA_TILE) * MLA_TILE
    return c


def split_ranges(L, splits, chunk):
    return [(min(s * chunk, L), min((s + 1) * chunk, L)) for s in range(splits)]


# ---------------------------------------------------------------------------------------------- case table
GS = (1, 2, 4, 8)
REGIMES = ("1", "2-7", "8-15", "16-64", "lowered", "none")
DTYPES = (BF, F16)
GQA_KERNELS = {"paged": ("tc", "simt"), "contig": ("tc", "simt"), "fp8": ("tc",)}
TC_PAGES = (1, 8, 16, 64, 256, 1024)
FP8_PAGES = (64, 256, 1024)
SIMT_GEOM = ((128, 48), (128, 100), (64, 64), (64, 16))     # (D, page) of the paged SIMT cases: D = 64 or odd pages
HINTS = ("exact", "below", "above", "zero")


def _regime(splits, picked, ws):
    if ws == "none":
        return "none"
    if ws == "lowered":
        return "lowered"
    return "1" if splits == 1 else "2-7" if splits < 8 else "8-15" if splits < 16 else "16-64"


def _lens(B, L_max, new, seed):
    """Cached lengths of a ragged batch: the longest request, a page or tile edge, a short one and (without new k / v)
    an empty one."""
    extra = [L_max // 3, 1, L_max - 2, 63, L_max // 2 + 5, 255]
    lens = [L_max - 1] + [max(min(extra[(i + seed) % len(extra)], L_max - 1), 0) for i in range(B - 1)]
    if not new and B > 1:
        lens[-1] = 0
    return lens


def _max_len(hint, L_max, bt_cols_len):
    return {"exact": L_max, "below": max(L_max // 3, 1), "above": 4 * L_max, "zero": bt_cols_len}[hint]


def _geometry(entry, kernel, i):
    if entry == "fp8":
        return 128, FP8_PAGES[i % len(FP8_PAGES)]
    if entry == "contig":
        return (128 if kernel == "tc" else 64), None
    if kernel == "tc":
        return 128, TC_PAGES[i % len(TC_PAGES)]
    return SIMT_GEOM[i % len(SIMT_GEOM)]


def _gqa_hint_value(c):
    """The max_seqlen_hint argument and the max_len the entry derives from it."""
    if c["hint"] == "zero":
        span = c["rows"] if c["entry"] == "contig" else c["bt_stride"] * c["page"]
        return 0, span
    v = _max_len(c["hint"], c["L_max"], None)
    return v, v


@functools.lru_cache(maxsize=None)
def gqa_case_table():
    """One case per (entry, kernel, dtype, G, regime): the cheapest batch / length / hint that lands in the cell."""
    cases = []
    i = 0
    for entry, kernels in GQA_KERNELS.items():
        for kernel in kernels:
            for dtype in DTYPES:
                for G in GS:
                    for regime in REGIMES:
                        i += 1
                        D, page = _geometry(entry, kernel, i)
                        best = None
                        for B in (2, 3, 5, 8):
                            for Hkv in (1, 2, 4):
                                for L_max in (40, 130, 300, 1000, 2500, 5000, 9000):
                                    for hint in HINTS[(i % 4):] + HINTS[:(i % 4)]:
                                        c = _gqa_case(entry, kernel, dtype, G, B, Hkv, D, page, L_max, hint, regime, i)
                                        if c is None:
                                            continue
                                        cost = B * Hkv * G * L_max * (c["splits"] + 4)
                                        if best is None or cost < best[0]:
                                            best = (cost, c)
                        if best is not None:
                            cases.append(best[1])
    return tuple(cases)


def _gqa_case(entry, kernel, dtype, G, B, Hkv, D, page, L_max, hint, regime, i):
    new = i % 3 != 0                       # with and without k / v
    lens = _lens(B, L_max, new, i)
    c = dict(entry=entry, kernel=kernel, dtype=dtype, G=G, B=B, Hkv=Hkv, Hq=G * Hkv, D=D, page=page, L_max=L_max,
             hint=hint, new=new, lens=lens, seed=i, rope=(entry == "paged" and kernel == "tc" and new and i % 2 == 0))
    if entry == "contig":
        c["rows"] = L_max + 3
    else:
        c["bt_stride"] = _cdiv(L_max + 1, page) + 1
    c["hint_arg"], max_len = _gqa_hint_value(c)
    picked = gqa_picked(kernel, B, Hkv, max_len)
    full = split_kv_bytes(B * G * Hkv, D, 64)
    if regime == "none":
        if picked < 2:
            return None
        ws = None
    elif regime == "lowered":
        if picked < 2:
            return None
        ws = split_kv_bytes(B * G * Hkv, D, picked // 2) + (0 if picked >= 4 else -1)
    else:
        ws = full
    splits = gqa_splits(kernel, B, G * Hkv, Hkv, D, max_len, ws)
    if regime not in ("none", "lowered") and _regime(splits, picked, "full") != regime:
        return None
    if regime == "lowered" and splits >= picked:
        return None
    c.update(ws=ws, picked=picked, splits=splits, regime=regime, max_len=max_len)
    return c


MLA_HS = (8, 16, 24, 32, 128)
MLA_REGIMES = ("1", "rem", "128")
MLA_PLANS = ("honoured", "refused")
REFUSALS = ("other_batch", "other_heads", "kps_below_per", "no_magic")
# (B, longest length) per (H, regime): one split, a count with a remainder mod 8 for the merge loops, 128 splits
MLA_SHAPES = {
    (8, "1"): (2, 150), (16, "1"): (3, 150), (24, "1"): (2, 100), (32, "1"): (2, 150), (128, "1"): (2, 150),
    (8, "rem"): (2, 900), (16, "rem"): (1, 1700), (24, "rem"): (2, 400), (32, "rem"): (1, 2700), (128, "rem"): (3, 1000),
    (8, "128"): (1, 16400), (16, "128"): (1, 16400),
}


def _mla_regime(splits):
    return "1" if splits == 1 else "128" if splits == MAX_SPLITS else "rem" if splits % 8 else "mult8"


@functools.lru_cache(maxsize=None)
def mla_case_table():
    cases = []
    i = n_refused = 0
    for H in MLA_HS:
        for regime in MLA_REGIMES:
            if (H, regime) not in MLA_SHAPES:
                continue
            B, L_max = MLA_SHAPES[(H, regime)]
            for plan in MLA_PLANS:
                for deferred in (False, True):
                    i += 1
                    new = i % 4 != 1
                    lens = _lens(B, L_max, new, i)
                    ws = split_kv_bytes(B * H, MLA_C, MAX_SPLITS)
                    splits = mla_num_splits(B, H, L_max, ws)
                    Ls = [L + new for L in lens]
                    c = dict(H=H, B=B, L_max=L_max, lens=lens, new=new, ws=ws, splits=splits, regime=regime,
                             plan=plan, deferred=deferred, seed=i, bt_stride=_cdiv(L_max + 1, MLA_TILE) + 1)
                    if plan == "honoured":
                        c["plan_words"] = attn_plan(Ls, H, MLA_TILE, L_max, ws)
                    else:
                        refusal = REFUSALS[n_refused % len(REFUSALS)]
                        n_refused += 1
                        words = attn_plan(Ls, H, MLA_TILE, L_max, ws)
                        if refusal == "other_batch":
                            words[W_BATCH] = B + 1
                        elif refusal == "other_heads":
                            words[W_HEADS] = H + 16
                        elif refusal == "kps_below_per":
                            words[W_KPS] = MLA_TILE // 2           # below every request's own keys per split
                        else:
                            words[W_MAGIC] = 0
                        c["refusal"], c["plan_words"] = refusal, words
                    kps = [plan_honoured(c["plan_words"], B, H, L, splits) for L in Ls]
                    c["kps"] = kps
                    c["honoured"] = any(k is not None for k in kps)
                    cases.append(c)
    return tuple(cases)


def _gqa_cells(table):
    return {(c["entry"], c["kernel"], c["dtype"], c["G"], c["regime"]) for c in table}


def _mla_out(c):
    return "deferred" if c["deferred"] else "direct" if c["splits"] == 1 else "merged"


def _mla_cells(table):
    return {(c["H"], _mla_regime(c["splits"]), "honoured" if c["honoured"] else "refused", _mla_out(c)) for c in table}


def test_case_table_covers_every_cell():
    """Every (entry, kernel, dtype, G, split regime) cell of the GQA decode entries and every (H, split regime, plan,
    output) cell of MLA decode has a case, and each case really is in its cell by the host model."""
    gqa = gqa_case_table()
    want = {(e, k, dt, G, r) for e, ks in GQA_KERNELS.items() for k in ks for dt in DTYPES for G in GS for r in REGIMES}
    assert _gqa_cells(gqa) == want
    for c in gqa:
        assert c["splits"] == gqa_splits(c["kernel"], c["B"], c["Hq"], c["Hkv"], c["D"], c["max_len"], c["ws"])
        assert (c["ws"] is None) == (c["regime"] == "none") and c["splits"] <= 64
        if c["regime"] == "lowered":
            assert 1 <= c["splits"] < c["picked"]
    paged = [c for c in gqa if c["entry"] == "paged"]
    assert {c["page"] for c in paged if c["kernel"] == "tc"} == set(TC_PAGES)
    assert {(c["D"], c["page"]) for c in paged if c["kernel"] == "simt"} == set(SIMT_GEOM)
    assert {c["hint"] for c in gqa} == set(HINTS) and any(c["rope"] for c in gqa)
    assert any(not c["new"] and 0 in c["lens"] for c in gqa)            # an empty request with nothing appended
    mla = mla_case_table()
    want = set()
    for H in MLA_HS:
        for r in MLA_REGIMES:
            if r == "128" and H > 16:
                continue                                                # 132 // (B * H / 16) < 128
            for p in MLA_PLANS:
                for o in (("direct", "deferred") if r == "1" else ("merged", "deferred")):
                    want.add((H, r, p, o))
    assert _mla_cells(mla) == want
    assert {c["refusal"] for c in mla if "refusal" in c} == set(REFUSALS)
    assert {c["splits"] % 8 for c in mla if _mla_regime(c["splits"]) == "rem"} >= {3, 5, 7}


def test_host_model_matches_the_library():
    """mla_num_splits against the exported chitu_b200_mla_num_splits over a grid of arguments."""
    from chitu_b200 import _lib
    lib = _lib.load()
    for B in (1, 2, 3, 5, 8, 33, 67, 200):
        for H in (1, 8, 16, 17, 24, 32, 40, 128):
            for hint in (1, 64, 191, 192, 900, 4096, 16384, 16448, 65536):
                for ws in (0, 100, 1 << 16, 1 << 20, 1 << 24, 1 << 30):
                    assert lib.chitu_b200_mla_num_splits(B, H, hint, ws) == mla_num_splits(B, H, hint, ws), (B, H, hint, ws)
    # the workspace size of a split count is the model's
    for args in ((1, 1, 64, 1), (16, 16, 512, 8), (3, 40, 128, 5)):
        assert lib.chitu_b200_attn_workspace_bytes(*args) == split_kv_bytes(args[0] * args[1], args[2], args[3])


def test_split_ranges_tile_the_keys():
    """Every kernel's split ranges cover [0, L) once, in order; the tensor-core GQA splits start on 16-key tiles and the
    MLA splits on 64-key pages; a request shorter than the others leaves trailing splits empty."""
    for kernel, align in (("simt", 1), ("tc", GQA_TILE), ("mla", MLA_TILE)):
        for L in (0, 1, 15, 16, 17, 100, 1000, 4097):
            for S in (1, 2, 7, 13, 64, 128):
                rg = split_ranges(L, S, chunk_of(kernel, L, S))
                assert rg[0][0] == 0 and rg[-1][1] == L
                assert all(a[1] == b[0] for a, b in zip(rg, rg[1:]))
                assert all(lo % align == 0 for lo, hi in rg if hi > lo)
    assert split_ranges(20, 8, chunk_of("tc", 20, 8))[2:] == [(20, 20)] * 6


# ------------------------------------------------------------------------------------------- reference and bound
U_OUT = {BF: 2.0 ** -8, F16: 2.0 ** -11, torch.float32: 0.0}
U_P = {BF: 2.0 ** -8, F16: 2.0 ** -11}
TAU = 4.0                  # P rounding: the error is a sum of independent roundings, ~N(0, u_p^2 / 3 sum w^2 v^2)
U_ACC = 2.0 ** -16         # fp32 accumulation, exponentials and the split merge
TAU_S = 2.0 ** -18         # fp32 scores: relative to scale sum |q k| (+ the largest such, for the exponent arguments)
LSE_TOL = 2e-3             # log2 domain


def ref_splits(q, K, V, L, S, chunk, scale):
    """fp64 attention of q [Hkv, G, Dk] over keys [0, L) of K [N, Hkv, Dk] / V [N, Hkv, Dv] in S ranges of `chunk`
    keys; L is one key count or a tensor [G] of per-row counts (row g sees keys [0, L[g]), as under a causal mask).
    Returns the per-range output o [Hkv, G, S, Dv], its log2-sum-exp lse [Hkv, G, S] (-inf when empty) and the three
    bound terms rss, l1, st [Hkv, G, S, Dv]."""
    Hkv, G, Dk = q.shape
    Dv = V.shape[-1]
    Lp = S * chunk
    n = int(L.max()) if torch.is_tensor(L) else L
    Kp = torch.zeros(Lp, Hkv, Dk, dtype=torch.float64, device=q.device)
    Vp = torch.zeros(Lp, Hkv, Dv, dtype=torch.float64, device=q.device)
    Kp[:n], Vp[:n] = K[:n], V[:n]
    s = torch.einsum("kgd,lkd->kgl", q, Kp) * scale
    a = torch.einsum("kgd,lkd->kgl", q.abs(), Kp.abs()) * scale
    valid = torch.arange(Lp, device=q.device) < (L[:, None] if torch.is_tensor(L) else L)
    a = torch.where(valid, a, 0.0)
    a = a + a.amax(dim=-1, keepdim=True) if Lp else a
    s = torch.where(valid, s, -math.inf).view(Hkv, G, S, chunk)
    m = s.amax(dim=-1, keepdim=True) if chunk else torch.full((Hkv, G, S, 1), -math.inf, dtype=s.dtype, device=s.device)
    mf = torch.where(torch.isfinite(m), m, 0.0)
    e = torch.exp(s - mf)                                          # 0 on masked keys
    lsum = e.sum(-1)
    w = e / torch.where(lsum > 0, lsum, 1.0)[..., None]
    Vs = Vp.view(S, chunk, Hkv, Dv).permute(2, 0, 1, 3)            # [Hkv, S, chunk, Dv]
    o = torch.einsum("kgsc,kscd->kgsd", w, Vs)
    rss = torch.einsum("kgsc,kscd->kgsd", w * w, Vs * Vs).sqrt()
    l1 = torch.einsum("kgsc,kscd->kgsd", w, Vs.abs())
    wa = w * a.view(Hkv, G, S, chunk)
    st = torch.einsum("kgsc,kscd->kgsd", wa, Vs.abs()) + o.abs() * wa.sum(-1)[..., None]
    lse = torch.where(lsum > 0, (mf[..., 0] + torch.log(torch.where(lsum > 0, lsum, 1.0))) / math.log(2), -math.inf)
    return o, lse, (rss, l1, st)


def bound(o, terms, u_out, u_p):
    rss, l1, st = terms
    return u_out * o.abs() + TAU * u_p * rss + U_ACC * l1 + TAU_S * st


def ratio(y, ref, bnd):
    """max over elements of |y - ref| / bound; inf when y is not finite or differs where the bound is 0."""
    y = y.to(ref.device).double()
    if not bool(torch.isfinite(y).all()):
        return math.inf
    err = (y - ref).abs()
    r = torch.where(bnd > 0, err / bnd.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------- injected-error self-test of the bound
def _needle(q, K, p, L, scale, mass=0.4, dtype=BF):
    """Turn key p into one that carries about `mass` of each head's softmax over keys [0, L) (p may be L: a row past
    the end, which then carries that mass relative to the real keys)."""
    others = [j for j in range(L) if j != p]
    s = torch.einsum("kgd,lkd->kgl", q, K[others]) * scale
    target = math.log(mass / (1 - mass)) + torch.logsumexp(s, dim=-1).mean(dim=-1)      # [Hkv]
    u = q.sum(dim=1)
    u = u / u.norm(dim=-1, keepdim=True)                                                # [Hkv, Dk]
    proj = torch.einsum("kgd,kd->kg", q, u).mean(dim=-1) * scale
    K[p] = (u * (target / proj)[:, None]).to(dtype).double()


def _selftest_shapes():
    """(kernel, dtype, G, D, page, L_cache, new, splits) from the case table, one request each."""
    out = set()
    for c in gqa_case_table():
        out.add((c["kernel"], c["dtype"], c["G"], c["D"], c["page"] or GQA_TILE, c["L_max"] - 1, c["new"], c["splits"]))
    for c in mla_case_table():
        out.add(("mla", BF, min(c["H"], 4), MLA_C + MLA_R, MLA_TILE, c["L_max"] - 1, c["new"], c["splits"]))
    return sorted(out, key=lambda t: (t[0], str(t[1]), t[2:]))


def _weights_out(q, K, V, idx, scale):
    """softmax attention over the key multiset `idx` (indices into K / V, repeats count twice): [Hkv, G, Dv]."""
    idx = torch.as_tensor(idx, dtype=torch.long)
    s = torch.einsum("kgd,lkd->kgl", q, K[idx]) * scale
    return torch.einsum("kgl,lkd->kgd", torch.softmax(s, dim=-1), V[idx])


def _injections(kernel, L_cache, new, S, page):
    """(name, needle position, the key multiset a kernel with that error attends to) for one request."""
    L = L_cache + new
    rg = [r for r in split_ranges(L, S, chunk_of(kernel, L, S)) if r[1] > r[0]]
    keys = list(range(L))
    mid = rg[len(rg) // 2]
    yield "first key of a split dropped", mid[0], [j for j in keys if j != mid[0]]
    yield "last key of a split dropped", mid[1] - 1, [j for j in keys if j != mid[1] - 1]
    if len(rg) > 1:
        b = mid[0] if mid[0] > 0 else rg[1][0]
        yield "boundary key in two splits", b, keys + [b]
    if new:
        yield "appended key dropped", L_cache, keys[:-1]
    yield "one key past the end", L, keys + [L]
    if L > page:
        # the keys of the last page boundary's tile read through the previous block-table entry: same offsets, one page
        # earlier (the page's own keys are lost, the previous page's are counted twice)
        p0 = ((L - 1) // page) * page
        moved = range(p0, min(p0 + min(page, MLA_TILE if kernel == "mla" else GQA_TILE), L))
        yield "tile through the wrong block-table entry", p0, [j - page if j in moved else j for j in keys]


def test_bound_rejects_injected_errors():
    """On the case table's shapes (one request, one or two kv heads) the bound admits the correctly rounded fp64
    reference and rejects each injected error."""
    names = set()
    g = torch.Generator().manual_seed(0)
    for kernel, dtype, G, D, page, L_cache, new, S in _selftest_shapes():
        Hkv = 2 if G == 1 else 1
        Dv = MLA_C if kernel == "mla" else D
        scale = 1.0 / math.sqrt(D) if kernel != "mla" else 0.1352337788
        qs = 0.3 if kernel == "mla" else 1.0
        L = L_cache + new
        N = L + 1                                                   # one row past the end
        u_p = 0.0 if kernel == "simt" else U_P[dtype]
        def data(pos, mass=0.4):
            q = (torch.randn(Hkv, G, D, generator=g) * qs).to(dtype).double()
            K = torch.randn(N, Hkv, D, generator=g).to(dtype).double()
            _needle(q, K, pos, L, scale, mass, dtype)
            if kernel == "mla":
                return q, K, K[..., :Dv]                            # V = the first 512 columns of the same row
            V = torch.randn(N, Hkv, Dv, generator=g).to(dtype).double()
            V[pos] *= 2
            return q, K, V

        for name, pos, keyset in _injections(kernel, L_cache, new, S, page):
            q, K, V = data(pos)
            o, _, terms = ref_splits(q, K, V, L, 1, L, scale)
            o, terms = o[:, :, 0], tuple(t[:, :, 0] for t in terms)
            bnd = bound(o, terms, U_OUT[dtype], u_p)
            assert ratio(o.to(dtype), o, bnd) <= 1.0, (kernel, name)
            wrong = _weights_out(q, K, V, keyset, scale)
            names.add(name)
            assert ratio(wrong.to(dtype), o, bnd) > 1.0, (name, kernel, dtype, G, D, page, L_cache, new, S)
        # two heads swapped, and the split LSEs merged in the natural-log domain
        chunk = chunk_of(kernel, L, S)
        rg = [r for r in split_ranges(L, S, chunk) if r[1] > r[0]]
        q, K, V = data(rg[-1][0], 0.5)
        o, _, terms = ref_splits(q, K, V, L, 1, L, scale)
        o, terms = o[:, :, 0], tuple(t[:, :, 0] for t in terms)
        bnd = bound(o, terms, U_OUT[dtype], u_p)
        flat = o.reshape(-1, Dv)
        swapped = flat.clone()
        swapped[[0, 1]] = flat[[1, 0]]
        names.add("two heads swapped")
        assert ratio(swapped.view_as(o).to(dtype), o, bnd) > 1.0, ("swap", kernel, G, L_cache, S)
        if len(rg) > 1:
            op, lse, _ = ref_splits(q, K, V, L, S, chunk, scale)
            lse_ln = torch.where(torch.isfinite(lse), lse * math.log(2), -math.inf)
            w = torch.softmax(lse_ln * math.log(2), dim=-1)             # weights exp2(lse_ln - max)
            merged = torch.einsum("kgs,kgsd->kgd", w, op)
            names.add("split LSE in the natural-log domain")
            assert ratio(merged.to(dtype), o, bnd) > 1.0, ("lse", kernel, G, L_cache, S)
    assert names == {"first key of a split dropped", "last key of a split dropped", "boundary key in two splits",
                     "appended key dropped", "one key past the end", "tile through the wrong block-table entry",
                     "two heads swapped", "split LSE in the natural-log domain"}


# ------------------------------------------------------------------------------------------------ refusals (host)
def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def _last_error():
    return _lib().chitu_b200_last_error().decode(errors="replace")


def test_decode_entries_refuse_what_the_kernels_cannot_load():
    """k / v batch strides that are not 8-element multiples and operands that are not 16-byte aligned are refused by
    every decode entry before anything is launched (the tensor-core kernels stage rows with 16-byte cp.async)."""
    from chitu_b200 import _lib as L
    lib = _lib()
    A, D = 4096, 128

    def paged(q=A, kc=A, vc=A, kn=A, vn=A, ksb=1024, vsb=1024, out=A, d=D, page=256):
        return lib.chitu_b200_gqa_paged_decode(q, kc, vc, kn, vn, ksb, vsb, A, A, 4, 2, 8, 2, d, page, 0, 0.1, out,
                                               None, 0, L.CB_BF16, None)

    def rope(q=A, kn=A, vn=A, ksb=1024, vsb=1024, out=A):
        return lib.chitu_b200_gqa_paged_decode_rope(q, 8 * D, A, A, kn, vn, ksb, vsb, A, A, A, A, 4, 2, 8, 2, D, 256, 0,
                                                    0.1, out, None, 0, L.CB_BF16, None)

    def contig(q=A, kc=A, kn=A, vn=A, ksb=1024, vsb=1024, out=A, d=D):
        return lib.chitu_b200_gqa_contiguous_attn(q, kc, A, 100 * 2 * d, 100, kn, vn, ksb, 2 * d, vsb, 2 * d, A, 2, 1,
                                                  8, 2, d, 0, 0, 0.1, out, None, 0, L.CB_BF16, None)

    def mla(qn=A, qp=A, kv=A, new=A):
        return lib.chitu_b200_mla_decode(qn, qp, kv, new, A, A, 4, 2, 16, 512, 64, 64, 8, 0, 0.1, A, None, 0, None)

    bad = [(paged, "gqa_paged_decode", dict(ksb=1028)), (paged, "gqa_paged_decode", dict(vsb=1028)),
           (paged, "gqa_paged_decode", dict(ksb=1028, d=64, page=48)),       # the SIMT path keeps the same rule
           (rope, "gqa_paged_decode_rope", dict(ksb=1028, vsb=1028))]
    for name in ("q", "kc", "vc", "kn", "vn", "out"):
        bad += [(paged, "gqa_paged_decode", {name: A + 8})]
    for name in ("q", "kn", "vn", "out"):
        bad += [(rope, "gqa_paged_decode_rope", {name: A + 8})]
    bad += [(contig, "gqa_contiguous_attn", dict(ksb=1028)), (contig, "gqa_contiguous_attn", dict(vsb=1028)),
            (contig, "gqa_contiguous_attn", dict(ksb=516, vsb=516, d=64)), (contig, "gqa_contiguous_attn", dict(kn=A + 8))]
    for name in ("qn", "qp", "kv", "new"):
        bad += [(mla, "mla_decode", {name: A + 8})]
    before = L.launch_count()
    for fn, entry, kw in bad:
        assert fn(**kw) < 0, (entry, kw)
        assert entry in _last_error(), (entry, kw, _last_error())
    assert L.launch_count() == before


# ---------------------------------------------------------------------------------------------------- GPU calls
PAD = 256          # bytes of pad before and after every operand view (keeps the views 16-byte aligned)
NAN_BYTE = 0xFF    # NaN in bf16, fp16, fp8 e4m3 and fp32
SENTINEL = 0xA5


class Padded:
    """A contiguous view in the middle of a larger byte buffer; the pads hold `pad` bytes."""

    def __init__(self, t=None, pad=NAN_BYTE, fill=None, shape=None, dtype=None):
        shape, dtype = (t.shape, t.dtype) if t is not None else (shape, dtype)
        nbytes = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        self.buf = torch.full((2 * PAD + nbytes,), pad, dtype=torch.uint8, device=DEV)
        self.pad, self.nbytes = pad, nbytes
        self.bytes = self.buf[PAD:PAD + nbytes]
        self.view = self.bytes.view(dtype).view(shape)
        if t is not None:
            self.view.copy_(t)
        elif fill is not None:
            self.bytes.fill_(fill)

    def pads_intact(self):
        return bool((self.buf[:PAD] == self.pad).all()) and bool((self.buf[PAD + self.nbytes:] == self.pad).all())


def _bits(t):
    return t.contiguous().view(torch.uint8)


def _rotary(x, cos, sin, dtype):
    """Interleaved rotary in the arithmetic of the fused kernel: fp32 products, one fp32 rounding of each fma, then the
    io dtype.  x [B, H, D]; cos / sin [B, D / 2] fp32."""
    x0, x1 = x.double()[..., 0::2], x.double()[..., 1::2]
    c, s = cos.double()[:, None, :], sin.double()[:, None, :]
    o0 = (x0 * c - (x1 * s).float().double()).float()
    o1 = (x1 * c + (x0 * s).float().double()).float()
    return torch.stack([o0, o1], dim=-1).flatten(-2).to(dtype)


def _shape_keys(q, K, pos, targets, scale, dtype):
    """Set keys `pos` of K [N, Hkv, Dk] so that their mean score over the heads of q [Hkv, G, Dk] is `targets`."""
    u = q.sum(dim=1)
    u = u / u.norm(dim=-1, keepdim=True)
    proj = torch.einsum("kgd,kd->kg", q, u).mean(dim=-1) * scale
    K[pos] = (u[None] * (targets[:, None, None] / proj[None, :, None])).to(dtype).to(K.dtype)


def _needle_positions(kernel, L_cache, new, S, chunk, page):
    L = L_cache + new
    cand = {0, L_cache - 1, L_cache if new else 0}
    for lo, hi in split_ranges(L, S, chunk):
        if hi > lo:
            cand |= {lo, hi - 1}
    if page:
        cand |= {p for p in range(page, L, page)} | {p - 1 for p in range(page, L, page)}
    cand |= {t for t in range(GQA_TILE, L, GQA_TILE)}
    return sorted(x for x in cand if 0 <= x < L)


def _keys(q_eff, B, Ls, kinds_pos, Hkv, Dk, dtype, scale, g, kernel, tile):
    """Per request the io-dtype keys [L_b, Hkv, Dk] (double): random, with a needle or a ramp of tile maxima."""
    Kd = []
    for b in range(B):
        L = Ls[b]
        K = torch.randn(L + 1, Hkv, Dk, generator=g, device=DEV).to(dtype).double()
        kind, pos = kinds_pos[b]
        if L > 1 and kind == "needle":
            others = torch.arange(L, device=DEV) != pos
            s = torch.einsum("kgd,lkd->kgl", q_eff[b], K[:L][others]) * scale
            t = math.log(0.4 / 0.6) + torch.logsumexp(s, dim=-1).mean(dim=-1).mean()
            _shape_keys(q_eff[b], K, torch.tensor([pos], device=DEV), t.reshape(1), scale, dtype)
        elif L > 0 and kind == "ramp":
            # tile maxima climbing by 5 (log2) per tile, below the MLA rescale threshold of 8, and a jump of 20 every
            # seventh tile
            starts = torch.arange(0, L, tile, device=DEV)
            tt = torch.arange(len(starts), device=DEV)
            targets = math.log(2) * (5.0 * (tt % 3) + 20.0 * (tt % 7 == 6)) + 1.0
            _shape_keys(q_eff[b], K, starts, targets.double(), scale, dtype)
        Kd.append(K[:L])
    return Kd


def _split_checks(o_part, lse, ref_fn, ranges, u_p, what):
    """o_part [Hq, S, Dv], lse [Hq, S] of one request against ref_fn() = (o [Hq, S, Dv], lse, terms)."""
    o, rl, terms = ref_fn()
    worst = 0.0
    for s, (lo, hi) in enumerate(ranges):
        if hi <= lo:
            assert bool((lse[:, s] == -math.inf).all()) and bool((o_part[:, s] == 0).all()), ("empty split", s) + what
            continue
        r = ratio(o_part[:, s], o[:, s], bound(o[:, s], tuple(t[:, s] for t in terms), 0.0, u_p))
        assert r <= 1.0, ("split partial outside the bound", s, r) + what
        err = float((lse[:, s].double() - rl[:, s]).abs().max())
        assert err <= LSE_TOL, ("split LSE", s, err) + what
        worst = max(worst, r)
    return worst


def _report(entry, n, worst):
    print(f"[attn bound] entry={entry} cases={n} max|y-ref|/bound={worst:.3f}")


def _block_table(B, npages, g, num_blocks=None, top=False):
    """Shuffled page ids (the top page among them), a NaN trap page behind every unused column."""
    need = sum(npages)
    nb = max(need + 4, num_blocks or 0)
    trap = nb - 2
    if top:
        ids = [p for p in range(nb - 1, -1, -1) if p != trap][:need]
    else:
        perm = torch.randperm(nb, generator=g, device=DEV).tolist()
        ids = [nb - 1] + [p for p in perm if p not in (trap, nb - 1)][:need - 1]
    stride = max(npages) + 1
    bt = torch.full((B, stride), trap, dtype=torch.int32)
    k = 0
    for b in range(B):
        bt[b, :npages[b]] = torch.tensor(ids[k:k + npages[b]], dtype=torch.int32)
        k += npages[b]
    return bt.to(DEV), nb, trap


def _data_kinds(b, seed, has_ramp):
    kinds = ("needle", "ramp") if has_ramp else ("needle",)
    return kinds[(b + seed) % len(kinds)]


def run_gqa(c, kind, num_blocks=None, top=False):
    """One GQA case through its entry with `kind` data ("needle", "diffuse" or "ramp" per request, needle positions
    from the model); returns the worst ratio to the bound."""
    from chitu_b200._lib import check, current_stream, ptr, dtype_code
    lib = _lib()
    entry, kernel, dt = c["entry"], c["kernel"], c["dtype"]
    B, Hq, Hkv, G, D, page = c["B"], c["Hq"], c["Hkv"], c["G"], c["D"], c["page"]
    new, lens, S = c["new"], c["lens"], c["splits"]
    Ls = [L + new for L in lens]
    g = torch.Generator(device=DEV).manual_seed(1000 * c["seed"] + len(kind))
    scale = 1.0 / math.sqrt(D)
    what = (entry, kernel, str(dt), G, B, Hkv, D, page, tuple(lens), new, c["hint"], c.get("regime"), S, kind)
    chunks = [chunk_of(kernel, L, S) for L in Ls]

    q = torch.randn(B, Hkv, G, D, generator=g, device=DEV).to(dt)
    qkv_w = (Hq + 2 * Hkv) * D
    qkv = torch.randn(B, qkv_w, generator=g, device=DEV).to(dt)          # k / v rows as views of a fused output
    qkv[:, :Hq * D] = q.view(B, Hq * D)
    cos = sin = None
    q_eff = q
    if c.get("rope"):
        cos = torch.randn(B, D // 2, generator=g, device=DEV)
        sin = torch.randn(B, D // 2, generator=g, device=DEV)
        q_eff = _rotary(q.view(B, Hq, D), cos, sin, dt).view(B, Hkv, G, D)
    picks = []
    for b in range(B):
        cand = _needle_positions(kernel, lens[b], new, S, chunks[b], page)
        if c.get("rope"):
            cand = [p for p in cand if p != lens[b]] or [0]
        k = kind if kind != "mixed" else _data_kinds(b, c["seed"], True)
        picks.append((k, cand[(7 * c["seed"] + 3 * b) % len(cand)] if cand else 0))
    Kd = _keys(q_eff.double(), B, Ls, picks, Hkv, D, dt, scale, g, kernel, GQA_TILE)
    Vd = [torch.randn(L, Hkv, D, generator=g, device=DEV).to(dt).double() for L in Ls]
    for b, (k, p) in enumerate(picks):
        if k == "needle" and Ls[b] > 0:
            Vd[b][p] *= 2
    store = F8 if entry == "fp8" else dt
    if entry == "fp8":
        Kd = [k.float().to(F8).double() for k in Kd]
        Vd = [v.float().to(F8).double() for v in Vd]
    # the new rows: k_new un-rotated in the fused buffer (rope: chosen so that its rotation is the needle-shaped key)
    kn_view = qkv[:, Hq * D:(Hq + Hkv) * D].view(B, Hkv, D)
    vn_view = qkv[:, (Hq + Hkv) * D:].view(B, Hkv, D)
    for b in range(B):
        if new:
            kn_view[b] = Kd[b][lens[b]].to(dt)
            vn_view[b] = Vd[b][lens[b]].to(dt)
    if c.get("rope") and new:
        rot = _rotary(kn_view, cos, sin, dt)
        for b in range(B):
            Kd[b][lens[b]] = rot[b].double()
    if entry == "fp8" and new:                          # the appended rows are attended in their stored (e4m3) form
        for b in range(B):
            Kd[b][lens[b]] = kn_view[b].float().clamp(-448, 448).to(F8).double()
            Vd[b][lens[b]] = vn_view[b].float().clamp(-448, 448).to(F8).double()

    # caches: NaN everywhere but the cached keys of every request
    if entry == "contig":
        rows = c["rows"]
        kc = torch.full((B + 1, rows, Hkv, D), float("nan"), dtype=dt, device=DEV)
        vc = kc.clone()
        for b in range(B):
            kc[b, :lens[b]] = Kd[b][:lens[b]].to(dt)
            vc[b, :lens[b]] = Vd[b][:lens[b]].to(dt)
        bt = None
    else:
        npages = [_cdiv(L + 1, page) for L in lens]
        bt, nb, trap = _block_table(B, npages, torch.Generator(device=DEV).manual_seed(c["seed"]), num_blocks, top)
        kc = torch.full((nb, page, Hkv, D), float("nan"), dtype=dt, device=DEV)
        if entry == "fp8":
            kc = kc.to(F8)
        vc = torch.full_like(kc, float("nan")) if entry != "fp8" else kc.clone()
        for b in range(B):
            j = torch.arange(lens[b], device=DEV)
            pg, off = bt[b, j // page].long(), j % page
            kc[pg, off] = Kd[b][:lens[b]].float().to(store)
            vc[pg, off] = Vd[b][:lens[b]].float().to(store)
    big = num_blocks is not None
    if big:
        used = torch.unique(torch.cat([bt.flatten().long()]))
        kc_before, vc_before = kc[used].clone(), vc[used].clone()
    else:
        kc_before, vc_before = kc.clone(), vc.clone()

    qp = Padded(qkv)                                     # q is the first Hq * D of each fused row
    out = Padded(shape=(B, Hq, D), dtype=dt, pad=SENTINEL, fill=NAN_BYTE)
    ws = Padded(shape=(c["ws"],), dtype=torch.uint8, pad=SENTINEL, fill=0xFF) if c["ws"] is not None else None
    wsp, wsn = (ptr(ws.view), c["ws"]) if ws is not None else (None, 0)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    qv = qp.view[:, :Hq * D]
    kn = ptr(qp.view[:, Hq * D:]) if new else None
    vn = ptr(qp.view[:, (Hq + Hkv) * D:]) if new else None
    st = current_stream()
    hint = c["hint_arg"]
    if entry == "contig":
        q_dense = Padded(qv.contiguous())
        call = lambda: lib.chitu_b200_gqa_contiguous_attn(
            ptr(q_dense.view), ptr(kc), ptr(vc), kc.stride(0), rows, kn, vn, qkv_w, Hkv * D, qkv_w, Hkv * D, ptr(lens_d),
            B, 1, Hq, Hkv, D, hint, 0, scale, ptr(out.view), wsp, wsn, dtype_code(dt), st)
    elif entry == "fp8":
        call = lambda: lib.chitu_b200_gqa_paged_attn_fp8kv(
            ptr(qv), qkv_w, ptr(kc), ptr(vc), kn, vn, qkv_w, 0, qkv_w, 0, None, None, ptr(lens_d), ptr(bt), bt.stride(0),
            B, 1, Hq, Hkv, D, page, kc.shape[0], hint, 0, scale, ptr(out.view), wsp, wsn, dtype_code(dt), st)
    elif c.get("rope"):
        call = lambda: lib.chitu_b200_gqa_paged_decode_rope(
            ptr(qv), qkv_w, ptr(kc), ptr(vc), kn, vn, qkv_w, qkv_w, ptr(cos), ptr(sin), ptr(lens_d), ptr(bt),
            bt.stride(0), B, Hq, Hkv, D, page, hint, scale, ptr(out.view), wsp, wsn, dtype_code(dt), st)
    else:
        q_dense = Padded(qv.contiguous())
        call = lambda: lib.chitu_b200_gqa_paged_decode(
            ptr(q_dense.view), ptr(kc), ptr(vc), kn, vn, qkv_w, qkv_w, ptr(lens_d), ptr(bt), bt.stride(0), B, Hq, Hkv, D,
            page, hint, scale, ptr(out.view), wsp, wsn, dtype_code(dt), st)
    check(call(), str(what))
    torch.cuda.synchronize()
    first = out.view.clone()
    ws_after = ws.bytes.clone() if ws is not None else None

    # pads, caches (bit for bit but the appended rows)
    assert out.pads_intact() and qp.pads_intact() and (ws is None or ws.pads_intact()), ("pad overwritten",) + what
    for cache, before, Xd in ((kc, kc_before, Kd), (vc, vc_before, Vd)):
        want = before
        for b in range(B):
            if not new or (entry == "contig" and lens[b] >= rows):
                continue
            row = Xd[b][lens[b]].float().to(store)
            if entry == "contig":
                want[b, lens[b]] = row
            else:
                pg = int(bt[b, lens[b] // page])
                if big:
                    pg = int((used == pg).nonzero())
                want[pg, lens[b] % page] = row
        got = cache[used] if big else cache
        assert torch.equal(_bits(got), _bits(want)), ("cache changed outside the appended rows",) + what

    # the output against the fp64 reference
    u_p = 0.0 if kernel == "simt" else U_P[dt]
    worst = 0.0
    y = first.view(B, Hkv, G, D)
    for b in range(B):
        o, _, terms = ref_splits(q_eff[b].double(), Kd[b], Vd[b], Ls[b], 1, Ls[b], scale)
        o, terms = o[:, :, 0], tuple(t[:, :, 0] for t in terms)
        r = ratio(y[b], o, bound(o, terms, U_OUT[dt], u_p))
        assert r <= 1.0, ("outside the bound", b, r) + what
        worst = max(worst, r)

    # the per-split partials: the model's split count and key ranges, the rest of the workspace untouched
    if ws is not None:
        rows_ = B * Hq
        n_part = rows_ * S * (D + 1) * 4 if S > 1 else 0
        assert bool((ws_after[n_part:] == 0xFF).all()), ("workspace written past the modelled partials",) + what
        if S > 1:
            o_part = ws_after[:rows_ * S * D * 4].view(torch.float32).view(B, Hkv, G, S, D)
            lse = ws_after[rows_ * S * D * 4:n_part].view(torch.float32).view(B, Hkv, G, S)
            assert bool((ws_after[:n_part].view(torch.int32) != -1).all()), ("partial not written",) + what
            for b in range(B):
                fn = lambda b=b: _flat(ref_splits(q_eff[b].double(), Kd[b], Vd[b], Ls[b], S, chunks[b], scale))
                _split_checks(o_part[b].reshape(Hq, S, D), lse[b].reshape(Hq, S), fn,
                              split_ranges(Ls[b], S, chunks[b]), u_p, what + (b,))

    # determinism: the same call again gives the same bits
    if ws is not None:
        ws.bytes.fill_(0xFF)
    check(call(), str(what))
    torch.cuda.synchronize()
    assert torch.equal(_bits(out.view), _bits(first)), ("not deterministic",) + what
    return worst


def _flat(res):
    """ref_splits' (o, lse, (rss, l1, st)) with the kv-head and group axes merged into heads."""
    o, lse, (rss, l1, st) = res
    Hkv, G = o.shape[:2]
    m = lambda t: t.reshape(Hkv * G, *t.shape[2:])
    return m(o), m(lse), (m(rss), m(l1), m(st))

MLA_SCALE = 0.1352337788


def run_mla(c, kind):
    """One MLA case: chitu_b200_mla_decode with the case's plan words (the device plan kernel's, or a plan the kernel
    must ignore) in the workspace tail, direct / merged into `out` or deferred into absorb-o; returns the worst ratio."""
    from chitu_b200._lib import check, current_stream, ptr
    from oracle import chitu_oracle as O
    lib = _lib()
    B, H, new, lens, S = c["B"], c["H"], c["new"], c["lens"], c["splits"]
    Ls = [L + new for L in lens]
    Dk = MLA_C + MLA_R
    g = torch.Generator(device=DEV).manual_seed(1000 * c["seed"] + len(kind))
    what = ("mla", H, B, tuple(lens), new, S, c["plan"], c.get("refusal"), c["deferred"], kind)
    kps = c["kps"]
    chunks = [chunk_of("mla", L, S, k) for L, k in zip(Ls, kps)]
    q = (torch.randn(B, 1, H, Dk, generator=g, device=DEV) * 0.3).to(BF)
    picks = []
    for b in range(B):
        cand = _needle_positions("mla", lens[b], new, S, chunks[b], MLA_TILE)
        k = kind if kind != "mixed" else _data_kinds(b, c["seed"], True)
        picks.append((k, cand[(7 * c["seed"] + 3 * b) % len(cand)] if cand else 0))
    Kd = _keys(q.double(), B, Ls, picks, 1, Dk, BF, MLA_SCALE, g, "mla", MLA_TILE)
    npages = [_cdiv(L + 1, MLA_TILE) for L in lens]
    bt, nb, trap = _block_table(B, npages, torch.Generator(device=DEV).manual_seed(c["seed"]))
    cache = torch.full((nb, MLA_TILE, Dk), float("nan"), dtype=BF, device=DEV)
    for b in range(B):
        j = torch.arange(lens[b], device=DEV)
        cache[bt[b, j // MLA_TILE].long(), j % MLA_TILE] = Kd[b][:lens[b], 0].to(BF)
    before = cache.clone()
    qn = Padded(q[:, 0, :, :MLA_C].contiguous())
    qpe = Padded(q[:, 0, :, MLA_C:].contiguous())
    new_kv = Padded(torch.stack([Kd[b][lens[b], 0] if new else torch.zeros(Dk, device=DEV, dtype=torch.float64)
                                 for b in range(B)]).to(BF)) if new else None
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ws = Padded(shape=(c["ws"],), dtype=torch.uint8, pad=SENTINEL, fill=0xFF)
    st = current_stream()
    plan_view = ws.bytes[c["ws"] - PLAN_BYTES:].view(torch.int32)
    if c["plan"] == "honoured":
        incl = torch.tensor(Ls, dtype=torch.int32, device=DEV)
        check(lib.chitu_b200_attn_plan(ptr(incl), B, H, MLA_TILE, c["L_max"], ptr(ws.view), c["ws"], st), "attn_plan")
        torch.cuda.synchronize()
        got = plan_view[:7].tolist()
        assert got == [c["plan_words"][w] for w in range(7)], ("plan words differ from the model", got) + what
    else:
        plan_view[:7] = torch.tensor([c["plan_words"][w] for w in range(7)], dtype=torch.int32, device=DEV)
    plan_before = plan_view.clone()
    out = None if c["deferred"] else Padded(shape=(B, H, MLA_C), dtype=BF, pad=SENTINEL, fill=NAN_BYTE)
    call = lambda: lib.chitu_b200_mla_decode(
        ptr(qn.view), ptr(qpe.view), ptr(cache), ptr(new_kv.view) if new else None, ptr(lens_d), ptr(bt), bt.stride(0),
        B, H, MLA_C, MLA_R, MLA_TILE, nb, c["L_max"], MLA_SCALE, ptr(out.view) if out else None, ptr(ws.view),
        c["ws"], st)
    check(call(), str(what))
    torch.cuda.synchronize()
    ws_after = ws.bytes.clone()
    assert ws.pads_intact() and qn.pads_intact() and qpe.pads_intact(), ("pad overwritten",) + what
    assert torch.equal(plan_view, plan_before), ("plan changed by the decode",) + what
    want = before
    for b in range(B):
        if new:
            want[int(bt[b, lens[b] // MLA_TILE]), lens[b] % MLA_TILE] = Kd[b][lens[b], 0].to(BF)
    assert torch.equal(_bits(cache), _bits(want)), ("cache changed outside the appended rows",) + what

    u_p = U_P[BF]
    worst = 0.0
    refs = []
    for b in range(B):
        Kb = Kd[b]
        o, _, terms = ref_splits(q[b].double(), Kb, Kb[..., :MLA_C], Ls[b], 1, Ls[b], MLA_SCALE)
        refs.append((o[0, :, 0], tuple(t[0, :, 0] for t in terms)))
    partials = c["deferred"] or S > 1
    rows = B * H
    n_part = rows * S * (MLA_C + 1) * 4 if partials else 0
    assert bool((ws_after[n_part:c["ws"] - PLAN_BYTES] == 0xFF).all()), ("workspace written past the partials",) + what
    if partials:
        assert bool((ws_after[:n_part].view(torch.int32) != -1).all()), ("partial not written",) + what
        o_part = ws_after[:rows * S * MLA_C * 4].view(torch.float32).view(B, H, S, MLA_C)
        lse = ws_after[rows * S * MLA_C * 4:n_part].view(torch.float32).view(B, H, S)
        for b in range(B):
            fn = lambda b=b: _flat(ref_splits(q[b].double(), Kd[b], Kd[b][..., :MLA_C], Ls[b], S, chunks[b], MLA_SCALE))
            _split_checks(o_part[b], lse[b], fn, split_ranges(Ls[b], S, chunks[b]), u_p, what + (b,))

    if not c["deferred"]:
        assert out.pads_intact(), ("output pad overwritten",) + what
        y = out.view.clone()
    else:
        dn = dv = 128
        wkv = (torch.randn(H, dn + dv, MLA_C, generator=g, device=DEV) * 0.05).to(BF)
        x = Padded(shape=(B, H, MLA_C), dtype=BF, pad=SENTINEL, fill=NAN_BYTE)
        o = Padded(shape=(B, H * dv), dtype=BF, pad=SENTINEL, fill=NAN_BYTE)
        q8 = Padded(shape=(B, H * dv), dtype=torch.uint8, pad=SENTINEL, fill=0)
        qs = Padded(shape=(B, H), dtype=torch.float32, pad=SENTINEL, fill=0)
        check(lib.chitu_b200_mla_absorb_o_merge_quant(ptr(ws.view), c["ws"], c["L_max"], ptr(wkv), ptr(x.view),
                                                      ptr(o.view), ptr(q8.view), ptr(qs.view), B, H, dn, dv, MLA_C, st),
              "absorb_o_merge")
        torch.cuda.synchronize()
        assert x.pads_intact() and o.pads_intact() and q8.pads_intact() and qs.pads_intact(), ("pad",) + what
        y = x.view.clone()
        # absorb-o: the fp64 einsum of the kernel's own merged latent with W_UV; act_quant of its own bf16 output
        x64, w64 = y.double(), wkv[:, dn:].double()
        ref_o = torch.einsum("bhc,hdc->bhd", x64, w64).reshape(B, H * dv)
        rss = torch.einsum("bhc,hdc->bhd", x64 * x64, w64 * w64).sqrt().reshape(B, H * dv)
        r = ratio(o.view, ref_o, U_OUT[BF] * ref_o.abs() + 2.0 ** -13 * rss)
        assert r <= 1.0, ("absorb-o outside the bound", r) + what
        qo, so = O.act_quant_deepseek_v3(o.view.cpu())
        assert torch.equal(qs.view.cpu(), so) and torch.equal(q8.view.cpu(), qo.view(torch.uint8)), ("act_quant",) + what
    for b in range(B):
        o_ref, terms = refs[b]
        r = ratio(y[b], o_ref, bound(o_ref, terms, U_OUT[BF], u_p))
        assert r <= 1.0, ("outside the bound", b, r) + what
        worst = max(worst, r)

    ws.bytes.fill_(0xFF)
    plan_view.copy_(plan_before)
    check(call(), str(what))
    torch.cuda.synchronize()
    assert torch.equal(_bits(ws.bytes), _bits(ws_after)), ("partials not deterministic",) + what
    if out is not None:
        assert torch.equal(_bits(out.view), _bits(y)), ("not deterministic",) + what
    return worst


# ------------------------------------------------------------------------------------- parity over the case table
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["paged", "contig", "fp8"])
def test_gqa_case_table_parity(entry):
    """Every GQA case of the entry, on needle / ramp data and on diffuse data: inside the bound, pads and caches
    untouched but for the appended rows, every modelled split partial and LSE written and within the bound over its
    own key range, empty splits exactly 0 with LSE -inf, deterministic."""
    for kernel in GQA_KERNELS[entry]:
        cases = [c for c in gqa_case_table() if c["entry"] == entry and c["kernel"] == kernel]
        worst = 0.0
        for c in cases:
            for kind in ("mixed", "diffuse"):
                worst = max(worst, run_gqa(c, kind))
        _report(f"{entry}-{kernel}", len(cases), worst)


@pytest.mark.gpu
def test_mla_case_table_parity():
    """Every MLA case (H, split regime, plan honoured or refused, direct / merged / deferred): the same checks, plus
    the plan words of chitu_b200_attn_plan against the model, absorb-o against the fp64 einsum of the merged latent and
    the fp8 payload and scales bit for bit against act_quant of its bf16 output."""
    cases = mla_case_table()
    worst = 0.0
    for c in cases:
        for kind in ("mixed", "diffuse"):
            worst = max(worst, run_mla(c, kind))
    _report("mla", len(cases), worst)


@pytest.mark.gpu
def test_mla_plan_through_prepare_metadata():
    """B200AttnBackend.prepare_metadata_for_decode writes the model's plan where mla_attn_with_kvcache's workspace keeps
    it, for a ragged batch."""
    from chitu_b200.attn_backend import B200AttnBackend
    B, H, L_max = 5, 16, 3000
    lens = _lens(B, L_max, True, 3)
    be = B200AttnBackend(max_seq_len=L_max, max_reqs=B, n_local_heads=H)
    dl = torch.tensor(lens, dtype=torch.int32, device=DEV)
    bt = torch.zeros(B, _cdiv(L_max + 1, 64), dtype=torch.int32, device=DEV)
    be.prepare_metadata_for_decode(dl, dl + 1, bt, 64)
    torch.cuda.synchronize()
    ws, n = be._ws(B, H, MLA_C, DEV)
    want = attn_plan([L + 1 for L in lens], H, 64, L_max, n)
    assert be.last_plan()[:7].tolist() == [want[w] for w in range(7)]


@pytest.mark.gpu
def test_cache_above_2g_elements():
    """A paged cache of more than 2^31 elements per tensor, the request's pages at the top of it: the int64 offset
    arithmetic of the tensor-core kernel and its append."""
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2 ** 30:
        pytest.skip("needs about 12 GB of free device memory")
    Hkv, D, page = 8, 128, 256
    nb = (2 ** 31) // (page * Hkv * D) + 2
    c = dict(entry="paged", kernel="tc", dtype=BF, G=1, B=2, Hkv=Hkv, Hq=Hkv, D=D, page=page, L_max=700, hint="exact",
             hint_arg=700, new=True, lens=[699, 300], seed=77, rope=False, regime="2-7",
             ws=split_kv_bytes(2 * Hkv, D, 64))
    c["splits"] = gqa_splits("tc", 2, Hkv, Hkv, D, 700, c["ws"])
    assert nb * page * Hkv * D > 2 ** 31
    r = run_gqa(c, "mixed", num_blocks=nb, top=True)
    _report("paged-tc-2g", 1, r)
    torch.cuda.empty_cache()
