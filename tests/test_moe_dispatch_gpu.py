"""The MoE block (csrc/moe.cu): `fused_experts` on both of its paths, `moe_gate` on every logits path and selection
branch, and the stand-alone grouped GEMM, against fp64 references of the exact operand values, on shapes chosen by a
restatement of what the C side decides.

`_moe_path` restates the host choice between the grouped wgmma path and the pair-GEMV fallback, `_moe_plan` what the
plan kernel must write (a stable counting sort of the (token, slot) pairs by expert, cut into chunks of BN rows, and the
tile lists of both GEMMs), `_grouped_split` the stream-K split the grouped GEMM derives on the device from the number of
active tiles (read back from the partial slots after every call), and `_moe_layout` where every intermediate lives in
the workspace.  The case table holds one routing per reachable (weight mode x path x BN x plan x GEMM x regime) cell.
That is the (GEMM1 regime x GEMM2 regime) product covered per GEMM: the two launches are separate stream-K schedules,
and one chunk count feeds both, so most joint pairs would need large shapes while each GEMM's regimes do not.  The GPU
tests call the C entries on buffers they own, fill the workspace with NaN first, read it back after the call and check
every stage teacher-forced: each stage against a reference built from the kernel's own input to that stage.

The bound is the GEMM file's: |y - ref| <= u_out |ref| + tau rss, tau = 2^-13 for fp32-accumulating paths and 2^-8 for
the fp8 wgmma path.  `test_stage_checks_reject_injected_errors` shows the checks see a pair routed to the wrong
expert, a dropped routed weight, a missing chunk, a pair counted twice and a wrong activation scale."""
import functools
import itertools
import math

import numpy as np
import pytest
import torch

from oracle import chitu_oracle as O
from test_gemm_dispatch_gpu import NAN_BYTE, SENTINEL, TAU_FP32, TAU_FP8_MMA, TICKET_BYTES, Padded
from test_gemm_dispatch_gpu import _ratio as _gemm_ratio

BF, F32, F8 = torch.bfloat16, torch.float32, torch.float8_e4m3fn
DEV = "cuda:0"
U_BF16 = 2.0 ** -8

# ----------------------------------------------------------------------------------------------- host model
WMODES = ("bf16", "fp8", "soft")              # bf16 experts, block-scaled fp8 (W8A8), soft fp8 (W8A16)
WCODE = {"bf16": 0, "fp8": 1, "soft": 2}
BNS = (16, 32, 64, 128)
CB = {16: 8, 32: 4, 64: 2, 128: 1}            # split contributors the last arriver reads per round trip
REGIMES = ("whole", "slot0", "slot1", "count_gt_cb")
PLANS = ("small", "large")
MAX_TILES = 65536                             # tc_max_tiles()
PLAN_SMALL_MAX = 1024                         # kPlanThreads: moe_plan_small up to this many pairs
# a split at BN = 128 always has more than CB = 1 contributors, so it is labelled count_gt_cb
UNREACHABLE = frozenset((w, "grouped", 128, pl, gemm, r) for w in WMODES for pl in PLANS for gemm in (1, 2)
                        for r in ("slot0", "slot1"))


def _cdiv(a, b):
    return -(-a // b)


def _ratio(y, ref, rss, u_out, tau):
    """The GEMM file's max |y - ref| / bound; 0 for no rows (every pair of the call on an absent expert)."""
    return 0.0 if y.numel() == 0 else _gemm_ratio(y, ref, rss, u_out, tau)


def _align256(v):
    return (v + 255) // 256 * 256


def _chunk_rows(P, E):
    """moe_chunk_rows: twice the mean number of rows per expert, 16 .. 128."""
    BN = 16
    while BN < 128 and BN < 2 * _cdiv(P, E):
        BN *= 2
    return BN


def _moe_path(T, topk, E, N1, K1, wmode, sms=132):
    """fused_experts_impl's choice (the condition in front of the grouped path); `sms` does not enter it."""
    P = T * topk
    chunks = E + P // 16 + 1
    grouped = (P <= 8192 and E <= 1024 and N1 % 256 == 0 and K1 % 128 == 0 and (wmode != "soft" or (N1 // 2) % 128 == 0)
               and chunks * (N1 // 128) <= MAX_TILES and chunks * (K1 // 128) <= MAX_TILES)
    return "grouped" if grouped else "pair"


def _moe_plan(ids, w, E, BN, N1, K1):
    """What moe_plan_small / moe_plan_large write: stable counting sort of the pairs by expert (absent experts: pos -1,
    no row), the routed weight of every sorted row, and both tile lists in chunk order."""
    ids = np.asarray(ids).reshape(-1).astype(np.int64)
    w = np.asarray(w, dtype=np.float32).reshape(-1)
    P = ids.size
    valid = (ids >= 0) & (ids < E)
    cnt = np.bincount(ids[valid], minlength=E)
    seg = np.zeros(E + 1, np.int64)
    seg[1:] = np.cumsum(cnt)
    order = np.argsort(np.where(valid, ids, E), kind="stable")[: seg[E]]
    pos = np.full(P, -1, np.int64)
    pos[order] = np.arange(seg[E])
    chunks, tiles1, tiles2 = [], [], []
    for e in range(E):
        for cc in range(_cdiv(int(cnt[e]), BN)):
            xrow, rows = int(seg[e]) + cc * BN, min(BN, int(cnt[e]) - cc * BN)
            chunks.append((e, cc, xrow, rows))
            tiles1 += [(e * N1 + i * 128, xrow, rows) for i in range(N1 // 128)]
            tiles2 += [(e * K1 + i * 128, xrow, rows) for i in range(K1 // 128)]
    return dict(pair_sorted=order, pos=pos, seg_start=seg, w_sorted=w[order], chunks=chunks,
                tile1=np.array(tiles1, np.int64).reshape(-1, 3), tile2=np.array(tiles2, np.int64).reshape(-1, 3),
                num_tiles1=len(tiles1), num_tiles2=len(tiles2), BN=BN)


def _stages(wmode, K):
    """128-byte pipeline stages of a K-long weight row: 64 bf16 or 128 fp8 elements each."""
    return K // 64 if wmode == "bf16" else K // 128


def _grouped_per(num_tiles, S, sms):
    """tc_gemm_kernel in grouped mode (gemm_tc.cu): stages per CTA, derived on the device from *g_num_tiles; the grid
    is always `sms` CTAs."""
    total = num_tiles * S
    per = max(_cdiv(total, sms), 4)                 # >= 64 KB of weights per CTA
    if per * 8 < S:
        per = _cdiv(S, 8)                           # <= 8 CTAs per tile
    if S * 4 <= per:
        per = _cdiv(per, S) * S                     # short reductions: whole tiles only
    return per


@functools.lru_cache(maxsize=None)
def _grouped_split(num_tiles, S, sms):
    """(per, {split tile: ((cta, slot), ...)}) of a grouped launch, as `_split` derives it for the dense GEMM."""
    per, total = _grouped_per(num_tiles, S, sms), num_tiles * S
    items = {}
    for c in range(sms):
        g, g_end = min(c * per, total), min(c * per + per, total)
        while g < g_end:
            t = g // S
            s_lo = g - t * S
            s_hi = min(S, s_lo + g_end - g)
            # a CTA keeps the partial of its first work item in slot 0 and of any later one in slot 1
            items.setdefault(t, []).append((c, 0 if (c * per) // S == t else 1))
            g += s_hi - s_lo
    split = {t: tuple(v) for t, v in items.items() if len(v) > 1}
    for t, v in split.items():                      # the kernel's contributor range of a tile
        assert len(v) == ((t + 1) * S - 1) // per - (t * S) // per + 1
    return per, split


@functools.lru_cache(maxsize=None)
def _regime(num_tiles, S, BN, sms):
    """One label per launch: count_gt_cb over slot1 over slot0 over whole.  Closed form of `_grouped_split` (checked
    against it by `test_regime_closed_form_matches_the_split`): tile t has ((t+1)S - 1) // per - tS // per + 1
    contributors, a split tile's first contributor started on an earlier tile (slot 1) iff tS % per != 0, and both
    repeat with period per / gcd(S, per) in t."""
    per = _grouped_per(num_tiles, S, sms)
    if per % S == 0 or num_tiles * S <= per:
        return "whole"
    most, slot1 = 1, False
    for t in range(min(num_tiles, per // math.gcd(S, per))):
        c = ((t + 1) * S - 1) // per - (t * S) // per + 1
        if c > 1:
            most, slot1 = max(most, c), slot1 or (t * S) % per != 0
    return "count_gt_cb" if most > CB[BN] else "slot1" if slot1 else "slot0"


def _regime_of_split(num_tiles, S, BN, sms):
    _, split = _grouped_split(num_tiles, S, sms)
    if not split:
        return "whole"
    if max(len(v) for v in split.values()) > CB[BN]:
        return "count_gt_cb"
    return "slot1" if any(s for v in split.values() for _, s in v) else "slot0"


def _tc_ws_bytes(sms):
    return TICKET_BYTES + sms * 2 * 128 * 128 * 4      # tc_workspace_bytes(128, 128)


def _moe_layout(T, topk, E, N1, K1, sms):
    """{path: {array: (byte offset, bytes)}} inside the fused-experts workspace (moe_plan_layout, fused_experts_impl)."""
    P, N2 = T * topk, N1 // 2
    A = _align256(_tc_ws_bytes(sms))
    chunks = E + P // 16 + 1
    g = dict(pair_sorted=(A, 4 * P), pos=(A + 4 * P, 4 * P), seg_start=(A + 8 * P, 4 * (E + 1)),
             num_tiles=(A + 4 * (2 * P + E + 1), 8), w_sorted=(A + 4 * (2 * P + E + 3), 4 * P))
    q = A + _align256((3 * P + E + 3) * 4)
    g["tile1"] = (q, 12 * chunks * (N1 // 128))
    q += _align256(chunks * (N1 // 128 + 1) * 12)
    g["tile2"] = (q, 12 * chunks * (K1 // 128))
    q += _align256(chunks * (K1 // 128 + 1) * 12)
    for name, nbytes, reserved in (("xs", P * K1 * 2, P * K1 * 2), ("xs_s", P * (K1 // 128) * 4, P * (K1 // 128 + 1) * 4),
                                   ("c1", P * N1 * 2, P * N1 * 2), ("a2", P * N2 * 2, P * N2 * 2),
                                   ("a2_s", P * (N2 // 128) * 4, P * (N2 // 128 + 1) * 4), ("c3", P * K1 * 2, P * K1 * 2)):
        g[name] = (q, nbytes)
        q += _align256(reserved)
    p, pair = A, {}
    for name, nbytes, reserved in (("a1_q", T * K1, T * K1), ("a1_s", T * (K1 // 128) * 4, T * (K1 // 128 + 1) * 4),
                                   ("c1", P * N1 * 2, P * N1 * 2), ("a2", P * N2 * 2, P * N2 * 2),
                                   ("a2_q", P * N2, P * N2), ("a2_s", P * (N2 // 128) * 4, P * (N2 // 128 + 1) * 4),
                                   ("c3", P * K1 * 2, P * K1 * 2)):
        pair[name] = (p, nbytes)
        p += _align256(reserved)
    return {"grouped": g, "pair": pair}


def _moe_ws_bytes(T, topk, E, N1, K1, sms):
    """chitu_b200_moe_workspace_bytes restated."""
    P, N2 = T * topk, N1 // 2
    b = sum(_align256(v) for v in (T * K1, T * (K1 // 128 + 1) * 4, P * N1 * 2, P * N2 * 2, P * N2,
                                   P * (N2 // 128 + 1) * 4, P * K1 * 2)) + _align256(_tc_ws_bytes(sms))
    chunks = E + P // 16 + 1
    g = sum(_align256(v) for v in (_tc_ws_bytes(sms), (3 * P + E + 3) * 4, chunks * (N1 // 128 + 1) * 12,
                                   chunks * (K1 // 128 + 1) * 12, P * K1 * 2, P * (K1 // 128 + 1) * 4, P * N1 * 2,
                                   P * N2 * 2, P * (N2 // 128 + 1) * 4, P * K1 * 2))
    return max(b, g) + 256


# ------------------------------------------------------------------------------------------------ case table
# search domain: P and E give BN (moe_chunk_rows) and the plan (P <= 1024: small); only the routed experts' weights are
# generated (the others are NaN), so the cost of a shape is its active weight
DOMAIN_P = {"small": (16, 32, 64, 128, 256, 512, 1024), "large": (1040, 2080, 4160, 8192)}
DOMAIN_E = (1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024)
DOMAIN_N1 = tuple(256 * j for j in (1, 2, 3, 4, 6, 8, 12, 16, 24, 31, 32, 62, 63, 64))
DOMAIN_K1 = tuple(128 * j for j in (1, 2, 3, 4, 6, 8, 12, 16, 17, 24, 31, 32, 48, 56, 62, 63, 64))
DOMAIN_CHUNKS = tuple(range(1, 49)) + (56, 64, 80, 96, 128, 160, 192, 256)
MAX_ACTIVE_WEIGHT = 1 << 25                       # elements of the routed experts' weights of one GEMM
MAX_WEIGHT = 1 << 28                              # elements of one whole expert stack (mostly NaN)

# explicit cases beside the cell table: (wmode, T, topk, E, N1, K1, routing, ids dtype, weight dtype, residual)
PAIR_CASES = (
    ("bf16", 5, 3, 6, 384, 256, "random", torch.int64, F32, True),        # N1 % 256 != 0
    ("bf16", 4, 2, 3, 384, 144, "random", torch.int32, BF, False),        # and K1 % 128 != 0
    ("soft", 5, 3, 6, 384, 256, "random", torch.int32, F32, True),        # (N1 / 2) % 128 != 0
    ("soft", 2, 4, 5, 384, 384, "random", torch.int64, BF, False),
    ("fp8", 3, 4, 1040, 256, 128, "random", torch.int64, F32, True),      # E > 1024
    ("fp8", 2100, 4, 8, 256, 128, "random", torch.int32, BF, False),      # P > 8192
)
GROUPED_EXTRAS = (
    (40, 3, 8, 256, 256, "shared", torch.int64, BF, True),     # every token's last id is expert 7 with weight 1: 2 chunks
    (1, 1, 1, 256, 128, "random", torch.int32, F32, False),    # E = 1, P = 1
    (40, 1, 1, 256, 256, "random", torch.int64, F32, True),    # E = 1, BN = 128
    (4, 2, 4, 256, 128, "absent", torch.int32, BF, True),      # every pair absent: no tile at all
    (6, 3, 5, 256, 256, "random", torch.int32, BF, False),     # duplicates and an all-absent token
)


def _chunk_counts(P, E, BN, na):
    """Chunks per routed expert for `na` chunks in all, or None when P pairs cannot fill them (every chunk needs a row).
    With two or more chunks, one expert gets at least two (spread over min(E, na - 1) experts) when the pairs allow."""
    for n in ((min(E, na - 1), min(E, na)) if na >= 2 else (1,)):
        nch = [na // n + (1 if k < na % n else 0) for k in range(n)]
        if sum((c - 1) * BN + 1 for c in nch) <= P:
            return nch
    return None


@functools.lru_cache(maxsize=None)
def _search(wmode, sms):
    """{grouped cell: (cost, T, topk, E, N1, K1, chunks)} over the search domain.  A cell is (wmode, "grouped", BN,
    plan, GEMM 1 | 2, that GEMM's regime): the issue's (GEMM1 regime x GEMM2 regime) product is covered per GEMM,
    since the two launches are independent stream-K schedules and one chunk count feeds both, which makes most joint
    pairs unreachable at small sizes."""
    best = {}
    for plan, ps in DOMAIN_P.items():
        for P in ps:
            for E in DOMAIN_E:
                BN = _chunk_rows(P, E)
                nas = [na for na in DOMAIN_CHUNKS if _chunk_counts(P, E, BN, na)]
                for N1 in DOMAIN_N1:
                    for K1 in DOMAIN_K1:
                        if E * N1 * K1 > MAX_WEIGHT:
                            continue
                        for na in nas:
                            active = min(E, na) * N1 * K1
                            if active > MAX_ACTIVE_WEIGHT:
                                continue
                            cost = (active + E * N1 * K1 // 16 + P * (N1 + K1), na)
                            for gemm, r in ((1, _regime(na * (N1 // 128), _stages(wmode, K1), BN, sms)),
                                            (2, _regime(na * (K1 // 128), _stages(wmode, N1 // 2), BN, sms))):
                                key = (wmode, "grouped", BN, plan, gemm, r)
                                if key not in best or cost < best[key][0]:
                                    best[key] = (cost, P // 2, 2, E, N1, K1, na)
    return best


@functools.lru_cache(maxsize=None)
def _case_table(sms):
    """Per weight mode: one routing per reachable grouped cell (the cheapest weight, then the fewest chunks; cells that
    share a routing share a case), then the pair-GEMV cases and the extras.  ids / weight dtypes and the residual rotate
    over the grouped cases."""
    cases = []
    for wmode in WMODES:
        shapes = {}
        for key, (_, *shape) in sorted(_search(wmode, sms).items()):
            shapes.setdefault(tuple(shape), set()).add(key)
        for i, ((T, topk, E, N1, K1, na), cells) in enumerate(shapes.items()):
            cases.append(dict(wmode=wmode, T=T, topk=topk, E=E, N1=N1, K1=K1, routing="chunks", na=na,
                              ids_dtype=(torch.int32, torch.int64)[i % 2], tw_dtype=(BF, F32)[(i // 2) % 2],
                              residual=(i // 4) % 2 == 1, cell=frozenset(cells)))
        for T, topk, E, N1, K1, routing, idt, twt, res in GROUPED_EXTRAS:
            cases.append(dict(wmode=wmode, T=T, topk=topk, E=E, N1=N1, K1=K1, routing=routing, na=None,
                              ids_dtype=idt, tw_dtype=twt, residual=res, cell=None))
    for wmode, T, topk, E, N1, K1, routing, idt, twt, res in PAIR_CASES:
        cases.append(dict(wmode=wmode, T=T, topk=topk, E=E, N1=N1, K1=K1, routing=routing, na=None, ids_dtype=idt,
                          tw_dtype=twt, residual=res, cell=frozenset({(wmode, "pair")})))
    for i, c in enumerate(cases):
        c["seed"] = 1000 + i
    return tuple(cases)


def _routing(case):
    """(ids [T, topk] int64, routed weights [T, topk] fp32 in [0.25, 1)) of a case."""
    T, topk, E = case["T"], case["topk"], case["E"]
    P = T * topk
    rng = np.random.default_rng(case["seed"])
    w = rng.uniform(0.25, 1.0, (T, topk)).astype(np.float32)
    if case["routing"] == "chunks":
        BN, na = _chunk_rows(P, E), case["na"]
        nch = _chunk_counts(P, E, BN, na)
        cnt = [(c - 1) * BN + 1 for c in nch]
        cap = [c * BN for c in nch]
        budget = P - sum(cnt)
        k = 0
        while budget > 0 and any(c < m for c, m in zip(cnt, cap)):
            if cnt[k] < cap[k]:
                cnt[k] += 1
                budget -= 1
            k = (k + 1) % len(cnt)
        experts = rng.permutation(E)[: len(cnt)]
        valid = np.repeat(experts, cnt)
        rng.shuffle(valid)
        ids = np.concatenate([np.full(P - valid.size, -1), valid]).reshape(T, topk)   # absent pairs first
    elif case["routing"] == "shared":
        ids = rng.integers(0, E - 1, (T, topk))
        ids[:, -1] = E - 1
        w[:, -1] = 1.0
        ids[0, 1] = ids[0, 0]
    elif case["routing"] == "absent":
        ids = np.full((T, topk), -1)
    else:
        ids = rng.integers(0, E, (T, topk))
        if T > 1:
            ids[0, :] = -1                                # a token whose experts are all absent
            ids[-1, 0] = -1
        if T > 2 and topk > 1:
            ids[1, 1] = ids[1, 0]                         # a duplicate id within a token
    return ids.astype(np.int64), w


def _case_cells(case, sms):
    """The cells a case lands in, from its routing: {(wmode, "pair")} or one grouped cell per GEMM."""
    wmode, T, topk, E, N1, K1 = (case[k] for k in ("wmode", "T", "topk", "E", "N1", "K1"))
    path = _moe_path(T, topk, E, N1, K1, wmode, sms)
    if path == "pair":
        return frozenset({(wmode, "pair")})
    P = T * topk
    ids, w = _routing(case)
    BN = _chunk_rows(P, E)
    plan = _moe_plan(ids, w, E, BN, N1, K1)
    pl = "small" if P <= PLAN_SMALL_MAX else "large"
    return frozenset({(wmode, "grouped", BN, pl, 1, _regime(plan["num_tiles1"], _stages(wmode, K1), BN, sms)),
                      (wmode, "grouped", BN, pl, 2, _regime(plan["num_tiles2"], _stages(wmode, N1 // 2), BN, sms))})


@pytest.mark.parametrize("sms", [132, 114])
def test_case_table_covers_every_reachable_cell(sms):
    """The routings land in their cells, and the table hits every (wmode x path x BN x plan x GEMM x regime) cell but the
    UNREACHABLE ones, which no shape can reach: at BN = 128 the fix-up reads CB = 1 contributor per round trip and a
    split tile has at least two, so every split launch there is count_gt_cb (checked below over a sweep of launches)."""
    table = _case_table(sms)
    hit = set()
    for c in table:
        cells = _case_cells(c, sms)
        if c["cell"] is not None:
            assert cells >= c["cell"], (c, cells)
        hit |= cells
    grouped = {(w, "grouped", bn, pl, g, r) for w in WMODES for bn in BNS for pl in PLANS for g in (1, 2) for r in REGIMES}
    everything = grouped | {(w, "pair") for w in WMODES}
    assert hit == everything - UNREACHABLE, sorted(everything - UNREACHABLE - hit)
    for nt in range(1, 200):
        for S in range(1, 130):
            assert _regime(nt, S, 128, sms) in ("whole", "count_gt_cb")
    print(f"[moe table] sms={sms} cases={len(table)} cells hit={len(hit)} unreachable={len(UNREACHABLE)}")


def test_regime_closed_form_matches_the_split():
    """`_regime` (closed form) == the regime of the CTA-by-CTA split `_grouped_split`, on a sweep and on every launch of
    the table."""
    for sms in (132, 114):
        keys = {(nt, S, bn) for nt in range(1, 70) for S in range(1, 70) for bn in BNS}
        for c in _case_table(sms):
            if c["routing"] == "chunks":
                nt1 = c["na"] * (c["N1"] // 128)
                nt2 = c["na"] * (c["K1"] // 128)
                bn = _chunk_rows(c["T"] * c["topk"], c["E"])
                keys |= {(nt1, _stages(c["wmode"], c["K1"]), bn), (nt2, _stages(c["wmode"], c["N1"] // 2), bn)}
        for nt, S, bn in keys:
            assert _regime(nt, S, bn, sms) == _regime_of_split(nt, S, bn, sms), (nt, S, bn, sms)


def test_table_covers_the_routing_edges():
    """Multi-chunk experts, the shared expert, duplicates, absent experts, an all-absent token, E = 1, P = 1, both id and
    weight dtypes and the residual on both paths of every weight mode."""
    table = _case_table(132)
    for wmode in WMODES:
        for path in ("grouped", "pair"):
            cs = [c for c in table if c["wmode"] == wmode and _moe_path(c["T"], c["topk"], c["E"], c["N1"], c["K1"],
                                                                        wmode) == path]
            assert {c["ids_dtype"] for c in cs} == {torch.int32, torch.int64}, (wmode, path)
            assert {c["tw_dtype"] for c in cs} == {BF, F32}, (wmode, path)
            assert {c["residual"] for c in cs} == {True, False}, (wmode, path)
            absent_token = dup = False
            for c in cs:
                ids, _ = _routing(c)
                absent_token |= bool(((ids < 0).all(axis=1)).any())
                dup |= any(len(set(r[r >= 0].tolist())) < int((r >= 0).sum()) for r in ids)
            assert absent_token and dup, (wmode, path)
        gs = [c for c in table if c["wmode"] == wmode and c["routing"] == "chunks"]
        assert any(max(_moe_plan(*_routing(c), c["E"], _chunk_rows(c["T"] * c["topk"], c["E"]), c["N1"],
                                 c["K1"])["chunks"], key=lambda ch: ch[1])[1] >= 1 for c in gs)      # an expert in 2 chunks
        assert {c["routing"] for c in table if c["wmode"] == wmode} >= {"shared", "absent"}
        assert any(c["E"] == 1 and c["T"] * c["topk"] == 1 for c in table if c["wmode"] == wmode)
    pair = [c for c in table if (c["wmode"], "pair") in (c["cell"] or ())]
    assert any(c["wmode"] == "fp8" and c["E"] > 1024 for c in pair)
    assert any(c["wmode"] == "fp8" and c["T"] * c["topk"] > 8192 for c in pair)


def test_plan_model_invariants():
    """The plan model is a stable permutation of the valid pairs; chunks tile every expert's rows with <= BN rows each;
    the tile lists fit the workspace's lists."""
    for c in _case_table(132):
        P = c["T"] * c["topk"]
        if _moe_path(c["T"], c["topk"], c["E"], c["N1"], c["K1"], c["wmode"]) != "grouped":
            continue
        ids, w = _routing(c)
        BN = _chunk_rows(P, c["E"])
        pl = _moe_plan(ids, w, c["E"], BN, c["N1"], c["K1"])
        flat = ids.reshape(-1)
        ps = pl["pair_sorted"]
        assert sorted(ps.tolist()) == [p for p in range(P) if 0 <= flat[p] < c["E"]]
        assert all(flat[a] < flat[b] or (flat[a] == flat[b] and a < b) for a, b in zip(ps, ps[1:]))
        assert sum(r for _, _, _, r in pl["chunks"]) == ps.size and all(0 < r <= BN for *_, r in pl["chunks"])
        chunks = c["E"] + P // 16 + 1
        assert len(pl["chunks"]) <= chunks


def test_layout_fits_the_workspace():
    """Every array of both paths lies inside chitu_b200_moe_workspace_bytes, none overlaps another, and the byte count
    restated here equals the library's."""
    from chitu_b200 import _lib as L
    lib = L.load()
    lib_sms = (lib.chitu_b200_linear_workspace_bytes(128, 128) - TICKET_BYTES) // (2 * 128 * 128 * 4)
    for c in _case_table(132):
        args = (c["T"], c["topk"], c["E"], c["N1"], c["K1"])
        nbytes = lib.chitu_b200_moe_workspace_bytes(*args)
        assert nbytes == _moe_ws_bytes(*args, lib_sms), args
        for sms in (lib_sms, 114, 132):
            for path, arrays in _moe_layout(*args, sms).items():
                spans = sorted(arrays.values())
                assert spans[0][0] >= _tc_ws_bytes(sms)                     # behind the tickets and partial slots
                assert all(a[0] + a[1] <= b[0] for a, b in zip(spans, spans[1:])), (path, args)
                assert spans[-1][0] + spans[-1][1] <= _moe_ws_bytes(*args, sms), (path, args)


# ------------------------------------------------------------------------------------------ operands, references
def _fp8_stack(E, N, K, g):
    """E block-quantised weights [E, N, K] fp8 + scales [E, ceil(N/128), ceil(K/128)]."""
    w = torch.randn(E, N, K, generator=g) * 0.05
    nb, kb = _cdiv(N, 128), _cdiv(K, 128)
    wp = torch.zeros(E, nb * 128, kb * 128)
    wp[:, :N, :K] = w
    blocks = wp.view(E, nb, 128, kb, 128)
    s = blocks.abs().amax(dim=(2, 4)).clamp(min=1e-8) / 448.0
    q = (blocks / s[:, :, None, :, None]).reshape(E, nb * 128, kb * 128)[:, :N, :K].to(F8)
    return q.contiguous(), s.float().contiguous()


def _operands(case):
    """Host operands of a case.  Only the routed experts get weights; every other expert's weights and scales are NaN,
    so a kernel that read them would produce NaN."""
    wmode, T, topk, E, N1, K1 = (case[k] for k in ("wmode", "T", "topk", "E", "N1", "K1"))
    g = torch.Generator().manual_seed(case["seed"])
    tok = 2.0 ** (torch.arange(T) % 4 - 1).float()[:, None]        # neighbouring tokens differ in scale
    op = dict(case=case, x=(torch.randn(T, K1, generator=g) * tok).to(BF))
    ids, w = _routing(case)
    active = torch.tensor(sorted({int(e) for e in ids.reshape(-1) if 0 <= e < E}), dtype=torch.long)
    na = active.numel()

    def stack(N, K):
        """(weights as the kernel reads them, block scales or None, weights the reference multiplies)."""
        if wmode == "bf16":
            full = torch.full((E, N, K), float("nan"), dtype=BF)
            if na:
                full[active] = (torch.randn(na, N, K, generator=g) * 0.05).to(BF)
            return full, None, full
        q = torch.full((E, N, K), NAN_BYTE, dtype=torch.uint8)
        sc = torch.full((E, _cdiv(N, 128), _cdiv(K, 128)), float("nan"))
        ref = torch.full((E, N, K), float("nan"), dtype=BF) if wmode == "soft" else None
        if na:
            qa, sa = _fp8_stack(na, N, K, g)
            q[active], sc[active] = qa.view(torch.uint8), sa
            if wmode == "soft":      # the weights the soft path multiplies: bf16(fp8 * s)
                ref[active] = O.weight_dequant_soft_fp8(qa, sa)
        q = q.view(F8)
        return q, sc, (q if ref is None else ref)

    op["w1"], op["w1_s"], op["w1r"] = stack(N1, K1)
    op["w2"], op["w2_s"], op["w2r"] = stack(K1, N1 // 2)
    op["ids"] = torch.from_numpy(ids).to(case["ids_dtype"])
    op["tw"] = torch.from_numpy(w).to(case["tw_dtype"])
    op["tw32"] = op["tw"].float()                                     # what the kernel multiplies
    op["res"] = (torch.randn(T, K1, generator=g)).to(BF) if case["residual"] else None
    return op


def _expert_gemm(a, a_s, wr, w_s, experts, fp8, scale=None):
    """fp64 reference and rss of rows a[i] . wr[experts[i]]^T, [R, N]; fp8: per 128-K block, (a . w) * a_s * w_s."""
    dev = a.device
    R, N, K = a.shape[0], wr.shape[1], wr.shape[2]
    ref = torch.zeros(R, N, dtype=torch.float64, device=dev)
    ss = torch.zeros_like(ref)
    for e in torch.unique(experts).tolist():
        idx = torch.nonzero(experts == e).flatten()
        A, W = a[idx].double(), wr[e].to(dev).double()
        if fp8:
            KB = K // 128
            A3, W3 = A.view(-1, KB, 128), W.view(N, KB, 128)
            sc = a_s[idx].double()[:, None, :] * w_s[e].to(dev).double().repeat_interleave(128, dim=0)[None, :N, :]
            ref[idx] = (torch.einsum("rkc,nkc->rnk", A3, W3) * sc).sum(-1)
            ss[idx] = (torch.einsum("rkc,nkc->rnk", A3 * A3, W3 * W3) * sc * sc).sum(-1)
        else:
            ref[idx] = A @ W.T
            ss[idx] = (A * A) @ (W * W).T
    if scale is not None:
        s = scale.to(dev).double()[:, None]
        ref, ss = ref * s, ss * s * s
    return ref, ss.sqrt()


def _ordered(v):
    """bf16 -> integer key that counts ulps across zero."""
    b = v.contiguous().view(torch.int16).int()
    return torch.where(b >= 0, b, -(b & 0x7FFF))


def _from_ordered(o):
    return torch.where(o >= 0, o, (-o) | 0x8000).to(torch.int32).to(torch.int16).view(BF)


def _bf16_step(v, d):
    return _from_ordered(_ordered(v) + d)


def _silu_window(c1):
    """[lo, hi] of bf16(bf16(silu(g)) u) with one bf16 ulp allowed at each of the two roundings (fp64 silu)."""
    N2 = c1.shape[1] // 2
    g, u = c1[:, :N2].double(), c1[:, N2:].double()
    s = (g / (1.0 + torch.exp(-g))).to(BF)
    cands = torch.stack([(_bf16_step(s, d).double() * u).to(BF).double() for d in (-1, 0, 1)])
    lo, hi = cands.min(dim=0)[0].to(BF), cands.max(dim=0)[0].to(BF)
    return _bf16_step(lo, -1).double(), _bf16_step(hi, 1).double()


def _fp8_in_window(q, s, lo, hi):
    """per_token_group_quant_fp8 of some bf16 a2 in [lo, hi] (the one-ulp-per-rounding window): every group's scale lies
    between those of the window's smallest and largest amax, and every fp8 value is the quantisation, with the kernel's
    own scale, of a value in the window (both maps are monotone)."""
    R, N = lo.shape
    g = lambda v: v.view(R, N // 128, 128)                                           # noqa: E731
    straddle = (lo <= 0) & (hi >= 0)
    mag_lo = torch.where(straddle, torch.zeros_like(lo), torch.minimum(lo.abs(), hi.abs()))
    mag_hi = torch.maximum(lo.abs(), hi.abs())
    s_lo = g(mag_lo).amax(-1).float().clamp(min=1e-10) / 448.0
    s_hi = g(mag_hi).amax(-1).float().clamp(min=1e-10) / 448.0
    sk = s.float()
    if not bool(((sk >= s_lo) & (sk <= s_hi)).all()):
        return False
    se = sk.repeat_interleave(128, dim=1)
    q_lo = (lo.float() / se).clamp(-448.0, 448.0).to(F8).float()
    q_hi = (hi.float() / se).clamp(-448.0, 448.0).to(F8).float()
    qk = q.float()
    return bool(((qk >= q_lo) & (qk <= q_hi)).all())


def _silu_mul_f32(c1):
    """moe_silu_quant_kernel's arithmetic: bf16(bf16(g / (1 + expf(-g))) * u) in fp32."""
    N2 = c1.shape[1] // 2
    g, u = c1[:, :N2].float(), c1[:, N2:].float()
    return ((g / (1.0 + torch.exp(-g))).to(BF).float() * u).to(BF)


def _bits(t):
    t = t.contiguous()
    return t.view(torch.uint8) if t.element_size() == 1 else t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _same_bits(a, b):
    return torch.equal(_bits(a.cpu()), _bits(b.cpu()))


def _quant(v):
    """per_token_group_quant_fp8 of bf16 rows (the oracle, on the host)."""
    return O.per_token_group_quant_fp8(v.float().cpu(), 128)


def _combine(c3, pos, T, topk, res):
    """out[t] = sum_j c3[pos[t, j]] in fp32, j in order, absent pairs skipped; residual: bf16(bf16(sum) + res)."""
    K1 = c3.shape[1]
    s = torch.zeros(T, K1, dtype=F32, device=c3.device)
    pos = pos.to(c3.device).view(T, topk)
    for j in range(topk):
        r = pos[:, j]
        ok = r >= 0
        s[ok] = s[ok] + c3[r[ok]].float()
    out = s.to(BF)
    if res is not None:
        out = (out.float() + res.to(c3.device).float()).to(BF)
    return out


def _tau(wmode, path):
    return TAU_FP8_MMA if wmode == "fp8" and path == "grouped" else TAU_FP32


def _check_grouped(op, got, pl):
    """Every stage of the grouped path against the model and a reference built from the kernel's own input to that
    stage.  Returns {stage: max |y - ref| / bound}; raises AssertionError on the first violation."""
    case = op["case"]
    wmode, T, topk, E, N1, K1 = (case[k] for k in ("wmode", "T", "topk", "E", "N1", "K1"))
    P, N2, fp8 = T * topk, N1 // 2, wmode == "fp8"
    tau = _tau(wmode, "grouped")
    what = (wmode, T, topk, E, N1, K1)
    tot = int(pl["seg_start"][E])
    for name in ("pos", "seg_start", "tile1", "tile2"):
        assert np.array_equal(np.asarray(got[name]), pl[name]), ("plan " + name,) + what
    assert np.array_equal(np.asarray(got["pair_sorted"])[:tot], pl["pair_sorted"]), ("plan pair_sorted",) + what
    assert np.array_equal(np.asarray(got["w_sorted"])[:tot], pl["w_sorted"]), ("plan w_sorted",) + what
    assert (got["num_tiles1"], got["num_tiles2"]) == (pl["num_tiles1"], pl["num_tiles2"]), ("plan num_tiles",) + what
    dev = got["c1"].device
    ps = torch.as_tensor(pl["pair_sorted"], device=dev)
    tok = ps // topk
    experts = op["ids"].to(dev).reshape(-1).long()[ps]
    x = op["x"].to(dev)
    # gathered activations: bit-exact
    xs, xs_s = got["xs"][:tot], got["xs_s"][:tot] if fp8 else None
    if fp8:
        q, s = _quant(x[tok])
        assert _same_bits(xs, q) and _same_bits(xs_s, s), ("xs quantisation",) + what
    else:
        assert _same_bits(xs, x[tok]), ("xs gather",) + what
    # c1: rows past the last valid one are never written
    c1 = got["c1"]
    assert bool((_bits(c1[tot:]) == -1).all()), ("c1 written past seg_start[E]",) + what
    ref, rss = _expert_gemm(xs, xs_s, op["w1r"], op["w1_s"], experts, fp8)
    stats = {"c1": _ratio(c1[:tot], ref, rss, U_BF16, tau)}
    assert stats["c1"] <= 1.0, ("c1 outside the bound", stats["c1"]) + what
    # a2 from the kernel's own c1
    c1v = c1[:tot]
    if fp8:
        a2, a2_s = got["a2"][:tot], got["a2_s"][:tot]
        assert _fp8_in_window(a2, a2_s, *_silu_window(c1v)), ("a2 quantisation outside the window",) + what
    else:
        lo, hi = _silu_window(c1v)
        a = got["a2"][:tot].double()
        assert bool(((a >= lo) & (a <= hi)).all()), ("a2 outside one ulp per rounding",) + what
        a2, a2_s = got["a2"][:tot], None
    # c3 from the kernel's own a2, times the routed weight of the sorted row
    wsorted = torch.as_tensor(pl["w_sorted"], device=dev)
    ref, rss = _expert_gemm(a2, a2_s, op["w2r"], op["w2_s"], experts, fp8, scale=wsorted)
    stats["c3"] = _ratio(got["c3"][:tot], ref, rss, U_BF16, tau)
    assert stats["c3"] <= 1.0, ("c3 outside the bound", stats["c3"]) + what
    want = _combine(got["c3"], torch.as_tensor(pl["pos"]), T, topk, op["res"])
    assert _same_bits(got["out"], want), ("combine not bit-exact",) + what
    return stats


def _check_pair(op, got):
    """Every stage of the pair-GEMV path (pair order, absent experts give exact zero rows)."""
    case = op["case"]
    wmode, T, topk, E, N1, K1 = (case[k] for k in ("wmode", "T", "topk", "E", "N1", "K1"))
    P, fp8 = T * topk, wmode == "fp8"
    what = (wmode, T, topk, E, N1, K1)
    dev = got["c1"].device
    ids = op["ids"].to(dev).reshape(-1).long()
    valid = (ids >= 0) & (ids < E)
    vi = torch.nonzero(valid).flatten()
    tok = torch.arange(P, device=dev) // topk
    x = op["x"].to(dev)
    if fp8:
        q, s = _quant(x)
        assert _same_bits(got["a1_q"], q) and _same_bits(got["a1_s"], s), ("a1 quantisation",) + what
        a, a_s = got["a1_q"][tok[vi]], got["a1_s"][tok[vi]]
    else:
        a, a_s = x[tok[vi]], None
    c1 = got["c1"]
    assert bool((_bits(c1[~valid]) == 0).all()), ("c1 of an absent pair not zero",) + what
    ref, rss = _expert_gemm(a, a_s, op["w1r"], op["w1_s"], ids[vi], fp8)
    stats = {"c1": _ratio(c1[vi], ref, rss, U_BF16, TAU_FP32)}
    assert stats["c1"] <= 1.0, ("c1 outside the bound", stats["c1"]) + what
    lo, hi = _silu_window(c1)
    a2 = got["a2"].double()
    assert bool(((a2 >= lo) & (a2 <= hi)).all()), ("a2 outside one ulp per rounding",) + what
    if fp8:
        q, s = _quant(got["a2"])
        assert _same_bits(got["a2_q"], q) and _same_bits(got["a2_s"], s), ("a2 quantisation",) + what
        a, a_s = got["a2_q"][vi], got["a2_s"][vi]
    else:
        a, a_s = got["a2"][vi], None
    c3 = got["c3"]
    assert bool((_bits(c3[~valid]) == 0).all()), ("c3 of an absent pair not zero",) + what
    ref, rss = _expert_gemm(a, a_s, op["w2r"], op["w2_s"], ids[vi], fp8, scale=op["tw32"].reshape(-1).to(dev)[vi])
    stats["c3"] = _ratio(c3[vi], ref, rss, U_BF16, TAU_FP32)
    assert stats["c3"] <= 1.0, ("c3 outside the bound", stats["c3"]) + what
    want = _combine(c3, torch.arange(P), T, topk, op["res"])            # moe_sum adds the zero rows of absent pairs
    assert _same_bits(got["out"], want), ("sum not bit-exact",) + what
    return stats


# ---------------------------------------------------------------------- injected-error self-test of the checks
def _simulate_grouped(op, pl):
    """The stages a correct kernel writes (fp64 references rounded once), on the host."""
    case = op["case"]
    wmode, T, topk, E, N1, K1 = (case[k] for k in ("wmode", "T", "topk", "E", "N1", "K1"))
    P, fp8 = T * topk, wmode == "fp8"
    tot = int(pl["seg_start"][E])
    ps = torch.as_tensor(pl["pair_sorted"])
    experts = op["ids"].reshape(-1).long()[ps]
    got = {k: pl[k] for k in ("pair_sorted", "pos", "seg_start", "w_sorted", "tile1", "tile2", "num_tiles1", "num_tiles2")}
    rows = op["x"][ps // topk]
    if fp8:
        got["xs"], got["xs_s"] = _quant(rows)
    else:
        got["xs"] = rows.clone()
    ref, _ = _expert_gemm(got["xs"], got.get("xs_s"), op["w1r"], op["w1_s"], experts, fp8)
    got["c1"] = torch.full((P, N1), -1, dtype=torch.int16).view(BF)
    got["c1"][:tot] = ref.to(BF)
    a2 = _silu_mul_f32(got["c1"][:tot])
    if fp8:
        got["a2"], got["a2_s"] = _quant(a2)
    else:
        got["a2"] = a2
    ref, _ = _expert_gemm(got["a2"], got.get("a2_s"), op["w2r"], op["w2_s"], experts, fp8,
                          scale=torch.as_tensor(pl["w_sorted"]))
    got["c3"] = ref.to(BF)
    got["out"] = _combine(got["c3"], torch.as_tensor(pl["pos"]), T, topk, op["res"])
    return got


def _self_test_case(wmode, routing, T, topk, E, N1, K1):
    case = dict(wmode=wmode, T=T, topk=topk, E=E, N1=N1, K1=K1, routing=routing, na=None, ids_dtype=torch.int64,
                tw_dtype=BF, residual=True, seed=77, cell=None)
    op = _operands(case)
    ids, w = _routing(case)
    pl = _moe_plan(ids, op["tw32"].numpy(), E, _chunk_rows(T * topk, E), N1, K1)
    return op, pl, _simulate_grouped(op, pl)


def test_stage_checks_reject_injected_errors():
    """The stage checks pass a correct simulation and reject: a pair routed to a neighbouring expert, a dropped routed
    weight, the second chunk of an expert missing, a pair counted twice in the combine, and an activation scale from the
    neighbouring 128-group."""
    op, pl, good = _self_test_case("bf16", "shared", 40, 3, 8, 256, 256)
    assert max(pl["chunks"], key=lambda c: c[1])[1] == 1          # expert 7 (40 rows, BN 32) has a second chunk
    _check_grouped(op, good, pl)
    ps = pl["pair_sorted"]
    experts = op["ids"].reshape(-1).long()[torch.as_tensor(ps)]

    def rejects(mutate):
        got = {k: (v.clone() if torch.is_tensor(v) else np.copy(v) if isinstance(v, np.ndarray) else v)
               for k, v in good.items()}
        mutate(got)
        with pytest.raises(AssertionError):
            _check_grouped(op, got, pl)

    r = 5
    e = int(experts[r])

    def neighbour(got):                                           # row r multiplied by expert e + 1's weights
        wrong = got["xs"][r:r + 1].double() @ op["w1r"][(e + 1) % 8].double().T
        got["c1"][r] = wrong.to(BF)[0]
    rejects(neighbour)
    r3 = int(np.argmax(np.abs(pl["w_sorted"] - 1.0)))              # the row whose weight is farthest from 1

    def no_weight(got):
        got["c3"][r3] = (got["c3"][r3].double() / float(pl["w_sorted"][r3])).to(BF)
    rejects(no_weight)
    e7, _, xrow, rows = [c for c in pl["chunks"] if c[1] == 1][0]

    def chunk_missing(got):                                       # its rows keep the workspace's NaN fill
        got["c1"][xrow:xrow + rows] = torch.full((rows, op["case"]["N1"]), -1, dtype=torch.int16).view(BF)
    rejects(chunk_missing)

    def chunk_dropped_from_plan(got):
        keep = got["tile1"][:, 1] != xrow
        got["tile1"], got["num_tiles1"] = got["tile1"][keep], int(keep.sum())
    rejects(chunk_dropped_from_plan)

    def counted_twice(got):
        t = int(ps[r]) // 3
        got["out"][t] = (got["out"][t].float() + got["c3"][r].float()).to(BF)
    rejects(counted_twice)

    op8, pl8, good8 = _self_test_case("fp8", "random", 6, 2, 4, 256, 256)
    _check_grouped(op8, good8, pl8)
    experts8 = op8["ids"].reshape(-1).long()[torch.as_tensor(pl8["pair_sorted"])]
    got = dict(good8)
    got["c1"] = good8["c1"].clone()
    a_s = good8["xs_s"].clone()
    a_s[0, 1] = a_s[0, 0]                                         # row 0's second group scaled with the first's scale
    wrong, _ = _expert_gemm(good8["xs"][:1], a_s[:1], op8["w1r"], op8["w1_s"], experts8[:1], True)
    got["c1"][0] = wrong.to(BF)[0]
    with pytest.raises(AssertionError):
        _check_grouped(op8, got, pl8)


# ---------------------------------------------------------------------------------------------------- GPU calls
def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fresh_ws(nbytes):
    """NaN everywhere but the ticket prefix, which must be zero between calls."""
    ws = torch.full((nbytes,), NAN_BYTE, dtype=torch.uint8, device=DEV)
    ws[:TICKET_BYTES].zero_()
    return ws


class FusedCall:
    """chitu_b200_fused_experts on buffers this test owns; x and out sit inside NaN / sentinel padding."""

    def __init__(self, op):
        c = op["case"]
        self.op, self.c = op, c
        self.x = Padded(op["x"])
        self.w1, self.w2 = op["w1"].to(DEV), op["w2"].to(DEV)
        self.w1_s = None if op["w1_s"] is None else op["w1_s"].to(DEV)
        self.w2_s = None if op["w2_s"] is None else op["w2_s"].to(DEV)
        self.ids, self.tw = op["ids"].to(DEV), op["tw"].to(DEV)
        self.res = None if op["res"] is None else Padded(op["res"])
        self.out = Padded(torch.empty(c["T"], c["K1"], dtype=BF), pad=SENTINEL, fill=NAN_BYTE)

    def __call__(self, ws, nbytes=None, T=None):
        from chitu_b200._lib import current_stream, dtype_code, ptr
        c = self.c
        return _lib().chitu_b200_fused_experts(
            ptr(self.x.view), ptr(self.w1), ptr(self.w2), ptr(self.w1_s), ptr(self.w2_s), ptr(self.tw),
            dtype_code(self.tw.dtype), ptr(self.ids), dtype_code(self.ids.dtype), c["T"] if T is None else T, c["topk"],
            c["E"], c["N1"], c["K1"], WCODE[c["wmode"]], ptr(self.out.view),
            None if self.res is None else ptr(self.res.view), ptr(ws), ws.numel() if nbytes is None else nbytes,
            current_stream())

    def run(self, ws):
        from chitu_b200._lib import check
        check(self(ws), f"fused_experts {self.c['wmode']} T={self.c['T']} E={self.c['E']}")
        torch.cuda.synchronize()
        return self.out.view


def _read_ws(ws, c, sms):
    """The intermediates of one call, read back from the workspace."""
    T, topk, E, N1, K1, fp8 = c["T"], c["topk"], c["E"], c["N1"], c["K1"], c["wmode"] == "fp8"
    P, N2 = T * topk, N1 // 2
    path = _moe_path(T, topk, E, N1, K1, c["wmode"], sms)
    lay = _moe_layout(T, topk, E, N1, K1, sms)[path]

    def arr(name, dtype, shape, nbytes=None):
        off = lay[name][0]
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size() if nbytes is None else nbytes
        return ws[off:off + n].view(dtype).view(shape)

    if path == "pair":
        got = dict(c1=arr("c1", BF, (P, N1)), a2=arr("a2", BF, (P, N2)), c3=arr("c3", BF, (P, K1)))
        if fp8:
            got.update(a1_q=arr("a1_q", F8, (T, K1)), a1_s=arr("a1_s", F32, (T, K1 // 128)),
                       a2_q=arr("a2_q", F8, (P, N2)), a2_s=arr("a2_s", F32, (P, N2 // 128)))
        return path, got
    ints = lambda name, n: arr(name, torch.int32, (n,)).cpu().numpy().astype(np.int64)   # noqa: E731
    nt = ints("num_tiles", 2)
    chunks = E + P // 16 + 1
    got = dict(pair_sorted=ints("pair_sorted", P), pos=ints("pos", P), seg_start=ints("seg_start", E + 1),
               w_sorted=arr("w_sorted", F32, (P,)).cpu().numpy(), num_tiles1=int(nt[0]), num_tiles2=int(nt[1]))
    for name, width, n in (("tile1", N1 // 128, int(nt[0])), ("tile2", K1 // 128, int(nt[1]))):
        raw = ints(name, 3 * chunks * width)
        got[name] = np.stack([raw[i * chunks * width:i * chunks * width + n] for i in range(3)], axis=1)
    got["xs"] = arr("xs", F8, (P, K1)) if fp8 else arr("xs", BF, (P, K1))
    got["c1"] = arr("c1", BF, (P, N1))
    got["a2"] = arr("a2", F8, (P, N2)) if fp8 else arr("a2", BF, (P, N2))
    got["c3"] = arr("c3", BF, (P, K1))
    if fp8:
        got["xs_s"] = arr("xs_s", F32, (P, K1 // 128))
        got["a2_s"] = arr("a2_s", F32, (P, N2 // 128))
    return path, got


def _written_slots(ws, BN, sms):
    """(cta, slot) partials a call left in the GEMM scratch (filled with 0xFF before the call)."""
    slots = ws[TICKET_BYTES:TICKET_BYTES + sms * 2 * BN * 128 * 4].view(torch.int32).view(sms, 2, BN * 128)
    return {(int(c), int(s)) for c, s in torch.nonzero(~(slots == -1).all(dim=-1)).tolist()}


def _model_slots(pl, wmode, N1, K1, sms):
    """The partial slots `_grouped_split` says GEMM1 and GEMM2 fill (both launches share the scratch)."""
    out = set()
    for nt, S in ((pl["num_tiles1"], _stages(wmode, K1)), (pl["num_tiles2"], _stages(wmode, N1 // 2))):
        if nt:
            out |= {cs for v in _grouped_split(nt, S, sms)[1].values() for cs in v}
    return out


_WORST = {}


def _run_case(case, sms):
    """One call on a NaN-filled workspace, every stage checked; returns (path, stats)."""
    op = _operands(case)
    c = case
    call = FusedCall(op)
    ws = _fresh_ws(_lib().chitu_b200_moe_workspace_bytes(c["T"], c["topk"], c["E"], c["N1"], c["K1"]))
    out = call.run(ws)
    what = (c["wmode"], c["T"], c["topk"], c["E"], c["N1"], c["K1"])
    assert call.x.pads_intact() and call.out.pads_intact(), ("padding overwritten",) + what
    assert call.res is None or call.res.pads_intact()
    assert bool(torch.isfinite(out).all()), ("non-finite output",) + what
    assert int(ws[:TICKET_BYTES].count_nonzero()) == 0, ("tickets left non-zero",) + what
    path, got = _read_ws(ws, c, sms)
    assert path == _moe_path(c["T"], c["topk"], c["E"], c["N1"], c["K1"], c["wmode"], sms)
    got["out"] = out
    P = c["T"] * c["topk"]
    BN = _chunk_rows(P, c["E"])
    if path == "pair":
        stats = _check_pair(op, got)
        assert bool((ws[TICKET_BYTES:_tc_ws_bytes(sms)] == NAN_BYTE).all()), ("GEMM scratch written",) + what
    else:
        pl = _moe_plan(op["ids"].numpy(), op["tw32"].numpy(), c["E"], BN, c["N1"], c["K1"])
        stats = _check_grouped(op, got, pl)
        assert _written_slots(ws, BN, sms) == _model_slots(pl, c["wmode"], c["N1"], c["K1"], sms), \
            ("partial slots differ from the grouped split model",) + what
    for stage, r in stats.items():
        key = (c["wmode"], path, stage)
        _WORST[key] = max(_WORST.get(key, 0.0), r)
    return path, stats


@pytest.mark.gpu
@pytest.mark.parametrize("wmode", WMODES)
def test_fused_experts_stage_by_stage(wmode):
    """Every case of the table for one weight mode, on the device's SM count: plan arrays exact, gathered / quantised
    activations bit-exact, c1 and c3 inside the bound, a2 within one ulp per rounding, the combine bit-exact, pads and
    tickets intact.  Both paths and, on the grouped path, both plans and every chunk width are reached."""
    sms = _sms()
    seen = set()
    for case in _case_table(sms):
        if case["wmode"] != wmode:
            continue
        path, _ = _run_case(case, sms)
        cells = _case_cells(case, sms)
        assert {c[1] for c in cells} == {path}
        seen |= cells
        if case["cell"] is not None:
            assert cells >= case["cell"]
    assert (wmode, "pair") in seen
    assert {c[2:4] for c in seen if c[1] == "grouped"} == {(bn, pl) for bn in BNS for pl in PLANS}
    for gemm in (1, 2):
        assert {c[5] for c in seen if c[1] == "grouped" and c[4] == gemm} == set(REGIMES)
    for (w, path, stage), r in sorted(_WORST.items()):
        if w == wmode:
            print(f"[moe bound] wmode={w} path={path} stage={stage} max|y-ref|/bound={r:.3f}")


@pytest.mark.gpu
def test_wrapper_cuts_long_batches_into_grouped_calls():
    """fused_experts with more than 8192 // topk tokens: the wrapper makes one C call per 4096 tokens (topk = 2), each on
    the grouped path with the large plan; its output equals the direct C calls on the same slices bit for bit, and each
    of those passes the stage checks."""
    from chitu_b200 import fused_moe
    sms = _sms()
    T, topk, E, N1, K1 = 5196, 2, 8, 256, 128
    base = dict(wmode="fp8", T=T, topk=topk, E=E, N1=N1, K1=K1, routing="random", na=None, ids_dtype=torch.int64,
                tw_dtype=BF, residual=False, seed=4242, cell=None)
    op = _operands(base)
    bounds = [(0, 4096), (4096, T)]
    for t0, t1 in bounds:
        P = (t1 - t0) * topk
        assert P > PLAN_SMALL_MAX and _moe_path(t1 - t0, topk, E, N1, K1, "fp8", sms) == "grouped"
    d = lambda t: t.to(DEV)     # noqa: E731
    got = fused_moe.fused_experts(d(op["x"]), d(op["w1"]), d(op["w2"]), d(op["tw"]), d(op["ids"]), use_fp8_w8a8=True,
                                  w1_scale=d(op["w1_s"]), w2_scale=d(op["w2_s"]), block_shape=[128, 128])
    torch.cuda.synchronize()
    for t0, t1 in bounds:
        part = dict(op)
        part["case"] = dict(base, T=t1 - t0)
        for k in ("x", "ids", "tw", "tw32"):
            part[k] = op[k][t0:t1].contiguous()
        call = FusedCall(part)
        ws = _fresh_ws(_lib().chitu_b200_moe_workspace_bytes(t1 - t0, topk, E, N1, K1))
        out = call.run(ws)
        path, stages = _read_ws(ws, part["case"], sms)
        stages["out"] = out
        pl = _moe_plan(part["ids"].numpy(), part["tw32"].numpy(), E, _chunk_rows((t1 - t0) * topk, E), N1, K1)
        _check_grouped(part, stages, pl)
        assert _same_bits(got[t0:t1], out), (t0, t1)


@pytest.mark.gpu
def test_deterministic_and_one_workspace_for_several_shapes():
    """The same inputs give the same bits twice; three shapes of different P and E alternating on one workspace each
    reproduce their first result, and the tickets end at zero."""
    sms = _sms()
    table = [c for c in _case_table(sms) if c["routing"] == "chunks"]
    picks = [next(c for c in table if any(x[2:4] == key for x in c["cell"]))
             for key in ((16, "small"), (128, "large"), (32, "large"))]
    picks.append(next(c for c in _case_table(sms) if c["cell"] == frozenset({("bf16", "pair")})))
    calls = [FusedCall(_operands(c)) for c in picks]
    nbytes = max(_lib().chitu_b200_moe_workspace_bytes(c["T"], c["topk"], c["E"], c["N1"], c["K1"]) for c in picks)
    ws = _fresh_ws(nbytes)
    first = [call.run(ws).clone() for call in calls]
    assert _same_bits(calls[0].run(ws), first[0])
    for _ in range(2):
        for call, f in zip(calls, first):
            assert _same_bits(call.run(ws), f), (call.c["wmode"], call.c["T"], call.c["E"])
    assert int(ws[:TICKET_BYTES].count_nonzero()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("wmode", WMODES)
def test_graph_replay_follows_new_routing(wmode):
    """Capture with routing A, overwrite the id and weight buffers with routing B (other experts, other chunk count),
    replay: the output equals an eager call with routing B bit for bit.  The plan runs on the device."""
    sms = _sms()
    base = dict(wmode=wmode, T=40, topk=3, E=8, N1=256, K1=256, routing="shared", na=None, ids_dtype=torch.int32,
                tw_dtype=F32, residual=True, seed=9)
    op = _operands(base)
    call = FusedCall(op)
    ws = _fresh_ws(_lib().chitu_b200_moe_workspace_bytes(40, 3, 8, 256, 256))
    routings = [_routing(dict(base, routing="random", seed=10)), _routing(dict(base, routing="chunks", na=3, seed=11)),
                _routing(dict(base, routing="absent"))]
    eager = []
    for ids, w in routings:
        call.ids.copy_(torch.from_numpy(ids).to(torch.int32))
        call.tw.copy_(torch.from_numpy(w))
        eager.append(call.run(ws).clone())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call(ws)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(ws)
    for (ids, w), want in zip(routings, eager):
        call.ids.copy_(torch.from_numpy(ids).to(torch.int32))
        call.tw.copy_(torch.from_numpy(w))
        call.out.view.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert _same_bits(call.out.view, want), wmode
    assert int(ws[:TICKET_BYTES].count_nonzero()) == 0


def _last_error():
    return _lib().chitu_b200_last_error().decode(errors="replace")


@pytest.mark.gpu
def test_refusals_launch_nothing():
    """P > 65535, a workspace one byte short, and shapes the weight modes cannot take return a status, launch nothing
    and leave the workspace and the output alone."""
    from chitu_b200._lib import launch_count
    base = dict(wmode="bf16", T=6, topk=2, E=4, N1=256, K1=256, routing="random", na=None, ids_dtype=torch.int32,
                tw_dtype=BF, residual=False, seed=3)
    lib = _lib()
    before = launch_count()
    refusals = []
    for over in (dict(T=16385, topk=4, K1=128), dict(), dict(wmode="fp8", K1=192), dict(wmode="fp8", N1=384),
                 dict(N1=40), dict(K1=200), dict(wmode="soft", N1=40)):
        case = dict(base, **over)
        op = _operands(case)
        call = FusedCall(op)
        need = lib.chitu_b200_moe_workspace_bytes(case["T"], case["topk"], case["E"], case["N1"], case["K1"])
        short = not over
        ws = _fresh_ws(need)
        rc = call(ws, need - 1 if short else need)
        torch.cuda.synchronize()
        assert rc != 0 and _last_error(), over
        assert int(ws[:TICKET_BYTES].count_nonzero()) == 0 and bool((ws[TICKET_BYTES:] == NAN_BYTE).all()), over
        assert bool((call.out.view.view(torch.int16) == -1).all()), over
        refusals.append(over)
    assert launch_count() == before
    zero = FusedCall(_operands(base))
    ws = _fresh_ws(lib.chitu_b200_moe_workspace_bytes(6, 2, 4, 256, 256))
    assert zero(ws, T=0) == 0 and launch_count() == before               # T = 0: nothing to do


# ----------------------------------------------------------------------------------------------------- moe_gate
SCORE_CODE = {"sigmoid": 1, "softmax": 0, "softmax_renorm": 2}
# (score, bias, E, n_groups, topk_groups, topk); "neg": every score + bias < 0, so masked zeros beat kept scores
GATE_CONFIGS = (
    ("sigmoid", "f32", 256, 8, 4, 8),         # DeepSeek-V3
    ("sigmoid", "bf16", 256, 8, 4, 8),
    ("sigmoid", None, 64, 8, 2, 2),
    ("sigmoid", "bf16_neg", 64, 8, 3, 8),
    ("sigmoid", "f32_neg", 384, 48, 6, 32),   # generic top-k, > 32 groups
    ("sigmoid", "f32", 384, 48, 8, 8),
    ("sigmoid", "f32", 8, 1, 1, 1),
    ("softmax", None, 8, 1, 1, 2),
    ("softmax", "bf16", 64, 8, 4, 8),         # fp32 scores + bf16 bias is an fp32 add
    ("softmax", "f32", 256, 8, 4, 8),
    ("softmax", "bf16", 384, 48, 8, 32),
    ("softmax", "bf16_neg", 256, 8, 2, 32),
    ("softmax", None, 384, 1, 1, 1),
    ("softmax_renorm", None, 8, 1, 1, 2),     # Mixtral
    ("softmax_renorm", None, 64, 1, 1, 8),
    ("softmax_renorm", None, 384, 1, 1, 1),
)


def _gate_inputs(T, dim, E, bias, seed, exact=False):
    """x, W (bf16) and the bias.  exact: dyadic values whose fp32 dot products are exact in any summation order, so
    every logits path gives the same bf16 logits."""
    g = torch.Generator().manual_seed(seed)
    if exact:
        x = (torch.randint(-4, 5, (T, dim), generator=g) / 4.0).to(BF)
        w = (torch.randint(-8, 9, (E, dim), generator=g) / 128.0).to(BF)     # |dot| < 2^9 in steps of 2^-9
    else:
        x = torch.randn(T, dim, generator=g).to(BF)
        w = (torch.randn(E, dim, generator=g) / math.sqrt(dim)).to(BF)
    b = None
    if bias is not None:
        b = torch.randn(E, generator=g) * 0.05 - (2.0 if bias.endswith("neg") else 0.0)
        b = b.to(BF) if bias.startswith("bf16") else b.float()
    return x, w, b


def _gate_scores(logits, bias, n_groups, mode):
    """GateDeepSeekV3.forward after the linear, in the reference's dtypes: (original scores, scores + bias, group
    scores or None)."""
    if mode == "sigmoid":
        scores = logits.sigmoid()
    else:
        scores = logits.softmax(dim=-1, dtype=torch.float32)
    orig = scores
    if bias is not None:
        scores = scores + bias
    gsc = None
    if n_groups > 1:
        s3 = scores.view(scores.shape[0], n_groups, -1)
        gsc = s3.amax(dim=-1) if bias is None else s3.topk(2, dim=-1)[0].sum(dim=-1)
    return orig, scores, gsc


def _ulp(v, dtype):
    m = 7 if dtype == BF else 23
    a = v.double().abs()
    e = torch.floor(torch.log2(torch.where(a > 0, a, torch.ones_like(a))))
    return torch.where(a > 0, torch.exp2(e - m), torch.zeros_like(a))


def _tol(v, mode):
    """A near tie: one ulp of the score dtype (bf16 for sigmoid scores, whose bf16 sigmoid may differ by one ulp from
    the kernel's; four fp32 ulps for softmax, whose exp and sum order are not the reference's)."""
    return _ulp(v, BF) if mode == "sigmoid" else 4 * _ulp(v, F32)


def _selection_ok(scores_t, gsc_t, idx, n_groups, topk_groups, topk, mode):
    """None when idx is the reference's selection up to exact ties; "tie" / "near" when it differs from it only by an
    exact tie / a near tie at a boundary (the selected scores equal the reference's top-k values within the tie
    tolerance, under the reference's group choice or one that differs from it by a near tie); False otherwise.  Exact
    ties must go to the lowest index: no unselected expert below a selected one has its score, and equal scores are
    picked in index order."""
    E = scores_t.numel()
    gs = E // n_groups
    masks = [None]
    if n_groups > 1:
        order = torch.argsort(gsc_t.double(), descending=True, stable=True)
        vals = gsc_t[order].double()
        bound = vals[topk_groups - 1]
        tol = float(_tol(bound, mode))
        sure = [int(g) for g, v in zip(order, vals) if v > bound + tol]
        tied = [int(g) for g, v in zip(order, vals) if abs(float(v - bound)) <= tol]
        masks = [sure + list(c) for c in itertools.combinations(tied, topk_groups - len(sure))]
        masks.sort(key=lambda m: set(m) != set(order[:topk_groups].tolist()))   # the reference's choice first
    kind = False
    for mi, m in enumerate(masks):
        s = scores_t.clone()
        if m is not None:
            keep = torch.zeros(n_groups, dtype=torch.bool, device=s.device)
            keep[m] = True
            s = s * keep.repeat_interleave(gs).to(s.dtype)
        top = torch.topk(s.double(), topk)[0]
        mine = s.double()[idx]
        if len(set(idx.tolist())) != topk or bool((mine[1:] > mine[:-1]).any()):
            return False
        diff = (mine - top).abs()
        if bool((diff == 0).all()):
            sel = torch.zeros(E, dtype=torch.bool, device=s.device)
            sel[idx] = True
            below = torch.arange(E, device=s.device)[None, :] < idx[:, None]
            if bool(((s.double()[None, :] == mine[:, None]) & below & ~sel[None, :]).any()):
                return False                            # a tie that did not go to the lowest index
            if bool(((mine[1:] == mine[:-1]) & (idx[1:] < idx[:-1])).any()):
                return False
            exact = mi == 0 and torch.equal(idx, torch.topk(s.double(), topk)[1])
            return None if exact else "tie"
        if bool((diff <= _tol(top, mode)).all()):
            kind = "near"
    return kind


def _gate_weights_ref(orig_t, idx, mode, route_scale):
    """The reference's weights of the kernel's selection."""
    wv = orig_t[idx][None]
    if mode in ("sigmoid", "softmax_renorm"):          # bf16 / fp32 renormalisation: the dtype is orig's
        wv = wv / wv.sum(dim=-1, keepdim=True)
    return (wv * route_scale).to(BF)[0]


class GateCall:
    def __init__(self, x, w, bias, E, n_groups, topk_groups, topk, mode, route_scale):
        self.x, self.w = x.to(DEV), w.to(DEV)
        self.bias = None if bias is None else bias.to(DEV)
        self.args = (E, n_groups, topk_groups, topk, mode, route_scale)
        T = x.shape[0]
        self.out_w = torch.full((T, topk), float("nan"), dtype=BF, device=DEV)
        self.out_i = torch.full((T, topk), -7, dtype=torch.int64, device=DEV)

    def run(self, ws):
        from chitu_b200._lib import check, current_stream, dtype_code, ptr
        E, G, TG, topk, mode, rs = self.args
        T, dim = self.x.shape
        check(_lib().chitu_b200_moe_gate(
            ptr(self.x), ptr(self.w), ptr(self.bias), dtype_code(self.bias.dtype) if self.bias is not None else 0, T,
            dim, E, G, TG, topk, SCORE_CODE[mode], float(rs), ptr(self.out_w), ptr(self.out_i), topk, ptr(ws),
            0 if ws is None else ws.numel(), current_stream()), "moe_gate")
        torch.cuda.synchronize()


_GATE_EXCUSED = {"tie": 0, "near": 0}


def _check_gate(call, logits, what):
    """Routing of the kernel against the reference's routing of `logits` (bf16, [T, E]); weights within one bf16 ulp
    of the reference's weights of the kernel's selection."""
    E, G, TG, topk, mode, rs = call.args
    orig, scores, gsc = _gate_scores(logits, call.bias, G, mode)
    idx_all, w_all = call.out_i, call.out_w
    for t in range(logits.shape[0]):
        idx = idx_all[t]
        assert bool(((idx >= 0) & (idx < E)).all()), ("index out of range",) + what
        kind = _selection_ok(scores[t], None if gsc is None else gsc[t], idx, G, TG, topk, mode)
        assert kind is not False, ("selection differs", t, idx.tolist()) + what
        if kind:
            _GATE_EXCUSED[kind] += 1
        want = _gate_weights_ref(orig[t], idx, mode, rs)
        err = (w_all[t].double() - want.double()).abs()
        assert bool((err <= _ulp(want, BF)).all()), ("weights", t, w_all[t].tolist(), want.tolist()) + what


def _gate_ws(T, E):
    ws = torch.full((_lib().chitu_b200_moe_gate_workspace_bytes(T, E),), NAN_BYTE, dtype=torch.uint8, device=DEV)
    ws[:TICKET_BYTES].zero_()
    return ws


def _gate_logits_path(T, dim):
    return "gemv" if T <= 16 and dim <= 8192 else "tc"


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [7168, 8192, 8200])
def test_gate_logits_in_the_workspace(dim):
    """The logits the gate leaves in its workspace ([GEMM scratch | logits]) against an fp64 dot inside the bound, for
    every token bucket of gate_logits_kernel (1, 4, 8, 16) and the wgmma linear (T > 16 or dim > 8192); then the routing
    of those logits."""
    sms = _sms()
    E = 256
    worst = {}
    for T in (1, 3, 4, 5, 8, 9, 16, 17, 200):
        x, w, b = _gate_inputs(T, dim, E, "f32", seed=T * 31 + dim)
        call = GateCall(x, w, b, E, 8, 4, 8, "sigmoid", 2.5)
        ws = _gate_ws(T, E)
        call.run(ws)
        bn = 16 if T <= 16 else 32 if T <= 32 else 64 if T <= 64 else 128
        off = _align256(TICKET_BYTES + sms * 2 * bn * 128 * 4)
        logits = ws[off:off + T * E * 2].view(BF).view(T, E)
        a64, w64 = call.x.double(), call.w.double()
        ref, rss = a64 @ w64.T, ((a64 * a64) @ (w64 * w64).T).sqrt()
        path = _gate_logits_path(T, dim)
        r = _ratio(logits, ref, rss, U_BF16, TAU_FP32)
        assert r <= 1.0, ("logits outside the bound", r, T, dim, path)
        worst[path] = max(worst.get(path, 0.0), r)
        assert int(ws[:TICKET_BYTES].count_nonzero()) == 0, (T, dim)
        _check_gate(call, logits, (T, dim, path))
    assert set(worst) == ({"gemv", "tc"} if dim <= 8192 else {"tc"})
    for path, r in sorted(worst.items()):
        print(f"[gate bound] dim={dim} logits={path} max|y-ref|/bound={r:.3f}")
    print(f"[gate] excused selections so far: {_GATE_EXCUSED}")


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", GATE_CONFIGS, ids=lambda c: "-".join(map(str, c)))
def test_gate_routing(cfg):
    """Every score mode, bias dtype (and a bias that makes every kept score negative), E on both sides of the register
    top-k, n_groups on both sides of 32, topk up to 32, through both logits kernels, the wgmma logits and the in-kernel
    GEMV (no workspace).  Inputs with exact dot products make all four paths' logits the bf16 rounding of the exact dot,
    so each is checked against the reference routing of the same logits."""
    mode, bias, E, G, TG, topk = cfg
    for T, dim, ws_kind in ((1, 1024, "ws"), (9, 1024, "ws"), (40, 1024, "ws"), (9, 1024, None), (3, 7168, None)):
        x, w, b = _gate_inputs(T, dim, E, bias, seed=GATE_CONFIGS.index(cfg) * 100 + T, exact=True)
        call = GateCall(x, w, b, E, G, TG, topk, mode, 1.0 if mode != "sigmoid" else 2.5)
        logits = (call.x.double() @ call.w.double().T).to(BF)       # the exact dot, rounded once
        ws = _gate_ws(T, E) if ws_kind else None
        call.run(ws)
        _check_gate(call, logits, (cfg, T, dim, ws_kind))
    print(f"[gate] {cfg}: excused selections so far: {_GATE_EXCUSED}")


# ------------------------------------------------------------------------------------- the stand-alone grouped GEMM
@pytest.mark.gpu
@pytest.mark.parametrize("wmode", WMODES)
@pytest.mark.parametrize("block_m", [16, 32, 64, 128])
def test_grouped_gemm_entry(wmode, block_m):
    """chitu_b200_moe_grouped_gemm on moe_align_block_size's blocks with expert_map-style absent experts (their rows
    exactly zero), padding entries, routed weight on / off in bf16 and fp32, top_k 1 and > 1: every valid row inside the
    bound, C's padding intact, tickets back at zero."""
    from chitu_b200._lib import check, current_stream, dtype_code, ptr
    lib = _lib()
    T, topk, E, N, K = 9, 3, 6, 256, 256
    worst = 0.0
    for top_k, mul, twt, seed in ((topk, False, BF, 1), (1, True, BF, 2), (1, True, F32, 3), (topk, True, F32, 4)):
        g = torch.Generator().manual_seed(seed * 100 + block_m)
        ids = torch.randint(0, E, (T, topk), generator=g)
        ids[0, 1] = ids[0, 0]                                  # a duplicate within a token
        tw = (torch.rand(T, topk, generator=g) * 0.75 + 0.25).to(twt)
        P = T * topk
        A = torch.randn(T if top_k > 1 else P, K, generator=g).to(BF)
        if wmode == "bf16":
            Bw, Bs = (torch.randn(E, N, K, generator=g) * 0.05).to(BF), None
            Br = Bw
        else:
            Bw, Bs = _fp8_stack(E, N, K, g)
            Br = Bw if wmode == "fp8" else O.weight_dequant_soft_fp8(Bw, Bs)
        sorted_ids, expert_ids, npp, _ = O.moe_align_block_size(ids.numpy(), block_m, E)
        emap = np.arange(E)
        emap[[1, 4]] = -1                                      # experts 1 and 4 live on another rank
        expert_ids = emap[expert_ids].astype(np.int32)
        EM = sorted_ids.size
        C = Padded(torch.empty(P, N, dtype=BF), pad=SENTINEL, fill=NAN_BYTE)
        ws = _fresh_ws(lib.chitu_b200_moe_grouped_gemm_workspace_bytes(EM, N, K))
        Ad, Bd = A.to(DEV), Bw.to(DEV)
        Bsd, twd = None if Bs is None else Bs.to(DEV), tw.to(DEV)
        sd, ed, nd = (torch.from_numpy(v).to(DEV) for v in (sorted_ids, expert_ids, npp))
        check(lib.chitu_b200_moe_grouped_gemm(ptr(Ad), ptr(Bd), ptr(C.view), ptr(Bsd), ptr(twd), dtype_code(twt),
                                              ptr(sd), ptr(ed), ptr(nd), EM, P, int(mul), top_k, block_m, E, N, K,
                                              WCODE[wmode], ptr(ws), ws.numel(), current_stream()), "grouped gemm")
        torch.cuda.synchronize()
        what = (wmode, block_m, top_k, mul, str(twt))
        assert C.pads_intact(), what
        assert int(ws[:TICKET_BYTES].count_nonzero()) == 0, what
        flat = ids.reshape(-1)
        absent = torch.from_numpy(emap)[flat] < 0
        got = C.view.cpu()
        assert bool((_bits(got[absent]) == 0).all()), ("absent rows not zero",) + what
        vi = torch.nonzero(~absent).flatten()
        rows = A[vi // top_k]
        if wmode == "fp8":
            a, a_s = _quant(rows)
        else:
            a, a_s = rows, None
        ref, rss = _expert_gemm(a.to(DEV), None if a_s is None else a_s.to(DEV), Br, Bs, flat[vi].to(DEV),
                                wmode == "fp8", scale=tw.float().reshape(-1)[vi] if mul else None)
        r = _ratio(got[vi].to(DEV), ref, rss, U_BF16, TAU_FP8_MMA if wmode == "fp8" else TAU_FP32)
        assert r <= 1.0, ("outside the bound", r) + what
        worst = max(worst, r)
    print(f"[moe_grouped_gemm bound] wmode={wmode} block_m={block_m} max|y-ref|/bound={worst:.3f}")


@pytest.mark.gpu
def test_grouped_gemm_refuses_a_k_tail():
    """The row gather works in whole 128-column groups, so K % 128 != 0 is refused with a status and no launch (before,
    16-bit weights were accepted at K % 16 == 0 and the tail columns of every gathered row were never written)."""
    from chitu_b200._lib import current_stream, dtype_code, launch_count, ptr
    lib = _lib()
    T, topk, E, N, K, block_m = 4, 2, 3, 128, 192, 16
    ids = np.array([[0, 1], [2, 0], [1, 1], [2, 2]])
    sorted_ids, expert_ids, npp, _ = O.moe_align_block_size(ids, block_m, E)
    A = torch.randn(T, K, device=DEV).to(BF)
    B = torch.randn(E, N, K, device=DEV).to(BF)
    C = torch.full((T * topk, N), float("nan"), dtype=BF, device=DEV)
    tw = torch.ones(T, topk, dtype=BF, device=DEV)
    sd, ed, nd = (torch.from_numpy(v).to(DEV) for v in (sorted_ids, expert_ids, npp))
    EM = sorted_ids.size
    ws = _fresh_ws(lib.chitu_b200_moe_grouped_gemm_workspace_bytes(EM, N, K))
    before = launch_count()
    rc = lib.chitu_b200_moe_grouped_gemm(ptr(A), ptr(B), ptr(C), None, ptr(tw), dtype_code(BF), ptr(sd), ptr(ed), ptr(nd),
                                         EM, T * topk, 0, topk, block_m, E, N, K, 0, ptr(ws), ws.numel(), current_stream())
    torch.cuda.synchronize()
    assert rc != 0 and _last_error() and launch_count() == before
    assert bool(torch.isnan(C).all())
