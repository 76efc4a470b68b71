"""Multi-token attention against an fp64 reference, on shapes chosen by a restatement of the host code that splits the
keys: GQA with seqlen_q > 1 through `chitu_b200_gqa_paged_prefill` (`gqa_prefill_kernel`),
`chitu_b200_gqa_contiguous_attn` (`gqa_prefill_contig_kernel`) and `chitu_b200_gqa_paged_attn_fp8kv`
(`gqa_prefill_e4m3_kernel`), all three the CTA `gqa_prefill_cta` (csrc/gqa_prefill.cu); absorbed MLA through
`chitu_b200_mla_paged_prefill` (`mla_paged_prefill_kernel`) and the varlen `chitu_b200_mla_prefill`
(`mla_prefill_kernel`), both the CTA `mla_prefill_cta` (csrc/mla_prefill.cu).

The host model restates `prefill_splits` (the decode kernels' wave rule over row tiles x kv heads x requests at two
CTAs per SM for GQA, over row tiles x requests at one for MLA, then `splits_that_fit` over B * sq * Hq partial rows; no
workspace: one split), the max_len each entry derives from its hint, and the key range of every (row, split): row r of
a request is token r / G, head r % G, it sees keys [0, lim(r)) (bottom-right causal), its 64-row tile has
ntiles = ceil(lim(last row) / 64) key tiles, and split s takes tiles [min(ntiles, s * per), min(ntiles, (s + 1) * per))
with per = ceil(ntiles / S), i.e. keys [64 t_begin, min(64 t_end, lim(r))).  Low row tiles under a causal mask, and hints
far above the real lengths, leave trailing splits empty.  Like the decode file it assumes 132 SMs.

The case table holds one case per (entry, dtype, G, split regime), (MLA H, split regime) and (MLA varlen H, causal)
cell.  The GPU tests run it on NaN-poisoned caches with a NaN trap page behind every unused block-table column, padded
operands and a 0xFF workspace, and check the cache, the split count, the launches, every split partial and LSE against
its key range, the output, and the pads; the bound and its injected-error self-test are those of
test_attn_decode_dispatch_gpu.py, with a per-row causal limit."""
import functools
import math

import pytest
import torch

from test_attn_decode_dispatch_gpu import (BF, DEV, F8, F16, MLA_C, MLA_R, MLA_SCALE, NAN_BYTE, SENTINEL, SMS,
                                           U_OUT, U_P, Padded, _bits, _block_table, _cdiv, _keys, _needle, _report,
                                           _shape_keys, _split_checks, _weights_out, bound, pick_splits_waves, ratio,
                                           ref_splits, split_kv_bytes, splits_that_fit)

# ---------------------------------------------------------------------------------------------- host model
ROWS = 64                  # query rows (token, head) per CTA of both kernels
TILE = 64                  # keys per tile
D = 128                    # GQA head dim
MLA_ROW = MLA_C + MLA_R
GQA_CTAS_PER_SM = 2        # gqa_prefill.cu kCtasPerSm; the MLA CTA takes a whole SM
MAX_SPLITS = 128           # _lib.ATTN_MAX_SPLITS
ATTN_CAP = 256 << 20       # workspace.attn_bytes' default cap


def lim(r, G, Lk, sq, causal):
    """Keys visible to row r (token r / G) of a request with Lk keys and sq query tokens."""
    return max(0, min(Lk, r // G + 1 + Lk - sq)) if causal else max(Lk, 0)


def tile_split(r0, nrows, G, Lk, sq, causal, S):
    """(ntiles, per): the key tiles of the row tile starting at row r0 and the tiles per split."""
    rlast = min(r0 + ROWS, nrows) - 1
    ntiles = _cdiv(lim(rlast, G, Lk, sq, causal), TILE)
    return ntiles, _cdiv(ntiles, S)


def key_ranges(r, G, nrows, Lk, sq, causal, S):
    """[(lo, hi)] of the S splits of row r: keys [64 t_begin, min(64 t_end, lim(r))), empty when hi <= lo."""
    ntiles, per = tile_split(r - r % ROWS, nrows, G, Lk, sq, causal, S)
    L = lim(r, G, Lk, sq, causal)
    out = []
    for s in range(S):
        tb = min(ntiles, s * per)
        te = min(ntiles, tb + per)
        out.append((min(TILE * tb, L), min(TILE * te, L)))
    return out


def prefill_splits(kind, B, sq, Hq, Hkv, max_len, ws_bytes):
    """(splits, picked): prefill_splits of gqa_prefill.cu / the split count of chitu_b200_mla_paged_prefill, and the
    count the wave rule picked before the workspace was consulted.  ws_bytes None: no workspace, one split."""
    if kind == "mla":
        picked = pick_splits_waves(_cdiv(sq * Hq, ROWS) * B, max_len, SMS)
        dv = MLA_C
    else:
        picked = pick_splits_waves(_cdiv(sq * (Hq // Hkv), ROWS) * Hkv * B, max_len, SMS * GQA_CTAS_PER_SM)
        dv = D
    return (splits_that_fit(picked, B * sq * Hq, dv, ws_bytes) if ws_bytes is not None else 1), picked


def entry_max_len(hint_arg, span):
    """max_len of an entry: the hint when positive, else the cache span (bt_stride * page paged, cache_rows contiguous)."""
    return hint_arg if hint_arg > 0 else span


def backend_attn_bytes(B, heads, dv, cap=ATTN_CAP):
    """workspace.attn_bytes: the partials of the largest split count, halving from 128, that fit `cap`, plus the plan."""
    s = MAX_SPLITS
    while s > 1 and split_kv_bytes(B * heads, dv, s) > cap:
        s //= 2
    return split_kv_bytes(B * heads, dv, s)


def backend_ws_bytes(B, heads, dv):
    """The size of the buffer workspace.get hands a fresh process for attn_bytes(B, heads, dv)."""
    from chitu_b200.workspace import _round_up_pow2
    return _round_up_pow2(backend_attn_bytes(B, heads, dv))


# ---------------------------------------------------------------------------------------------- case table
GS = (1, 2, 4, 8)
REGIMES = ("1", "2-7", "8-15", "16-64", "lowered", "none")
DTYPES = (BF, F16)
ENTRIES = ("paged", "contig", "fp8")
PAGED_PAGES = (64, 128, 192, 256, 320, 1024)
FP8_PAGES = (64, 128, 256, 1024)
HINTS = ("exact", "below", "above", "zero")
SQ_KINDS = ("under", "full", "over")          # sq * G < 64, = 64, > 64 with a partial last row tile


def _regime(S):
    return "1" if S == 1 else "2-7" if S < 8 else "8-15" if S < 16 else "16-64"


def _sq(kind, G):
    return {"under": 3, "full": ROWS // G, "over": ROWS // G + 3}[kind]


def _prefill_lens(B, L_max, sq, new, seed):
    """Cached lengths of a ragged batch: the longest request has L_max keys with its new rows; the others are a third of
    it, one key, 63 and so on; without new rows the second is sq / 2 (causal: leading rows that see nothing) and a third
    is empty."""
    first = max(L_max - (sq if new else 0), 0)
    extra = [L_max // 3, 1, 63, 2 * L_max // 3 + 5]
    lens = [first] + [min(extra[(k + seed) % len(extra)], first) for k in range(B - 1)]
    if not new and B > 1:
        lens[1] = sq // 2
    if not new and B > 2:
        lens[-1] = 0
    return lens


def _batch_ok(B, new, i):
    """Without new rows a batch has the blind request, and every fourth such case the empty one too."""
    return new or B >= (3 if i % 4 == 0 else 2)


def _hint(hint, Lks, span):
    """(max_seqlen_hint argument, the max_len the entry derives from it)."""
    if hint == "zero":
        return 0, span
    m = max(Lks)
    v = {"exact": m, "below": max(m // 3, 1), "above": 4 * m}[hint]
    return v, entry_max_len(v, span)


def make_gqa_case(entry, dtype, G, B, Hkv, sq, lens, new, causal, page, hint, ws, seed):
    """A GQA case; ws is the workspace size in bytes or None."""
    Lks = [L + (sq if new else 0) for L in lens]
    c = dict(kind="gqa", entry=entry, dtype=dtype, G=G, B=B, Hkv=Hkv, Hq=G * Hkv, sq=sq, lens=lens, Lks=Lks, new=new,
             causal=causal, page=page, hint=hint, ws=ws, seed=seed)
    if entry == "contig":
        c["rows"] = max(Lks) + 3
        span = c["rows"]
    else:
        c["npages"] = [_cdiv(L, page) for L in Lks]
        c["bt_stride"] = max(c["npages"]) + 1            # _block_table: one trap column past the longest request
        span = c["bt_stride"] * page
    c["hint_arg"], c["max_len"] = _hint(hint, Lks, span)
    c["splits"], c["picked"] = prefill_splits("gqa", B, sq, G * Hkv, Hkv, c["max_len"], ws)
    return c


def _gqa_cell_case(entry, dtype, G, regime, i, B, Hkv, L_max, hint, sq):
    new, causal = i % 3 != 0, i % 2 == 0
    if not _batch_ok(B, new, i):
        return None
    pages = FP8_PAGES if entry == "fp8" else PAGED_PAGES
    page = None if entry == "contig" else pages[i % len(pages)]
    lens = _prefill_lens(B, L_max, sq, new, i)
    Hq = G * Hkv
    if regime == "none":
        c = make_gqa_case(entry, dtype, G, B, Hkv, sq, lens, new, causal, page, hint, None, i)
        return c if c["picked"] >= 2 else None
    if regime == "lowered":               # the workspace the backend sizes for B * Hq rows
        c = make_gqa_case(entry, dtype, G, B, Hkv, sq, lens, new, causal, page, hint, backend_ws_bytes(B, Hq, D), i)
        return c if c["splits"] < c["picked"] else None
    c = make_gqa_case(entry, dtype, G, B, Hkv, sq, lens, new, causal, page, hint, split_kv_bytes(B * sq * Hq, D, 64), i)
    return c if _regime(c["splits"]) == regime else None


@functools.lru_cache(maxsize=None)
def gqa_case_table():
    """One case per (entry, dtype, G, regime): the cheapest batch / length / hint that lands in the cell, with sq * G
    under, at or over one row tile by rotation (the lowered cells search sq: only a long query outgrows the backend's
    workspace)."""
    cases = []
    i = 0
    for entry in ENTRIES:
        for dtype in DTYPES:
            for G in GS:
                for regime in REGIMES:
                    i += 1
                    sqs = ((16, 24, 40, 64) if regime == "lowered" else (_sq(SQ_KINDS[i % len(SQ_KINDS)], G),))
                    best = None
                    for sq in sqs:
                        for B in (1, 2, 3):
                            for Hkv in (1, 2):
                                for L_max in (40, 128, 300, 640, 1500, 3000, 6400):
                                    for hint in HINTS[(i % 4):] + HINTS[:(i % 4)]:
                                        c = _gqa_cell_case(entry, dtype, G, regime, i, B, Hkv, L_max, hint, sq)
                                        if c is None:
                                            continue
                                        c["regime"] = regime
                                        cost = B * Hkv * G * sq * (max(c["Lks"]) + TILE) * (c["splits"] + 4)
                                        if best is None or cost < best[0]:
                                            best = (cost, c)
                    if best is not None:
                        cases.append(best[1])
    return tuple(cases)


MLA_HS = (8, 16, 24, 32, 128)
MLA_REGIMES = ("1", "rem", "many")


def _mla_regime(S):
    return "1" if S == 1 else "many" if S >= 32 else "rem" if S % 8 else "mult8"


def make_mla_case(H, B, sq, lens, new, causal, hint, ws, seed):
    Lks = [L + (sq if new else 0) for L in lens]
    c = dict(kind="mla", H=H, G=H, Hkv=1, Hq=H, B=B, sq=sq, lens=lens, Lks=Lks, new=new, causal=causal, page=TILE,
             hint=hint, ws=ws, seed=seed, dtype=BF)
    c["npages"] = [_cdiv(L, TILE) for L in Lks]
    c["bt_stride"] = max(c["npages"]) + 1
    c["hint_arg"], c["max_len"] = _hint(hint, Lks, c["bt_stride"] * TILE)
    c["splits"], c["picked"] = prefill_splits("mla", B, sq, H, 1, c["max_len"], ws)
    return c


@functools.lru_cache(maxsize=None)
def mla_case_table():
    """One case per (H, regime): one split, a count with a remainder mod 8 (the merge's loops), 32 or more; sq by
    rotation (searched for the many-split cells, which need few row tiles)."""
    cases = []
    i = 0
    for H in MLA_HS:
        for regime in MLA_REGIMES:
            i += 1
            new, causal = i % 3 != 2, i % 2 == 1
            best = None
            for sq in ((2, 3, 4, 7) if regime == "many" else ((3, 2, 7, 4)[i % 4],)):
                for B in (1, 2, 3):
                    for L_max in (40, 130, 300, 1000, 3000, 9000):
                        for hint in HINTS[(i % 4):] + HINTS[:(i % 4)]:
                            if not _batch_ok(B, new, i):
                                continue
                            lens = _prefill_lens(B, L_max, sq, new, i)
                            c = make_mla_case(H, B, sq, lens, new, causal, hint, split_kv_bytes(B * sq * H, MLA_C, 64), i)
                            if _mla_regime(c["splits"]) != regime:
                                continue
                            c["regime"] = regime
                            cost = B * sq * H * (max(c["Lks"]) + TILE) * (c["splits"] + 4)
                            if best is None or cost < best[0]:
                                best = (cost, c)
            if best is not None:
                cases.append(best[1])
    return tuple(cases)


VARLEN_HS = (1, 8, 16, 24, 128)
# (Lq, Lk) per sequence: no query, no key, Lk > Lq (a chunk on a prefix), Lq > Lk (causal: leading rows see nothing),
# a whole tile, a single token, and lengths off the tile edges
VARLEN_SEQS = ((0, 37), (19, 0), (70, 200), (90, 40), (64, 64), (1, 1), (33, 130))
VARLEN_SEQS_WIDE = ((0, 37), (9, 0), (20, 150), (30, 12), (1, 1))       # H = 128: 64 % H == 0 and few rows


@functools.lru_cache(maxsize=None)
def varlen_case_table():
    cases = []
    for i, H in enumerate(VARLEN_HS):
        for causal in (True, False):
            seqs = VARLEN_SEQS_WIDE if H >= 64 else VARLEN_SEQS
            rot = (i + causal) % len(seqs)
            seqs = seqs[rot:] + seqs[:rot]
            cases.append(dict(kind="varlen", H=H, G=H, Hkv=1, causal=causal, lens_q=[s[0] for s in seqs],
                              lens_k=[s[1] for s in seqs], shared_v=(i + causal) % 2 == 0, seed=100 + 2 * i + causal,
                              dtype=BF))
    return tuple(cases)


def _has_empty_split(c):
    """A row tile of the case whose last split (at least) takes no key tile."""
    G, sq, S = c["G"], c["sq"], c["splits"]
    for Lk in c["Lks"]:
        for r0 in range(0, sq * G, ROWS):
            ntiles, per = tile_split(r0, sq * G, G, Lk, sq, c["causal"], S)
            if S > 1 and min(ntiles, (S - 1) * per) >= ntiles:
                return True
    return False


def _more_splits_than_tiles(c):
    G, sq = c["G"], c["sq"]
    return any(c["splits"] > tile_split(r0, sq * G, G, Lk, sq, c["causal"], c["splits"])[0] > 0
               for Lk in c["Lks"] for r0 in range(0, sq * G, ROWS))


def test_case_table_covers_every_cell():
    """Every (entry, dtype, G, split regime), (MLA H, split regime) and (varlen H, causal) cell has a case, and the
    table as a whole reaches every axis the kernels branch on."""
    gqa = gqa_case_table()
    assert {(c["entry"], c["dtype"], c["G"], c["regime"]) for c in gqa} == {
        (e, dt, G, r) for e in ENTRIES for dt in DTYPES for G in GS for r in REGIMES}
    for c in gqa:
        S, picked = prefill_splits("gqa", c["B"], c["sq"], c["Hq"], c["Hkv"], c["max_len"], c["ws"])
        assert S == c["splits"] and (c["ws"] is None) == (c["regime"] == "none") and S <= 64
        if c["regime"] == "lowered":
            assert S < picked and c["ws"] == backend_ws_bytes(c["B"], c["Hq"], D)
    mla = mla_case_table()
    assert {(c["H"], c["regime"]) for c in mla} == {(H, r) for H in MLA_HS for r in MLA_REGIMES}
    assert {c["splits"] % 8 for c in mla if c["regime"] == "rem"} - {0}
    varlen = varlen_case_table()
    assert {(c["H"], c["causal"]) for c in varlen} == {(H, cz) for H in VARLEN_HS for cz in (True, False)}
    # the axes
    tabled = gqa + mla
    assert {c["causal"] for c in tabled} == {True, False} and {c["new"] for c in tabled} == {True, False}
    for G_rows in ("under", "full", "over"):
        want = {"under": lambda n: n < ROWS, "full": lambda n: n == ROWS, "over": lambda n: n > ROWS and n % ROWS}[G_rows]
        assert any(want(c["sq"] * c["G"]) for c in gqa), G_rows
        assert any(want(c["sq"] * c["G"]) for c in mla) or G_rows == "full", G_rows
    assert {Lk % TILE == 0 for c in tabled for Lk in c["Lks"]} == {True, False}
    assert any(c["causal"] and not c["new"] and 0 < Lk < c["sq"] for c in tabled for Lk in c["Lks"])  # blind rows
    assert any(Lk == 0 for c in tabled for Lk in c["Lks"])                                         # an empty request
    assert any(_has_empty_split(c) for c in gqa) and any(_has_empty_split(c) for c in mla)
    assert any(_more_splits_than_tiles(c) for c in gqa) and any(_more_splits_than_tiles(c) for c in mla)
    assert {c["page"] for c in gqa if c["entry"] == "paged"} == set(PAGED_PAGES)
    assert {c["page"] for c in gqa if c["entry"] == "fp8"} == set(FP8_PAGES)
    assert {c["hint"] for c in gqa} == set(HINTS) and {c["hint"] for c in mla} >= {"exact", "above"}
    for c in varlen:
        pairs = list(zip(c["lens_q"], c["lens_k"]))
        assert any(q == 0 for q, _ in pairs) and any(k == 0 and q > 0 for q, k in pairs)
        assert any(k > q > 0 for q, k in pairs) and any(q > k > 0 for q, k in pairs)
    assert any(64 % c["H"] for c in varlen) and {c["shared_v"] for c in varlen} == {True, False}


def test_split_ranges_cover_each_rows_keys_once():
    """For every row of every row tile the splits' key ranges cover [0, lim(r)) exactly once, in order, from 64-key
    tile starts; causal low row tiles and hints above the lengths leave trailing splits empty."""
    empty = 0
    for sq in (1, 3, 16, 70):
        for G in (1, 2, 8, 24):
            for Lk in (0, 1, 5, 63, 64, 65, 200, 1000):
                for causal in (True, False):
                    for S in (1, 2, 7, 64):
                        nrows = sq * G
                        for r in range(nrows):
                            rg = [x for x in key_ranges(r, G, nrows, Lk, sq, causal, S) if x[1] > x[0]]
                            L = lim(r, G, Lk, sq, causal)
                            ends = [0] + [hi for _, hi in rg]         # in order, each starting where the last ended
                            assert [lo for lo, _ in rg] == ends[:-1] and ends[-1] == L, (sq, G, Lk, causal, S, r)
                            assert all(lo % TILE == 0 for lo, _ in rg)
                            empty += len(rg) < S
    assert empty
    # causal, one row tile per token group: the first tile of a 128-row request ends 64 / G tokens in, so with 4 splits
    # over its one key tile three are empty, while the second tile's splits all take keys
    assert [hi > lo for lo, hi in key_ranges(0, 1, 128, 128, 128, True, 4)] == [True, False, False, False]
    assert all(hi > lo for lo, hi in key_ranges(127, 1, 128, 256, 128, True, 2))


def test_backend_workspace_lowers_the_split_count():
    """The backend sizes its workspace for B * Hq rows (workspace.attn_bytes, rounded up to a power of two by
    workspace.get); the prefill partials need B * sq * Hq rows, so the split count falls to about 128 / sq there."""
    from chitu_b200 import workspace
    for B, H, dv in ((1, 32, D), (2, 8, D), (3, 40, D), (1, 16, MLA_C), (4, 128, MLA_C), (64, 128, MLA_C)):
        assert workspace.attn_bytes(B, H, dv) == backend_attn_bytes(B, H, dv)
    B, Hq, Hkv = 1, 32, 8
    ws = backend_ws_bytes(B, Hq, D)
    assert ws == 1 << 22
    got = {}
    for sq in (2, 4, 8, 16, 32, 64, 128):
        S, picked = prefill_splits("gqa", B, sq, Hq, Hkv, 32768, ws)
        cap = (ws - 256) // (B * sq * Hq * (D + 1) * 4)
        assert S == max(min(picked, cap), 1)
        got[sq] = (S, picked)
    # (splits, picked): the wave rule's count until the partials of 128 / sq splits outgrow the buffer
    assert got == {2: (33, 33), 4: (33, 33), 8: (31, 33), 16: (15, 33), 32: (7, 16), 64: (3, 8), 128: (1, 4)}
    ws = backend_ws_bytes(1, 16, MLA_C)
    assert [prefill_splits("mla", 1, sq, 16, 1, 32768, ws) for sq in (2, 4, 7, 16)] == [(64, 64), (63, 64), (36, 64),
                                                                                          (15, 33)]


# ------------------------------------------------------------------------- injected-error self-test of the bound
def _selftest_shapes():
    """(dtype, G, Dk, Dv, page, L_cache, sq, new, causal, S) of the case tables, one request each, short enough for
    the CPU."""
    out = set()
    for c in gqa_case_table():
        if max(c["Lks"]) <= 3000:
            out.add((c["dtype"], c["G"], D, D, c["page"] or TILE, c["lens"][0], c["sq"], c["new"], c["causal"],
                     c["splits"]))
    for c in mla_case_table():
        if max(c["Lks"]) <= 3000:
            out.add((BF, min(c["H"], 8), MLA_ROW, MLA_C, TILE, c["lens"][0], c["sq"], c["new"], c["causal"],
                     c["splits"]))
    return sorted(out, key=lambda t: (str(t[0]), t[1:]))


def _prefill_injections(G, sq, L_cache, new, causal, S, page):
    """(name, token, needle key, the keys a kernel with that error gives the token's rows) for one request; the key
    index Lk + 1 stands for a stale cache slot."""
    Lk = L_cache + (sq if new else 0)
    nrows = sq * G
    li = lambda i: lim(i * G, G, Lk, sq, causal)
    seeing = [i for i in range(sq) if li(i) >= 2]
    if not seeing:
        return
    i = seeing[-1]
    L = li(i)
    yield "diagonal one key early", i, L - 1, list(range(L - 1))
    if causal and i > 0 and li(i - 1) >= 1 and li(i - 1) < Lk:
        j = i - 1
        yield "diagonal one key late", j, li(j), list(range(li(j) + 1))
    r0 = (i * G) // ROWS * ROWS
    first = lim(r0, G, Lk, sq, causal)
    if first < L:
        yield "tile masked with its first row's limit", i, L - 1, list(range(first))
    rg = [x for x in key_ranges(i * G, G, nrows, Lk, sq, causal, S) if x[1] > x[0]]
    if len(rg) > 1:
        b = rg[1][0]
        yield "key dropped at a split boundary", i, b, [k for k in range(L) if k != b]
        yield "key counted twice at a split boundary", i, b, list(range(L)) + [b]
    if new and L > L_cache:
        # new row k written at L_cache + k + 1: the token's last visible new row is lost, a stale slot is seen
        yield "appended rows one position late", i, L - 1, list(range(L_cache)) + [Lk + 1] + list(range(L_cache, L - 1))
    if L > page:
        p0 = ((L - 1) // page) * page
        moved = range(p0, min(p0 + TILE, L))
        yield "tile through the wrong block-table entry", i, p0, [k - page if k in moved else k for k in range(L)]


def test_bound_rejects_injected_errors():
    """On the case tables' prefill shapes (one request, one or two kv heads, needle data on the affected token) the
    bound admits the correctly rounded fp64 reference and rejects each injected error: the causal diagonal one key off
    either way, a tile masked with its first row's limit, a key dropped or counted twice at a split boundary, the
    appended rows one position off, a tile through the wrong block-table entry, token and head swapped in the row map,
    and a split LSE taken in the natural-log domain."""
    names = set()
    g = torch.Generator().manual_seed(0)
    for dtype, G, Dk, Dv, page, L_cache, sq, new, causal, S in _selftest_shapes():
        mla = Dk == MLA_ROW
        Hkv = 2 if G == 1 else 1
        scale = MLA_SCALE if mla else 1.0 / math.sqrt(Dk)
        Lk = L_cache + (sq if new else 0)
        N = Lk + 2                                                  # the stale slot at Lk + 1
        u_p = U_P[dtype]

        def data(i, pos, mass=0.4):
            q = (torch.randn(Hkv, sq * G, Dk, generator=g) * (0.3 if mla else 1.0)).to(dtype).double()
            K = torch.randn(N, Hkv, Dk, generator=g).to(dtype).double()
            _needle(q[:, i * G:(i + 1) * G], K, pos, lim(i * G, G, Lk, sq, causal), scale, mass, dtype)
            if mla:
                return q, K, K[..., :Dv]
            V = torch.randn(N, Hkv, Dv, generator=g).to(dtype).double()
            V[pos] *= 2
            return q, K, V

        def token_ref(q, K, V, i):
            L = lim(i * G, G, Lk, sq, causal)
            o, _, terms = ref_splits(q[:, i * G:(i + 1) * G], K, V, L, 1, max(L, 1), scale)
            o, terms = o[:, :, 0], tuple(t[:, :, 0] for t in terms)
            return o, bound(o, terms, U_OUT[dtype], u_p)

        for name, i, pos, keyset in _prefill_injections(G, sq, L_cache, new, causal, S, page):
            q, K, V = data(i, pos)
            o, bnd = token_ref(q, K, V, i)
            assert ratio(o.to(dtype), o, bnd) <= 1.0, (name, G, sq, L_cache)
            wrong = _weights_out(q[:, i * G:(i + 1) * G], K, V, keyset, scale)
            names.add(name)
            assert ratio(wrong.to(dtype), o, bnd) > 1.0, (name, dtype, G, Dk, page, L_cache, sq, new, causal, S)
        # token and head swapped in the row map (r -> token r % sq, head r // sq), over the whole request
        i = sq - 1
        if G > 1 and lim(i * G, G, Lk, sq, causal) >= 1:
            q, K, V = data(i, lim(i * G, G, Lk, sq, causal) - 1)
            lims = torch.tensor([lim(r, G, Lk, sq, causal) for r in range(sq * G)])
            o, _, terms = ref_splits(q, K, V, lims, 1, max(Lk, 1), scale)
            o, terms = o[:, :, 0], tuple(t[:, :, 0] for t in terms)
            bnd = bound(o, terms, U_OUT[dtype], u_p)
            assert ratio(o.to(dtype), o, bnd) <= 1.0
            r = torch.arange(sq * G)
            swapped = torch.empty_like(o)
            swapped[:, (r % sq) * G + r // sq] = o
            names.add("token and head swapped")
            assert ratio(swapped.to(dtype), o, bnd) > 1.0, ("swap", G, sq, L_cache, causal)
        # the split LSEs merged in the natural-log domain, for the last token's rows
        rg = [x for x in key_ranges(i * G, G, sq * G, Lk, sq, causal, S) if x[1] > x[0]]
        if len(rg) > 1:
            q, K, V = data(i, rg[-1][0], 0.8)          # unequal split LSEs: the domain matters
            o, bnd = token_ref(q, K, V, i)
            L = lim(i * G, G, Lk, sq, causal)
            _, per = tile_split(i * G - (i * G) % ROWS, sq * G, G, Lk, sq, causal, S)
            op, lse, _ = ref_splits(q[:, i * G:(i + 1) * G], K, V, L, S, TILE * per, scale)
            lse_ln = torch.where(torch.isfinite(lse), lse * math.log(2), -math.inf)
            w = torch.softmax(lse_ln * math.log(2), dim=-1)
            merged = torch.einsum("kgs,kgsd->kgd", w, op)
            names.add("split LSE in the natural-log domain")
            assert ratio(merged.to(dtype), o, bnd) > 1.0, ("lse", G, sq, L_cache, S)
    assert names == {"diagonal one key early", "diagonal one key late", "tile masked with its first row's limit",
                     "key dropped at a split boundary", "key counted twice at a split boundary",
                     "appended rows one position late", "tile through the wrong block-table entry",
                     "token and head swapped", "split LSE in the natural-log domain"}


# ---------------------------------------------------------------------------------------------------- GPU calls
def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def _diagonal_needles(q_tok, K, V, tokens, lim_tok, scale, dtype, scale_v=True):
    """Key lim(i) - 1 of each token i (its last visible key) carries about 40 % of token i's softmax mass: a causal
    limit one key short or long moves that token's rows far outside the bound.  q_tok(i) is [Hkv, G, Dk] double."""
    for i in tokens:
        L = lim_tok(i)
        if L < 2:
            continue
        p = L - 1
        qt = q_tok(i)
        s = torch.einsum("kgd,lkd->kgl", qt, K[:p]) * scale
        t = math.log(0.4 / 0.6) + torch.logsumexp(s, dim=-1).mean()
        _shape_keys(qt, K, torch.tensor([p], device=K.device), t.reshape(1), scale, dtype)
        if scale_v:
            V[p] *= 2


def _needle_tokens(sq, causal):
    return sorted({sq - 1, sq // 2, 0} if causal else {sq - 1})


def _make_keys(c, kind, q_tok, Dk, Dv, dt, scale, g, mla):
    """Per request K [Lk, Hkv, Dk] and V [Lk, Hkv, Dv] (double, exact io-dtype values): random, diagonal needles or a
    ramp of tile maxima ("mixed": needle and ramp by request)."""
    B, sq, Hkv, G = len(c["Lks"]), c["sq"], c["Hkv"], c["G"]
    kinds = []
    for b in range(B):
        k = kind if kind != "mixed" else ("needle", "ramp")[(b + c["seed"]) % 2]
        kinds.append(k)
    q_last = [q_tok(b, sq - 1) for b in range(B)]
    picks = [("ramp" if k == "ramp" else "random", 0) for k in kinds]
    Kd = _keys(q_last, B, c["Lks"], picks, Hkv, Dk, dt, scale, g, "prefill", TILE)
    Vd = [None] * B if mla else [torch.randn(L, Hkv, Dv, generator=g, device=DEV).to(dt).double() for L in c["Lks"]]
    for b in range(B):
        if kinds[b] == "needle" and c["Lks"][b] > 1:
            li = lambda i, b=b: lim(i * G, G, c["Lks"][b], sq, c["causal"])
            _diagonal_needles(lambda i, b=b: q_tok(b, i), Kd[b], Vd[b], _needle_tokens(sq, c["causal"]), li, scale,
                              dt, scale_v=not mla)
    return Kd, Vd, kinds


def _check_request(y, o_part, lse, q_rows, K, V, G, Lk, sq, causal, S, scale, dt, what):
    """One request: y [Hkv, nrows, Dv] against the fp64 reference, row tile by row tile with each row's causal limit;
    with S > 1 also the split partials o_part [Hkv, nrows, S, Dv] and LSEs [Hkv, nrows, S] against each row's key ranges
    (rows grouped by how many of their splits take keys).  Returns the worst ratio."""
    Hkv, nrows, _ = q_rows.shape
    u_p = U_P[dt]
    worst = 0.0
    for r0 in range(0, nrows, ROWS):
        r1 = min(r0 + ROWS, nrows)
        lims = [lim(r, G, Lk, sq, causal) for r in range(r0, r1)]
        lt = torch.tensor(lims, device=q_rows.device)
        qt = q_rows[:, r0:r1]
        o, _, terms = ref_splits(qt, K, V, lt, 1, max(max(lims), 1), scale)
        o, terms = o[:, :, 0], tuple(t[:, :, 0] for t in terms)
        r = ratio(y[:, r0:r1], o, bound(o, terms, U_OUT[dt], u_p))
        assert r <= 1.0, ("outside the bound", r0, r) + what
        worst = max(worst, r)
        if S == 1:
            continue
        _, per = tile_split(r0, nrows, G, Lk, sq, causal, S)
        res = ref_splits(qt, K, V, lt, S, TILE * max(per, 1), scale)
        ranges = [key_ranges(rr, G, nrows, Lk, sq, causal, S) for rr in range(r0, r1)]
        counts = [sum(hi > lo for lo, hi in rg) for rg in ranges]
        for n in sorted(set(counts)):
            sel = torch.tensor([k for k, cnt in enumerate(counts) if cnt == n], device=q_rows.device)
            pick = lambda t, sel=sel: t[:, sel].reshape(-1, *t.shape[2:])
            fn = lambda pick=pick: (pick(res[0]), pick(res[1]), tuple(pick(t) for t in res[2]))
            w = _split_checks(pick(o_part[:, r0:r1]), pick(lse[:, r0:r1]), fn, ranges[counts.index(n)], u_p,
                              what + (r0, n))
            worst = max(worst, w)
    return worst


def _check_workspace(ws_after, n_part, S, what):
    """S > 1: exactly the first n_part bytes written (no 0xFFFFFFFF word left); S == 1: no byte changed."""
    assert bool((ws_after[n_part:] == 0xFF).all()), ("workspace written past the modelled partials",) + what
    if S > 1:
        assert bool((ws_after[:n_part].view(torch.int32) != -1).all()), ("partial not written",) + what


def run_gqa(c, kind, via="c"):
    """One GQA case through its C entry (via="c") or B200AttnBackend.attn_with_kvcache (via="backend", c["ws"] the size
    of the backend's buffer); returns the worst ratio to the bound."""
    from chitu_b200 import _lib as L
    from chitu_b200._lib import check, current_stream, dtype_code, ptr
    lib = _lib()
    entry, dt = c["entry"], c["dtype"]
    B, sq, Hq, Hkv, G, page = c["B"], c["sq"], c["Hq"], c["Hkv"], c["G"], c["page"]
    new, causal, lens, Lks, S = c["new"], c["causal"], c["lens"], c["Lks"], c["splits"]
    g = torch.Generator(device=DEV).manual_seed(1000 * c["seed"] + len(kind))
    scale = 1.0 / math.sqrt(D)
    what = (entry, str(dt), G, B, Hkv, sq, tuple(lens), new, causal, page, c["hint"], c.get("regime"), S, kind, via)

    q = torch.randn(B, sq, Hq, D, generator=g, device=DEV).to(dt)
    q_tok = lambda b, i: q[b, i].view(Hkv, G, D).double()
    Kd, Vd, _ = _make_keys(c, kind, q_tok, D, D, dt, scale, g, False)
    store = F8 if entry == "fp8" else dt
    if entry == "fp8":
        Kd = [k.float().clamp(-448, 448).to(F8).double() for k in Kd]
        Vd = [v.float().clamp(-448, 448).to(F8).double() for v in Vd]
    # the new rows as strided views of a fused qkv output [B, sq, (Hq + 2 Hkv) D] (the q part is NaN)
    W = (Hq + 2 * Hkv) * D
    qkv = Padded(shape=(B, sq, W), dtype=dt, fill=NAN_BYTE)
    kn = qkv.view[..., Hq * D:(Hq + Hkv) * D].view(B, sq, Hkv, D)
    vn = qkv.view[..., (Hq + Hkv) * D:].view(B, sq, Hkv, D)
    if new:
        for b in range(B):
            kn[b] = Kd[b][lens[b]:].to(dt)
            vn[b] = Vd[b][lens[b]:].to(dt)

    if entry == "contig":
        rows = c["rows"]
        kc = torch.full((B + 1, rows, Hkv, D), float("nan"), dtype=dt, device=DEV)
        vc = kc.clone()
        for b in range(B):
            kc[b, :lens[b]] = Kd[b][:lens[b]].to(dt)
            vc[b, :lens[b]] = Vd[b][:lens[b]].to(dt)
        bt = None
    else:
        bt, nb, _ = _block_table(B, c["npages"], torch.Generator(device=DEV).manual_seed(c["seed"]))
        assert bt.shape[1] == c["bt_stride"]
        kc = torch.full((nb, page, Hkv, D), float("nan"), dtype=dt, device=DEV).to(store)
        vc = kc.clone()
        for b in range(B):
            j = torch.arange(lens[b], device=DEV)
            pg, off = bt[b, j // page].long(), j % page
            kc[pg, off] = Kd[b][:lens[b]].float().to(store)
            vc[pg, off] = Vd[b][:lens[b]].float().to(store)
    want_k, want_v = kc.clone(), vc.clone()
    if new:
        for b in range(B):
            j = torch.arange(lens[b], Lks[b], device=DEV)
            if entry == "contig":
                want_k[b, j], want_v[b, j] = Kd[b][j].float().to(store), Vd[b][j].float().to(store)
            else:
                pg, off = bt[b, j // page].long(), j % page
                want_k[pg, off], want_v[pg, off] = Kd[b][j].float().to(store), Vd[b][j].float().to(store)

    qp = Padded(q)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ksb, kst = (kn.stride(0), kn.stride(1)) if new else (0, 0)
    st = current_stream()
    before = L.launch_count()
    if via == "backend":
        from chitu_b200.attn_backend import B200AttnBackend
        be = B200AttnBackend()
        ws_buf, n = be._ws(B, Hq, D, DEV)
        assert n == c["ws"], ("the backend's workspace is not the modelled one", n) + what
        ws_buf.fill_(0xFF)
        y = be.attn_with_kvcache(qp.view, kc, vc, kn if new else None, vn if new else None, lens_d, block_table=bt,
                                 causal=causal)
        torch.cuda.synchronize()
        ws_after = ws_buf.clone()
        ws_buf.zero_()
        out = None
    else:
        out = Padded(shape=(B, sq, Hq, D), dtype=dt, pad=SENTINEL, fill=NAN_BYTE)
        ws = Padded(shape=(c["ws"],), dtype=torch.uint8, pad=SENTINEL, fill=0xFF) if c["ws"] is not None else None
        wsp, wsn = (ptr(ws.view), c["ws"]) if ws is not None else (None, 0)
        knp, vnp = (ptr(kn), ptr(vn)) if new else (None, None)
        if entry == "paged":
            rc = lib.chitu_b200_gqa_paged_prefill(
                ptr(qp.view), ptr(kc), ptr(vc), knp, vnp, ksb, kst, ksb, kst, ptr(lens_d), ptr(bt), bt.stride(0), B, sq,
                Hq, Hkv, D, page, kc.shape[0], c["hint_arg"], int(causal), scale, ptr(out.view), wsp, wsn,
                dtype_code(dt), st)
        elif entry == "contig":
            rc = lib.chitu_b200_gqa_contiguous_attn(
                ptr(qp.view), ptr(kc), ptr(vc), kc.stride(0), rows, knp, vnp, ksb, kst, ksb, kst, ptr(lens_d), B, sq, Hq,
                Hkv, D, c["hint_arg"], int(causal), scale, ptr(out.view), wsp, wsn, dtype_code(dt), st)
        else:
            rc = lib.chitu_b200_gqa_paged_attn_fp8kv(
                ptr(qp.view), sq * Hq * D, ptr(kc), ptr(vc), knp, vnp, ksb, kst, ksb, kst, None, None, ptr(lens_d),
                ptr(bt), bt.stride(0), B, sq, Hq, Hkv, D, page, kc.shape[0], c["hint_arg"], int(causal), scale,
                ptr(out.view), wsp, wsn, dtype_code(dt), st)
        check(rc, str(what))
        torch.cuda.synchronize()
        y = out.view
        ws_after = ws.bytes.clone() if ws is not None else None
        assert out.pads_intact() and (ws is None or ws.pads_intact()), ("pad overwritten",) + what
    assert L.launch_count() - before == int(new) + 1 + int(S > 1), ("launches",) + what
    assert qp.pads_intact() and qkv.pads_intact(), ("pad overwritten",) + what
    assert torch.equal(_bits(kc), _bits(want_k)) and torch.equal(_bits(vc), _bits(want_v)), \
        ("the cache differs from the reference scatter",) + what

    rows_ = B * sq * Hq
    n_part = rows_ * S * (D + 1) * 4 if S > 1 else 0
    if ws_after is not None:
        _check_workspace(ws_after, n_part, S, what)
    if S > 1:
        o_part = ws_after[:rows_ * S * D * 4].view(torch.float32).view(B, sq, Hkv, G, S, D)
        lse = ws_after[rows_ * S * D * 4:n_part].view(torch.float32).view(B, sq, Hkv, G, S)
    worst = 0.0
    for b in range(B):
        to_rows = lambda t: t.transpose(0, 1).reshape(Hkv, sq * G, *t.shape[3:])    # [sq, Hkv, G, ...] -> rows
        q_rows = to_rows(q[b].view(sq, Hkv, G, D)).double()
        yb = to_rows(y[b].view(sq, Hkv, G, D))
        op, lp = (to_rows(o_part[b]), to_rows(lse[b])) if S > 1 else (None, None)
        worst = max(worst, _check_request(yb, op, lp, q_rows, Kd[b], Vd[b], G, Lks[b], sq, causal, S, scale, dt,
                                          what + (b,)))
    return worst


def run_mla(c, kind, via="c"):
    """One MLA paged case through chitu_b200_mla_paged_prefill or B200AttnBackend.mla_attn_with_kvcache."""
    from chitu_b200 import _lib as L
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib()
    B, sq, H, new, causal, lens, Lks, S = (c[k] for k in ("B", "sq", "H", "new", "causal", "lens", "Lks", "splits"))
    g = torch.Generator(device=DEV).manual_seed(1000 * c["seed"] + len(kind))
    what = ("mla", H, B, sq, tuple(lens), new, causal, c["hint"], c.get("regime"), S, kind, via)
    q = (torch.randn(B, sq, H, MLA_ROW, generator=g, device=DEV) * 0.3).to(BF)
    q_tok = lambda b, i: q[b, i][None].double()
    Kd, _, _ = _make_keys(c, kind, q_tok, MLA_ROW, MLA_C, BF, MLA_SCALE, g, True)
    bt, nb, _ = _block_table(B, c["npages"], torch.Generator(device=DEV).manual_seed(c["seed"]))
    assert bt.shape[1] == c["bt_stride"]
    cache = torch.full((nb, TILE, MLA_ROW), float("nan"), dtype=BF, device=DEV)
    for b in range(B):
        j = torch.arange(lens[b], device=DEV)
        cache[bt[b, j // TILE].long(), j % TILE] = Kd[b][:lens[b], 0].to(BF)
    want = cache.clone()
    new_kv = None
    if new:
        new_kv = Padded(torch.stack([Kd[b][lens[b]:, 0] for b in range(B)]).to(BF))
        for b in range(B):
            j = torch.arange(lens[b], Lks[b], device=DEV)
            want[bt[b, j // TILE].long(), j % TILE] = Kd[b][j, 0].to(BF)
    qn = Padded(q[..., :MLA_C].contiguous())
    qpe = Padded(q[..., MLA_C:].contiguous())
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    before = L.launch_count()
    if via == "backend":
        from chitu_b200.attn_backend import B200AttnBackend
        be = B200AttnBackend()
        ws_buf, n = be._ws(B, H, MLA_C, DEV)
        assert n == c["ws"], ("the backend's workspace is not the modelled one", n) + what
        ws_buf.fill_(0xFF)
        y = be.mla_attn_with_kvcache(qn.view, qpe.view, cache, new_kv.view if new else None, lens_d, None, bt,
                                     causal=causal, softmax_scale=MLA_SCALE)
        torch.cuda.synchronize()
        ws_after = ws_buf.clone()
        ws_buf.zero_()
    else:
        out = Padded(shape=(B, sq, H, MLA_C), dtype=BF, pad=SENTINEL, fill=NAN_BYTE)
        ws = Padded(shape=(c["ws"],), dtype=torch.uint8, pad=SENTINEL, fill=0xFF)
        check(lib.chitu_b200_mla_paged_prefill(
            ptr(qn.view), ptr(qpe.view), ptr(cache), ptr(new_kv.view) if new else None, ptr(lens_d), ptr(bt),
            bt.stride(0), B, sq, H, MLA_C, MLA_R, TILE, nb, c["hint_arg"], int(causal), MLA_SCALE, ptr(out.view),
            ptr(ws.view), c["ws"], current_stream()), str(what))
        torch.cuda.synchronize()
        y = out.view
        ws_after = ws.bytes.clone()
        assert out.pads_intact() and ws.pads_intact(), ("pad overwritten",) + what
    assert L.launch_count() - before == int(new) + 1 + int(S > 1), ("launches",) + what
    assert qn.pads_intact() and qpe.pads_intact() and (new_kv is None or new_kv.pads_intact()), ("pad",) + what
    assert torch.equal(_bits(cache), _bits(want)), ("the cache differs from the reference scatter",) + what
    rows_ = B * sq * H
    n_part = rows_ * S * (MLA_C + 1) * 4 if S > 1 else 0
    _check_workspace(ws_after, n_part, S, what)
    if S > 1:
        o_part = ws_after[:rows_ * S * MLA_C * 4].view(torch.float32).view(B, 1, sq * H, S, MLA_C)
        lse = ws_after[rows_ * S * MLA_C * 4:n_part].view(torch.float32).view(B, 1, sq * H, S)
    worst = 0.0
    for b in range(B):
        q_rows = q[b].reshape(1, sq * H, MLA_ROW).double()
        K = Kd[b]
        worst = max(worst, _check_request(y[b].reshape(1, sq * H, MLA_C), o_part[b] if S > 1 else None,
                                          lse[b] if S > 1 else None, q_rows, K, K[..., :MLA_C], H, Lks[b], sq, causal,
                                          S, MLA_SCALE, BF, what + (b,)))
    return worst


def run_varlen(c, kind, via="c"):
    """One varlen MLA case through chitu_b200_mla_prefill or B200AttnBackend.attn_varlen_func, k and v as strided views
    of NaN-padded buffers (v the first 512 columns of k's rows, or its own buffer)."""
    from chitu_b200 import _lib as L
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib()
    H, causal, lens_q, lens_k = c["H"], c["causal"], c["lens_q"], c["lens_k"]
    g = torch.Generator(device=DEV).manual_seed(1000 * c["seed"] + len(kind))
    what = ("varlen", H, causal, tuple(lens_q), tuple(lens_k), c["shared_v"], kind, via)
    Tq, Tk = sum(lens_q), sum(lens_k)
    q = (torch.randn(Tq, H, MLA_ROW, generator=g, device=DEV) * 0.3).to(BF)
    kbuf = Padded(shape=(Tk, 1, 640), dtype=BF, fill=NAN_BYTE)
    vbuf = Padded(shape=(Tk, 1, 520), dtype=BF, fill=NAN_BYTE)
    Ks, Vs = [], []
    ok = oq = 0
    for s, (lq, lk) in enumerate(zip(lens_q, lens_k)):
        cs = dict(Lks=[lk], sq=lq, Hkv=1, G=H, causal=causal, seed=c["seed"] + s)
        q_tok = lambda b, i, oq=oq: q[oq + i][None].double()
        if lq > 0:
            K, _, _ = _make_keys(cs, kind, q_tok, MLA_ROW, MLA_C, BF, MLA_SCALE, g, True)
            K = K[0]
        else:
            K = torch.randn(lk, 1, MLA_ROW, generator=g, device=DEV).to(BF).double()
        V = K[..., :MLA_C] if c["shared_v"] else torch.randn(lk, 1, MLA_C, generator=g, device=DEV).to(BF).double()
        kbuf.view[ok:ok + lk, :, :MLA_ROW] = K.to(BF)
        vbuf.view[ok:ok + lk, :, :MLA_C] = V.to(BF)
        Ks.append(K)
        Vs.append(V)
        ok += lk
        oq += lq
    k = kbuf.view[:, :, :MLA_ROW]
    v = k[..., :MLA_C] if c["shared_v"] else vbuf.view[:, :, :MLA_C]
    qp = Padded(q)
    cu = lambda lens: torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32, device=DEV)
    cq, ck = cu(lens_q), cu(lens_k)
    before = L.launch_count()
    if via == "backend":
        from chitu_b200.attn_backend import B200AttnBackend
        y = B200AttnBackend().attn_varlen_func(qp.view, k, v, cq, ck, max(lens_q), max(lens_k), causal=causal,
                                               softmax_scale=MLA_SCALE)
        torch.cuda.synchronize()
    else:
        out = Padded(shape=(Tq, H, MLA_C), dtype=BF, pad=SENTINEL, fill=NAN_BYTE)
        check(lib.chitu_b200_mla_prefill(ptr(qp.view), ptr(k), k.stride(0), ptr(v), v.stride(0), ptr(cq), ptr(ck),
                                          len(lens_q), H, Tq, Tk, max(lens_q), int(causal), MLA_SCALE, ptr(out.view),
                                          current_stream()), str(what))
        torch.cuda.synchronize()
        y = out.view
        assert out.pads_intact(), ("output pad overwritten",) + what
    assert L.launch_count() - before == 1, ("launches",) + what
    assert qp.pads_intact() and kbuf.pads_intact() and vbuf.pads_intact(), ("pad",) + what
    worst = 0.0
    oq = 0
    for s, (lq, lk) in enumerate(zip(lens_q, lens_k)):
        if lq:
            q_rows = q[oq:oq + lq].reshape(1, lq * H, MLA_ROW).double()
            ys = y[oq:oq + lq].reshape(1, lq * H, MLA_C)
            worst = max(worst, _check_request(ys, None, None, q_rows, Ks[s], Vs[s], H, lk, lq, causal, 1, MLA_SCALE,
                                              BF, what + (s,)))
        oq += lq
    return worst


KINDS = ("mixed", "random")


# ------------------------------------------------------------------------------------- parity over the case table
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ENTRIES)
def test_gqa_prefill_case_table_parity(entry):
    """Every GQA case of the entry on needle / ramp and on random data: the cache bit-exact with the reference scatter,
    the modelled split count and launches, every split partial and LSE within the bound over its key range, empty splits
    exactly 0 with LSE -inf, the rest of the workspace untouched, the output within the bound, blind rows exactly 0, the
    pads intact."""
    cases = [c for c in gqa_case_table() if c["entry"] == entry]
    worst = 0.0
    for c in cases:
        for kind in KINDS:
            worst = max(worst, run_gqa(c, kind))
    _report(f"prefill-{entry}", len(cases), worst)


@pytest.mark.gpu
def test_mla_paged_prefill_case_table_parity():
    cases = mla_case_table()
    worst = 0.0
    for c in cases:
        for kind in KINDS:
            worst = max(worst, run_mla(c, kind))
    _report("prefill-mla-paged", len(cases), worst)


@pytest.mark.gpu
def test_mla_varlen_case_table_parity():
    cases = varlen_case_table()
    worst = 0.0
    for c in cases:
        for kind in KINDS:
            worst = max(worst, run_varlen(c, kind))
    _report("prefill-mla-varlen", len(cases), worst)


@pytest.mark.gpu
def test_through_the_backend():
    """attn_with_kvcache (paged, contiguous, fp8), mla_attn_with_kvcache and attn_varlen_func with seqlen_q > 1: the
    split count the backend's own workspace yields is the modelled one, and the output is within the bound."""
    from chitu_b200.attn_backend import B200AttnBackend
    be = B200AttnBackend()
    worst = 0.0
    for entry, dt, G, B, Hkv, sq, lens, page in (("paged", BF, 4, 2, 2, 16, [3000, 500], 256),
                                                  ("contig", F16, 2, 1, 4, 32, [4000], None),
                                                  ("fp8", BF, 8, 1, 1, 40, [5000], 128)):
        Hq = G * Hkv
        n = be._ws(B, Hq, D, DEV)[1]
        c = make_gqa_case(entry, dt, G, B, Hkv, sq, lens, True, True, page, "zero", n, 7 + sq)
        fresh = make_gqa_case(entry, dt, G, B, Hkv, sq, lens, True, True, page, "zero", backend_ws_bytes(B, Hq, D), 0)
        assert fresh["splits"] < fresh["picked"]              # a fresh backend lowers these counts
        worst = max(worst, run_gqa(c, "mixed", via="backend"))
    n = be._ws(1, 16, MLA_C, DEV)[1]
    c = make_mla_case(16, 1, 7, [9000], True, True, "zero", n, 11)
    fresh = make_mla_case(16, 1, 7, [9000], True, True, "zero", backend_ws_bytes(1, 16, MLA_C), 0)
    assert fresh["splits"] < fresh["picked"]
    worst = max(worst, run_mla(c, "mixed", via="backend"))
    worst = max(worst, run_varlen(varlen_case_table()[4], "mixed", via="backend"))
    _report("prefill-backend", 5, worst)
