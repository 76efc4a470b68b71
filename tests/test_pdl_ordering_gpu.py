"""Reads that happen before `griddepcontrol.wait`, pinned against a writer that is still in flight.

Every kernel of the library is launched with programmatic dependent launch (PDL, csrc/common.cuh): almost all of them
run `griddepcontrol.launch_dependents` first, so the next kernel of the stream can become resident while its
predecessor is still blocked in its own `griddepcontrol.wait`.  Only that wait makes a predecessor's writes visible.
What a kernel reads before it is safe only if the writer does not trigger early, so nothing after the writer starts
before the writer has exited.

The harness makes the overlap happen on purpose, with no race to win: on one stream, with nothing launched in between,
  1. `chitu_b200_argmax` over one long row, a single CTA that triggers at once and runs for about 25 ms (sized from one
     timed launch);
  2. the writer, which becomes resident and blocks in its wait on the argmax;
  3. the reader, which becomes resident as soon as every CTA of the writer has started, and makes its pre-wait reads
     while the writer has written nothing.
Every grid is at most 64 CTAs (noted per case), so all three kernels fit in one wave on the 132 SMs of an H100.  The slots
the writer fills hold 0xFF bytes beforehand (NaN in bf16 and e4m3), so a stale read shows up as NaN or a wrong value.
The reference runs the same three launches with a device synchronisation after each; the overlapped run, and the same
launches captured in a CUDA graph (where PDL becomes programmatic edges) and replayed once, must leave every tensor of
the case bit-identical to it.  Each case also runs the reader without its writer and checks that the result changes:
a case whose reader does not depend on the writer would prove nothing.

KV cases: each KV writer (the prompt scatter in three layouts, the two appends, the seqlen_q > 1 entries and a
seqlen_q = 1 decode appending row L) before each seqlen_q = 1 reader of the same cache, on rows that lie in the
reader's first tiles (GQA, the tensor-core mmaT kernels) or pages (MLA).  Contract cases: readers that legitimately
read before their wait (GEMM and absorb-o weights, the MLA split plan, lengths and block table) after the writers that
must therefore never trigger early.  `test_pdl_source_audit` (CPU) keeps the list of early readers and the
non-triggering writers in step with csrc/*.cu."""
import math
import os
import re

import pytest
import torch

from chitu_b200 import _lib

DEV = "cuda:0"
BF, E4M3 = torch.bfloat16, torch.float8_e4m3fn
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "chitu_b200", "csrc")

SLOW_MS = 25.0             # the predecessor's run time the harness aims for (>= 10 ms leaves the host ample time)


# ---------------------------------------------------------------------------------------------------- harness
def _call(name, *args):
    _lib.check(getattr(_lib.load(), name)(*args), name)


def _st():
    return _lib.current_stream()


def _bits(t):
    return t.view(torch.uint8) if t.element_size() == 1 else t.view(torch.int16 if t.element_size() == 2 else torch.int32)


@pytest.fixture(scope="module")
def slow_row():
    """(logits, out) for one argmax that runs for about SLOW_MS: its length is scaled from one timed launch."""
    v0 = 1 << 22
    logits = torch.zeros(v0, dtype=BF, device=DEV)
    out = torch.zeros(1, dtype=torch.int64, device=DEV)
    _call("chitu_b200_argmax", logits.data_ptr(), out.data_ptr(), 1, v0, _lib.CB_BF16, _st())     # module load
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    _call("chitu_b200_argmax", logits.data_ptr(), out.data_ptr(), 1, v0, _lib.CB_BF16, _st())
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1)
    V = min(int(v0 * SLOW_MS / max(ms, 1e-3)) // 1024 * 1024 + 1024, 1 << 29)
    print(f"argmax over {v0} bf16: {ms:.3f} ms; slow row: {V} elements, about {ms * V / v0:.1f} ms")
    assert ms * V / v0 >= 10.0, "the slow predecessor would run for less than 10 ms"
    return torch.zeros(V, dtype=BF, device=DEV), out


def _slow(row):
    logits, out = row
    _call("chitu_b200_argmax", logits.data_ptr(), out.data_ptr(), 1, logits.numel(), _lib.CB_BF16, _st())


def _snapshot(state):
    return {k: _bits(v).clone() for k, v in state.items() if torch.is_tensor(v)}


def _differs(a, b):
    return [k for k in a if not torch.equal(a[k], b[k])]


def run_case(case, row):
    """case: (build, writer, reader); build() returns a fresh state dict of device tensors, writer / reader enqueue
    their launches on the current stream."""
    build, writer, reader = case
    # reference: the predecessor, the writer and the reader each complete before the next starts
    S = build()
    torch.cuda.synchronize()
    for f in (lambda: _slow(row), lambda: writer(S), lambda: reader(S)):
        f()
        torch.cuda.synchronize()
    ref = _snapshot(S)
    # the reader alone must see something else: the case depends on the writer
    S = build()
    torch.cuda.synchronize()
    reader(S)
    torch.cuda.synchronize()
    assert _differs(_snapshot(S), ref), "the reader's result does not depend on the writer"
    # overlapped: back to back on one stream
    S = build()
    torch.cuda.synchronize()
    _slow(row)
    writer(S)
    reader(S)
    torch.cuda.synchronize()
    bad = _differs(_snapshot(S), ref)
    assert not bad, f"back to back on one stream: {bad} differ from the synchronised launches"
    # the same launches as a CUDA graph, replayed once
    S = build()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _slow(row)
        writer(S)
        reader(S)
    g.replay()
    torch.cuda.synchronize()
    bad = _differs(_snapshot(S), ref)
    del g
    assert not bad, f"graph replay: {bad} differ from the synchronised launches"
    return ref


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rand(shape, g, dtype=BF, scale=1.0):
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def _ff(shape, dtype):
    """A tensor whose every byte is 0xFF: NaN in bf16 and e4m3."""
    es = torch.empty((), dtype=dtype).element_size()
    return torch.full((*shape[:-1], shape[-1] * es), 0xFF, dtype=torch.uint8, device=DEV).view(dtype)


def _i32(x):
    return torch.tensor(x, dtype=torch.int32, device=DEV)


def _p(t):
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------------- GQA caches
# B = 2 requests, Hkv = 2 kv heads of G = 2 query heads, D = 128, 64-token pages (a power of two: the mmaT kernels).
# Reader: one decode step with k / v appended at L_cache = (64, 48), max_seqlen_hint 65 -> one split: grid (1, 2, 2) =
# 4 CTAs.  Every cached row the writers below fill lies in the first two tiles of some warp (keys 0-255, wholly below
# L_cache): the tiles its prologue stages, and the ones a kernel that loaded tiles before its wait would take early.
GB, GHKV, GG, GD, GPAGE, GBT = 2, 2, 2, 128, 64, 4
GHQ = GHKV * GG
G_ROWS = ((32, 16), 32)            # scatter / seqlen_q > 1 writers: positions start .. start + 31
G_ROW = ((63, 47), 1)              # append / decode writers: row 63 (the last of tile 3) and 47
G_ROWS_CONTIG = 128                # rows per request of the non-paged cache
GSCALE = 1.0 / math.sqrt(GD)


def _gqa_build(layout, writes, seed):
    """A state over a GQA cache of `layout` (paged | e4m3 | contig): rows below the writer's start positions are
    cached data, the writer's slots and everything else 0xFF; the writer's sources and the reader's inputs."""
    starts, n = writes
    g = _gen(seed)
    cdt = E4M3 if layout == "e4m3" else BF
    S = {}
    if layout == "contig":
        shape = (GB, G_ROWS_CONTIG, GHKV, GD)
    else:
        nb = GB * GBT
        S["bt"] = torch.randperm(nb, generator=torch.Generator().manual_seed(seed)).to(torch.int32).view(GB, GBT).to(DEV)
        shape = (nb, GPAGE, GHKV, GD)
    for c in ("k", "v"):
        cache = _ff(shape, cdt)
        for b in range(GB):
            rows = _rand((starts[b], GHKV, GD), g, scale=2.0).float().clamp(-448, 448).to(cdt)
            if layout == "contig":
                _bits(cache)[b, :starts[b]] = _bits(rows)
            else:
                pos = torch.arange(starts[b], device=DEV)
                _bits(cache).view(-1, GHKV, GD)[S["bt"][b].long()[pos // GPAGE] * GPAGE + pos % GPAGE] = _bits(rows)
        S[c + "_cache"] = cache
    S["starts"] = _i32(list(starts))
    S["lens"] = _i32([s + n for s in starts])                   # the reader's L_cache
    S["src_k"], S["src_v"] = _rand((GB, n, GHKV, GD), g), _rand((GB, n, GHKV, GD), g)
    S["cu"] = _i32([0, n, 2 * n])
    S["wq"] = _rand((GB, n, GHQ, GD), g)                        # seqlen_q > 1 and decode writers
    S["wout"] = _ff((GB, n, GHQ, GD), BF)
    S["q"] = _rand((GB, GHQ, GD), g)
    S["k_new"], S["v_new"] = _rand((GB, GHKV, GD), g), _rand((GB, GHKV, GD), g)
    ang = torch.rand((GB, GD // 2), generator=g, device=DEV) * 6.0
    S["cos"], S["sin"] = ang.cos(), ang.sin()
    S["out"] = _ff((GB, GHQ, GD), BF)
    S["ws_bytes"] = int(_lib.load().chitu_b200_attn_workspace_bytes(GB, GHQ, GD, 8))
    S["ws"] = _ff((S["ws_bytes"],), torch.uint8)
    S["layout"] = layout
    return S


def _gqa_bt(S):
    return (_p(S["bt"]), GBT) if "bt" in S else (None, 0)


def _gqa_scatter(S):
    # one CTA per source row: 64 CTAs of 128 threads
    layout = S["layout"]
    n = S["src_k"].shape[1]
    bt, bts = _gqa_bt(S)
    cache_sb = G_ROWS_CONTIG * GHKV * GD if layout == "contig" else 0
    _call("chitu_b200_scatter_kv", _p(S["k_cache"]), _p(S["v_cache"]), _p(S["src_k"]), GHKV * GD, _p(S["src_v"]),
          GHKV * GD, _p(S["cu"]), _p(S["starts"]), bt, bts, GPAGE if bt else 0, cache_sb,
          G_ROWS_CONTIG if layout == "contig" else 0, GB, GB * n, GHKV * GD, _lib.CB_BF16,
          _lib.CB_FP8_E4M3 if layout == "e4m3" else _lib.CB_BF16, _st())


def _gqa_append(S):
    # append_paged_kv: one launch per cache, B = 2 CTAs each
    for c in ("k", "v"):
        src = S["src_" + c]
        if S["layout"] == "e4m3":
            _call("chitu_b200_append_paged_kv_e4m3", _p(S[c + "_cache"]), _p(S["bt"]), _p(src), _p(S["starts"]), GB,
                  GBT, GHKV * GD, _lib.CB_BF16, _st())
        else:
            _call("chitu_b200_append_paged_kv", _p(S[c + "_cache"]), _p(S["bt"]), _p(src), _p(S["starts"]), GB, GBT,
                  GPAGE, GPAGE, GHKV * GD * 2, _st())


def _gqa_multi(S):
    """The attention entry of the layout over S's writer tensors: seqlen_q = n (> 1: append + multi-token kernel,
    no workspace so no split: grids of B x Hkv x (query tiles) CTAs; 1: the decode kernel, 4 CTAs)."""
    layout = S["layout"]
    n = S["src_k"].shape[1]
    sb, st = n * GHKV * GD, GHKV * GD
    common = (_p(S["src_k"]), _p(S["src_v"]), sb, st, sb, st)
    if layout == "paged" and n > 1:
        _call("chitu_b200_gqa_paged_prefill", _p(S["wq"]), _p(S["k_cache"]), _p(S["v_cache"]), *common,
              _p(S["starts"]), _p(S["bt"]), GBT, GB, n, GHQ, GHKV, GD, GPAGE, GB * GBT, 128, 1, GSCALE,
              _p(S["wout"]), None, 0, _lib.CB_BF16, _st())
    elif layout == "paged":
        _call("chitu_b200_gqa_paged_decode", _p(S["wq"]), _p(S["k_cache"]), _p(S["v_cache"]), _p(S["src_k"]),
              _p(S["src_v"]), GHKV * GD, GHKV * GD, _p(S["starts"]), _p(S["bt"]), GBT, GB, GHQ, GHKV, GD, GPAGE, 65,
              GSCALE, _p(S["wout"]), None, 0, _lib.CB_BF16, _st())
    elif layout == "e4m3":
        _call("chitu_b200_gqa_paged_attn_fp8kv", _p(S["wq"]), n * GHQ * GD, _p(S["k_cache"]), _p(S["v_cache"]),
              *common, None, None, _p(S["starts"]), _p(S["bt"]), GBT, GB, n, GHQ, GHKV, GD, GPAGE, GB * GBT, 128, 1,
              GSCALE, _p(S["wout"]), None, 0, _lib.CB_BF16, _st())
    else:
        _call("chitu_b200_gqa_contiguous_attn", _p(S["wq"]), _p(S["k_cache"]), _p(S["v_cache"]),
              G_ROWS_CONTIG * GHKV * GD, G_ROWS_CONTIG, *common, _p(S["starts"]), GB, n, GHQ, GHKV, GD, 128, 1, GSCALE,
              _p(S["wout"]), None, 0, _lib.CB_BF16, _st())


def _gqa_read(kind):
    """The seqlen_q = 1 reader: decode at L_cache = S["lens"] with k / v appended, mmaT kernel, one split."""
    def read(S):
        ws, wsb = _p(S["ws"]), S["ws_bytes"]
        kn, vn, sb = _p(S["k_new"]), _p(S["v_new"]), GHKV * GD
        if kind == "decode":
            _call("chitu_b200_gqa_paged_decode", _p(S["q"]), _p(S["k_cache"]), _p(S["v_cache"]), kn, vn, sb, sb,
                  _p(S["lens"]), _p(S["bt"]), GBT, GB, GHQ, GHKV, GD, GPAGE, 65, GSCALE, _p(S["out"]), ws, wsb,
                  _lib.CB_BF16, _st())
        elif kind == "decode_rope":
            _call("chitu_b200_gqa_paged_decode_rope", _p(S["q"]), GHQ * GD, _p(S["k_cache"]), _p(S["v_cache"]), kn,
                  vn, sb, sb, _p(S["cos"]), _p(S["sin"]), _p(S["lens"]), _p(S["bt"]), GBT, GB, GHQ, GHKV, GD, GPAGE,
                  65, GSCALE, _p(S["out"]), ws, wsb, _lib.CB_BF16, _st())
        elif kind == "fp8kv":
            _call("chitu_b200_gqa_paged_attn_fp8kv", _p(S["q"]), GHQ * GD, _p(S["k_cache"]), _p(S["v_cache"]), kn,
                  vn, sb, sb, sb, sb, _p(S["cos"]), _p(S["sin"]), _p(S["lens"]), _p(S["bt"]), GBT, GB, 1, GHQ, GHKV,
                  GD, GPAGE, GB * GBT, 65, 1, GSCALE, _p(S["out"]), ws, wsb, _lib.CB_BF16, _st())
        else:
            _call("chitu_b200_gqa_contiguous_attn", _p(S["q"]), _p(S["k_cache"]), _p(S["v_cache"]),
                  G_ROWS_CONTIG * GHKV * GD, G_ROWS_CONTIG, kn, vn, sb, sb, sb, sb, _p(S["lens"]), GB, 1, GHQ, GHKV,
                  GD, 65, 1, GSCALE, _p(S["out"]), ws, wsb, _lib.CB_BF16, _st())
    return read


GQA_WRITERS = {          # writer -> (writes, launch)
    "scatter": (G_ROWS, _gqa_scatter),
    "append": (G_ROW, _gqa_append),
    "multi": (G_ROWS, _gqa_multi),           # seqlen_q > 1: gqa_paged_prefill / gqa_paged_attn_fp8kv / contiguous_attn
    "decode": (G_ROW, _gqa_multi),           # seqlen_q = 1 with k / v: appends row L
}
GQA_READERS = {"paged": ("decode", "decode_rope"), "e4m3": ("fp8kv",), "contig": ("contig",)}
GQA_CASES = [(layout, w, r) for layout, readers in GQA_READERS.items() for w in GQA_WRITERS for r in readers
             if not (layout == "contig" and w == "append")]


@pytest.mark.gpu
@pytest.mark.parametrize("layout,writer,reader", GQA_CASES, ids=["-".join(c) for c in GQA_CASES])
def test_gqa_kv_rows_written_in_flight(slow_row, layout, writer, reader):
    writes, launch = GQA_WRITERS[writer]
    ref = run_case((lambda: _gqa_build(layout, writes, seed=7), launch, _gqa_read(reader)), slow_row)
    assert not torch.isnan(ref["out"].view(BF).float()).any()


# ---------------------------------------------------------------------------------------------------- MLA caches
# B = 2 requests, H = 16 heads (one head group), 64-row pages of 576 elements.  Reader: one decode step with new_kv at
# L_cache = lens, max_seqlen_hint <= 191 -> one split: grid (1, 1, 2) = 2 CTAs; its producer streams every page.
MB, MH, MC, MR, MPAGE, MBT = 2, 16, 512, 64, 64, 4
MROW = MC + MR
M_ROWS = ((32, 70), 32)            # scatter / seqlen_q > 1 writers
M_ROW = ((127, 100), 1)            # append / decode writers: row 127 ends a full page (L % 64 == 63), row 100 is in
                                   # the page that holds the reader's sequence end
MSCALE = 1.0 / math.sqrt(MROW)


def _mla_build(e4m3, writes, seed):
    starts, n = writes
    g = _gen(seed)
    cdt = E4M3 if e4m3 else BF
    nb = MB * MBT
    S = {"bt": torch.randperm(nb, generator=torch.Generator().manual_seed(seed)).to(torch.int32).view(MB, MBT).to(DEV)}
    cache = _ff((nb, MPAGE, MROW), cdt)
    for b in range(MB):
        pos = torch.arange(starts[b], device=DEV)
        _bits(cache).view(-1, MROW)[S["bt"][b].long()[pos // MPAGE] * MPAGE + pos % MPAGE] = \
            _bits(_rand((starts[b], MROW), g, scale=2.0).float().clamp(-448, 448).to(cdt))
    S["kv_cache"] = cache
    S["starts"] = _i32(list(starts))
    S["lens"] = _i32([s + n for s in starts])
    S["src"] = _rand((MB, n, MROW), g)
    S["cu"] = _i32([0, n, 2 * n])
    S["wq_nope"], S["wq_pe"] = _rand((MB, n, MH, MC), g), _rand((MB, n, MH, MR), g)
    S["wout"] = _ff((MB, n, MH, MC), BF)
    S["q_nope"], S["q_pe"] = _rand((MB, MH, MC), g), _rand((MB, MH, MR), g)
    S["new_kv"] = _rand((MB, MROW), g)
    S["out"] = _ff((MB, MH, MC), BF)
    S["ws_bytes"] = int(_lib.load().chitu_b200_attn_workspace_bytes(MB, MH, MC, 4))
    S["ws"] = _ff((S["ws_bytes"],), torch.uint8)
    S["e4m3"] = e4m3
    return S


def _mla_scatter(S):
    n = S["src"].shape[1]
    _call("chitu_b200_scatter_kv", _p(S["kv_cache"]), None, _p(S["src"]), MROW, None, 0, _p(S["cu"]), _p(S["starts"]),
          _p(S["bt"]), MBT, MPAGE, 0, 0, MB, MB * n, MROW, _lib.CB_BF16,
          _lib.CB_FP8_E4M3 if S["e4m3"] else _lib.CB_BF16, _st())


def _mla_append(S):
    if S["e4m3"]:
        _call("chitu_b200_append_paged_kv_e4m3", _p(S["kv_cache"]), _p(S["bt"]), _p(S["src"]), _p(S["starts"]), MB,
              MBT, MROW, _lib.CB_BF16, _st())
    else:
        _call("chitu_b200_append_paged_kv", _p(S["kv_cache"]), _p(S["bt"]), _p(S["src"]), _p(S["starts"]), MB, MBT,
              MPAGE, MPAGE, MROW * 2, _st())


def _mla_multi(S):
    """mla_paged_prefill / mla_attn_fp8kv with seqlen_q = n (no workspace: no split, B x (query tiles) CTAs), or
    mla_decode / mla_attn_fp8kv with seqlen_q = 1 (2 CTAs)."""
    n = S["src"].shape[1]
    if n == 1 and not S["e4m3"]:
        _call("chitu_b200_mla_decode", _p(S["wq_nope"]), _p(S["wq_pe"]), _p(S["kv_cache"]), _p(S["src"]),
              _p(S["starts"]), _p(S["bt"]), MBT, MB, MH, MC, MR, MPAGE, MB * MBT, 191, MSCALE, _p(S["wout"]), None, 0,
              _st())
        return
    name = "chitu_b200_mla_attn_fp8kv" if S["e4m3"] else "chitu_b200_mla_paged_prefill"
    _call(name, _p(S["wq_nope"]), _p(S["wq_pe"]), _p(S["kv_cache"]), _p(S["src"]), _p(S["starts"]), _p(S["bt"]), MBT,
          MB, n, MH, MC, MR, MPAGE, MB * MBT, 191, 1, MSCALE, _p(S["wout"]), None, 0, _st())


def _mla_read(S):
    if S["e4m3"]:
        _call("chitu_b200_mla_attn_fp8kv", _p(S["q_nope"]), _p(S["q_pe"]), _p(S["kv_cache"]), _p(S["new_kv"]),
              _p(S["lens"]), _p(S["bt"]), MBT, MB, 1, MH, MC, MR, MPAGE, MB * MBT, 191, 1, MSCALE, _p(S["out"]),
              _p(S["ws"]), S["ws_bytes"], _st())
    else:
        _call("chitu_b200_mla_decode", _p(S["q_nope"]), _p(S["q_pe"]), _p(S["kv_cache"]), _p(S["new_kv"]),
              _p(S["lens"]), _p(S["bt"]), MBT, MB, MH, MC, MR, MPAGE, MB * MBT, 191, MSCALE, _p(S["out"]), _p(S["ws"]),
              S["ws_bytes"], _st())


MLA_WRITERS = {
    "scatter": (M_ROWS, _mla_scatter),
    "append": (M_ROW, _mla_append),
    "multi": (M_ROWS, _mla_multi),           # seqlen_q > 1: mla_paged_prefill / mla_attn_fp8kv
    "decode": (M_ROW, _mla_multi),           # seqlen_q = 1 with new_kv: mla_decode / mla_attn_fp8kv
}


@pytest.mark.gpu
@pytest.mark.parametrize("writer", list(MLA_WRITERS))
@pytest.mark.parametrize("cache", ["bf16", "e4m3"])
def test_mla_kv_rows_written_in_flight(slow_row, cache, writer):
    writes, launch = MLA_WRITERS[writer]
    ref = run_case((lambda: _mla_build(cache == "e4m3", writes, seed=11), launch, _mla_read), slow_row)
    assert not torch.isnan(ref["out"].view(BF).float()).any()


# ---------------------------------------------------------------------------------------------------- contracts
def _fp8_weight(shape, g):
    return (torch.randn(shape, generator=g, device=DEV) * 40.0).clamp(-448, 448).to(E4M3)


def _dequant(S):
    # weight_dequant_fp8 over the weight's elements as ONE row (M = 1, scales [1, numel / 128]): grid (64, 1, 1) = 64
    # CTAs of 256 threads (the entry caps a row at 64 CTAs; one CTA per weight row would be 256 / 2048 CTAs, several
    # waves, and the reader might only start once the writer is done).  It waits and never triggers early.
    n = S["w8"].numel()
    _call("chitu_b200_weight_dequant_fp8", _p(S["w8"]), _p(S["ws8"]), _p(S["w"]), 1, 1, n, 128, 0, _st())


def _weight_scales(n, g):
    return torch.rand((1, n // 128), generator=g, device=DEV) * 0.01 + 1e-3


def _build_linear():
    g = _gen(21)
    M, N, K = 4, 256, 512
    S = {"w8": _fp8_weight((N, K), g), "ws8": _weight_scales(N * K, g), "w": _ff((N, K), BF), "x": _rand((M, K), g),
         "y": _ff((M, N), BF)}
    S["lws_bytes"] = int(_lib.load().chitu_b200_linear_workspace_bytes(M, N))
    S["lws"] = torch.zeros(S["lws_bytes"], dtype=torch.uint8, device=DEV)
    return S


def _linear(S):
    # the wgmma path (impl = 2): for M = 4, N = 256, K = 512 its grid is 2 CTAs, one 128-row weight tile each, whose 8
    # K stages (of at most 10 in the ring) are all issued before griddepcontrol.wait
    M, K = S["x"].shape
    _call("chitu_b200_linear_bf16", _p(S["x"]), _p(S["w"]), None, None, _p(S["y"]), M, S["w"].shape[0], K,
          _lib.CB_BF16, _p(S["lws"]), S["lws_bytes"], 2, _st())


def _build_absorb():
    g = _gen(22)
    B, H, dn, dv, C = 2, 8, 128, 128, 512
    return {"w8": _fp8_weight((H * (dn + dv), C), g), "ws8": _weight_scales(H * (dn + dv) * C, g),
            "w": _ff((H * (dn + dv), C), BF), "x": _rand((B, H, C), g), "out": _ff((B, H * dv), BF),
            "q_out": _ff((B, H * dv), torch.uint8), "q_scales": _ff((B, H * dv // 128), torch.float32)}


def _absorb(S):
    # mla_absorb_o_quant: grid (H, B / 2) = 8 CTAs; the first rows of wkv_b are requested before griddepcontrol.wait
    B, H, C = S["x"].shape
    _call("chitu_b200_mla_absorb_o_quant", _p(S["x"]), _p(S["w"]), _p(S["out"]), _p(S["q_out"]), _p(S["q_scales"]), B,
          H, 128, 128, C, _st())


def _build_plan():
    """Requests of 1000 and 200 keys at max_seqlen_hint 2048: 16 splits of 64 keys without the plan, 128 with it."""
    g = _gen(23)
    B, H, pages = 2, 16, 16
    nb = B * pages
    S = {"bt": torch.randperm(nb, generator=torch.Generator().manual_seed(23)).to(torch.int32).view(B, pages).to(DEV),
         "kv_cache": _rand((nb, MPAGE, MROW), g, scale=2.0), "lens": _i32([999, 199]), "incl": _i32([1000, 200]),
         "q_nope": _rand((B, H, MC), g), "q_pe": _rand((B, H, MR), g), "new_kv": _rand((B, MROW), g),
         "out": _ff((B, H, MC), BF)}
    S["ws_bytes"] = int(_lib.load().chitu_b200_attn_workspace_bytes(B, H, MC, 16))
    S["ws"] = _ff((S["ws_bytes"],), torch.uint8)
    return S


def _plan(S):
    # attn_plan: one 32-thread CTA; it waits and never triggers early
    _call("chitu_b200_attn_plan", _p(S["incl"]), 2, 16, MPAGE, 2048, _p(S["ws"]), S["ws_bytes"], _st())


def _plan_decode(S):
    # mla_decode: grid (16 splits, 1, 2) = 32 CTAs; the plan words are read before griddepcontrol.wait
    B, pages = S["bt"].shape
    _call("chitu_b200_mla_decode", _p(S["q_nope"]), _p(S["q_pe"]), _p(S["kv_cache"]), _p(S["new_kv"]), _p(S["lens"]),
          _p(S["bt"]), pages, B, 16, MC, MR, MPAGE, B * pages, 2048, MSCALE, _p(S["out"]), _p(S["ws"]), S["ws_bytes"],
          _st())


def _build_prepare(mla):
    """Lengths one short of a page end: decode_prepare advances them by one and opens a new page for request 0 from the
    free-page stack.  The new block-table column first holds another valid page, whose rows differ."""
    g = _gen(24)
    B, bts = 2, 4
    nb = B * bts + 2
    bt = torch.randperm(B * bts, generator=torch.Generator().manual_seed(24)).to(torch.int32).view(B, bts)
    bt[0, 2 if mla else 1] = nb - 2                              # stale entry: a valid page of cached data
    S = {"bt": bt.to(DEV), "free": _i32([0, 0, 0, nb - 1]), "free_count": _i32([4]), "status": _i32([0])}
    S["lens"] = _i32([127, 100] if mla else [63, 47])
    if mla:
        S.update(kv_cache=_rand((nb, MPAGE, MROW), g, scale=2.0), q_nope=_rand((B, MH, MC), g),
                 q_pe=_rand((B, MH, MR), g), new_kv=_rand((B, MROW), g), out=_ff((B, MH, MC), BF))
        S["ws_bytes"] = int(_lib.load().chitu_b200_attn_workspace_bytes(B, MH, MC, 4))
    else:
        S.update(k_cache=_rand((nb, GPAGE, GHKV, GD), g, scale=2.0), v_cache=_rand((nb, GPAGE, GHKV, GD), g, scale=2.0),
                 q=_rand((B, GHQ, GD), g), k_new=_rand((B, GHKV, GD), g), v_new=_rand((B, GHKV, GD), g),
                 out=_ff((B, GHQ, GD), BF))
        S["ws_bytes"] = int(_lib.load().chitu_b200_attn_workspace_bytes(B, GHQ, GD, 8))
    S["ws"] = _ff((S["ws_bytes"],), torch.uint8)
    return S


def _prepare(mla):
    def launch(S):
        # decode_prepare: one 128-thread CTA; it waits and never triggers early
        _call("chitu_b200_decode_prepare", _p(S["lens"]), None, _p(S["bt"]), 4, _p(S["free"]), _p(S["free_count"]),
              _p(S["status"]), 2, MPAGE if mla else GPAGE, 1, _st())
    return launch


def _prepared_decode(mla):
    def read(S):
        # the decode kernels read the lengths (and MLA, before the fix, the block table) before griddepcontrol.wait
        if mla:
            _call("chitu_b200_mla_decode", _p(S["q_nope"]), _p(S["q_pe"]), _p(S["kv_cache"]), _p(S["new_kv"]),
                  _p(S["lens"]), _p(S["bt"]), 4, 2, MH, MC, MR, MPAGE, S["kv_cache"].shape[0], 191, MSCALE,
                  _p(S["out"]), _p(S["ws"]), S["ws_bytes"], _st())
        else:
            _call("chitu_b200_gqa_paged_decode", _p(S["q"]), _p(S["k_cache"]), _p(S["v_cache"]), _p(S["k_new"]),
                  _p(S["v_new"]), GHKV * GD, GHKV * GD, _p(S["lens"]), _p(S["bt"]), 4, 2, GHQ, GHKV, GD, GPAGE, 65,
                  GSCALE, _p(S["out"]), _p(S["ws"]), S["ws_bytes"], _lib.CB_BF16, _st())
    return read


CONTRACTS = {
    "dequant-linear_wgmma": (_build_linear, _dequant, _linear, "y"),
    "dequant-mla_absorb_o": (_build_absorb, _dequant, _absorb, "out"),
    "attn_plan-mla_decode": (_build_plan, _plan, _plan_decode, "out"),
    "decode_prepare-mla_decode": (lambda: _build_prepare(True), _prepare(True), _prepared_decode(True), "out"),
    "decode_prepare-gqa_paged_decode": (lambda: _build_prepare(False), _prepare(False), _prepared_decode(False),
                                        "out"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CONTRACTS))
def test_reads_before_the_wait_after_a_non_triggering_writer(slow_row, case):
    build, writer, reader, out = CONTRACTS[case]
    ref = run_case((build, writer, reader), slow_row)
    assert not torch.isnan(ref[out].view(BF).float()).any()


# ---------------------------------------------------------------------------------------------------- source audit
# Every function of csrc/*.cu that triggers its dependents early (pdl_launch_dependents() itself, or pdl_prologue()) and
# loads global memory before its griddepcontrol.wait: what it reads there, and the test that pins it.  Any other early
# trigger must wait before its first load.
EARLY_READERS = {
    "gqa_decode_mmaT_cta": ("cache_seqlens, and the block table to prefetch its first tiles into L2", "test_reads_before_the_wait_after_a_non_triggering_writer"
                                             "[decode_prepare-gqa_paged_decode]"),
    "mla_decode_cta": ("seqlens_excl, the split plan, and the block table to prefetch its first pages into L2",
                       "test_reads_before_the_wait_after_a_non_triggering_writer[attn_plan-mla_decode], "
                       "[decode_prepare-mla_decode]"),
    "mla_absorb_o_kernel": ("the first rows of wkv_b",
                            "test_reads_before_the_wait_after_a_non_triggering_writer[dequant-mla_absorb_o]"),
    "tc_gemm_kernel": ("the first weight stages (TMA)",
                       "test_reads_before_the_wait_after_a_non_triggering_writer[dequant-linear_wgmma]"),
    "gate_logits_kernel": ("the MoE gate weight rows", "weights written by host copies only (moe_gate takes a bf16 "
                                                       "gate weight that no kernel of the library produces)"),
}
# Kernels whose output a later kernel may read before its own wait: they wait and never trigger early.
NON_TRIGGERING_WRITERS = ("weight_dequant_fp8_kernel", "decode_prepare_kernel", "attn_plan_kernel")

_LOADS = re.compile(r"\b(ld_stream8?|tma_load_\w+|cp_async\w*|__ldg)\s*\(|ld\.global|cp\.async")
_WAIT = re.compile(r"\bpdl_(wait|prologue)\s*\(\s*\)")


def _strip_comments(src):
    src = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _match_brace(src, i, open_="{", close="}"):
    """Index just past the bracket that closes the one at src[i]."""
    depth = 0
    for j in range(i, len(src)):
        if src[j] == open_:
            depth += 1
        elif src[j] == close:
            depth -= 1
            if depth == 0:
                return j + 1
    raise ValueError("unbalanced braces")


def _functions(src):
    """(name, parameter text, body) of every function definition at namespace scope."""
    out = []
    for m in re.finditer(r"\b(\w+)\s*\(([^;{}()]*)\)\s*(?:const\s*)?\{", src):
        name = m.group(1)
        if name in ("if", "for", "while", "switch", "catch", "sizeof", "return") or m.start() == 0:
            continue
        line_start = src.rfind("\n", 0, m.start()) + 1
        if src[line_start:m.start()].startswith((" ", "\t")) and not re.search(r"__global__|__device__",
                                                                             src[max(0, line_start - 200):m.start()]):
            continue
        open_brace = m.end() - 1
        out.append((name, m.group(2), src[open_brace:_match_brace(src, open_brace)]))
    return out


_DEREF = r"(?:^|[=(,;{}?:]|\breturn)\s*\*\s*"       # a unary *: after an operator, a bracket or `return`


def _reads(text, ptrs, structs):
    """True when `text` loads through one of the pointers `ptrs` or a pointer member of one of `structs`: p[i], *p,
    *(p + i), *(const T*)p, a reinterpret_cast of an expression of p that is dereferenced or indexed, s.m[i], *s.m."""
    for p in map(re.escape, ptrs):
        if re.search(r"\b%s\s*\[" % p, text) or re.search(_DEREF + r"\(?\s*%s\b" % p, text, re.M) or \
                re.search(_DEREF + r"\(\s*(?:const\s+)?[\w:]+\s*\*\s*\)\s*\(?\s*%s\b" % p, text, re.M):
            return True
    for s in map(re.escape, structs):
        if re.search(r"\b%s\.\w+\s*\[" % s, text) or re.search(_DEREF + r"\(?\s*%s\.\w+" % s, text, re.M):
            return True
    for m in re.finditer(r"\breinterpret_cast\s*<[^;()]*?>\s*\(", text):
        close = _match_brace(text, m.end() - 1, "(", ")")
        arg = text[m.end():close - 1]
        if not any(re.search(r"\b%s\b" % re.escape(n), arg) for n in set(ptrs) | set(structs)):
            continue
        if re.match(r"\s*(\[|->)", text[close:]) or re.search(_DEREF + r"$", text[:m.start()], re.M):
            return True
    return False


def _loads_before_wait(params, body):
    """True when `body` may load global memory before its griddepcontrol.wait (the first pdl_wait() / pdl_prologue(),
    after pdl_launch_dependents() where the function calls that itself): a load instruction or helper, or a load
    through a pointer parameter or a local pointer derived from one (`_reads`), or a call of a lambda that does either.
    Lambda bodies count where the lambda is called, not where it is defined."""
    trig = re.search(r"\bpdl_launch_dependents\s*\(\s*\)", body)
    m = _WAIT.search(body, trig.end() if trig else 0)
    pre = body[:m.start()] if m else body
    decls = [d.strip() for d in params.split(",")]
    ptrs = {re.findall(r"\w+", d)[-1] for d in decls if "*" in d}
    structs = {re.findall(r"\w+", d)[-1] for d in decls if "*" not in d and re.search(r"\b(Params|PagedAppend)\b", d)}
    # local pointers derived from a pointer parameter
    for lp in re.finditer(r"\*\s*(?:const\s+)?(?:__restrict__\s+)?(\w+)\s*=\s*([^;]*);", pre):
        if any(re.search(r"\b%s\b" % re.escape(p), lp.group(2)) for p in ptrs | structs):
            ptrs.add(lp.group(1))
    loaders = set()
    # lambdas: strip their bodies from the pre-wait text, remembering the ones that load
    while True:
        lm = re.search(r"\bauto\s+(\w+)\s*=\s*\[[^\]]*\]\s*\([^)]*\)[^{;]*\{", pre)
        if not lm:
            break
        end = _match_brace(pre, lm.end() - 1)
        lam = pre[lm.end() - 1:end]
        if _LOADS.search(lam) or _reads(lam, ptrs, structs) or any(re.search(r"\b%s\s*\(" % re.escape(n), lam)
                                                                   for n in loaders):
            loaders.add(lm.group(1))
        pre = pre[:lm.start()] + pre[end:]
    return bool(_LOADS.search(pre) or any(re.search(r"\b%s\s*\(" % re.escape(n), pre) for n in loaders) or
                _reads(pre, ptrs, structs))


def pdl_audit(csrc=None):
    """(early readers, non-triggering writers that trigger or do not wait, missing writers) over csrc/*.cu."""
    csrc = csrc or CSRC
    readers, bad_writers, seen = set(), [], set()
    for fn in sorted(os.listdir(csrc)):
        if not fn.endswith(".cu"):
            continue
        with open(os.path.join(csrc, fn)) as f:
            src = _strip_comments(f.read())
        for name, params, body in _functions(src):
            triggers = re.search(r"\bpdl_launch_dependents\s*\(\s*\)", body) or re.search(r"\bpdl_prologue\s*\(", body)
            if name in NON_TRIGGERING_WRITERS:
                seen.add(name)
                if triggers or not re.search(r"\bpdl_wait\s*\(\s*\)", body):
                    bad_writers.append(name)
                continue
            if triggers and _loads_before_wait(params, body):
                readers.add(name)
    return readers, bad_writers, sorted(set(NON_TRIGGERING_WRITERS) - seen)


def test_pdl_source_audit():
    readers, bad_writers, missing = pdl_audit()
    assert not missing, f"non-triggering writers not found in csrc: {missing}"
    assert not bad_writers, f"these writers must wait and never trigger their dependents early: {bad_writers}"
    assert readers == set(EARLY_READERS), (
        f"early-triggering functions that load before griddepcontrol.wait: {sorted(readers)}; the table lists "
        f"{sorted(EARLY_READERS)}.  A new one needs a case here whose writer cannot still be in flight.")
