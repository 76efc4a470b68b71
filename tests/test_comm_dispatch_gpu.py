"""The tensor-parallel reduce (csrc/comm.cu) and the push epilogues that feed it, on one GPU: the pull kernel
`allreduce_norm_kernel` at W = 1, the push consumer `allreduce_consume_kernel` at W = 1 ... 8, the GEMM push epilogue
(`tc_gemm_kernel<KIND_16 | KIND_FP8, BN, EPI_PUSH>`) and the push branch of `moe_combine_kernel` at W = 1, a CUDA graph
of two produce + consume layers, and the producers at W = 2 and 4 as processes sharing one GPU over CUDA IPC.

None of this needs a second GPU.  At W = 1 the pull kernel waits only on the flag it has just set itself and the
producers write only into their own push area.  The consumer reads only its own rank's area, which `comm_create` sizes
for `world` sources, so a communicator created as (rank 0, world W) and never connected can be consumed once the test
has written all W sources' words itself (`chitu_b200_debug_comm_push_area` gives the area and the call counter).  Before
every consume the host checks that each word the consumer will poll already carries the epoch, so a producer that
misses a word fails as an assertion instead of a consumer waiting for it.

Reference.  h = bf16(bf16(fp32 sum over ranks r = 0 .. W-1, in order, of partial_r) + residual), the first rounding
only without a residual, compared bit for bit.  Ranks 0 and 1 commute (the sum starts from 0); every later adjacent pair
is pinned by a column holding 1, 2^24, -2^24 at ranks r - 1, r, r + 1, which sums to 0 in rank order and to 1 with r
and r + 1 swapped.  y is checked against the fp64 RMSNorm of the reference h with the RMSNorm bound of
`test_step_ops_dispatch_gpu` (n = 8 per vector of 8 elements a thread owns, 5 butterfly levels, one per warp partial);
q / qs bit for bit against `act_quant_deepseek_v3` of the kernel's own y, and the q-only run against the run that also
writes y.  The pushed GEMM words are checked against the fp64 GEMM with `test_gemm_dispatch_gpu`'s bound, and after a
consume with a residual h equals the plain entry given the same residual bit for bit: both compute
bf16(bf16(v) + residual) over the same schedule.  The expert-combine push equals `chitu_b200_fused_experts` likewise.
`test_bound_rejects_injected_errors` shows on the host that these checks reject a dropped source, the sources summed in
reverse order, the residual added before the first rounding, a dropped eps, words in the wrong slot or with the wrong
epoch, and the scales of the neighbouring group."""
import ctypes
import os
import tempfile
import traceback

import pytest
import torch

from oracle import chitu_oracle as O
from test_gemm_dispatch_gpu import (SENTINEL, TICKET_BYTES, U_OUT, Call, Padded, _case_table, _ratio, _reference,
                                    _schedule, _split_case, _tau, _to_device, _workspace)
from test_gemm_dispatch_gpu import _operands as _gemm_operands
from test_moe_dispatch_gpu import WCODE, WMODES, FusedCall, _fresh_ws, _moe_path
from test_moe_dispatch_gpu import _operands as _moe_operands
from test_step_ops_dispatch_gpu import EPS, bound, ratio, rms_ref

BF, F32 = torch.bfloat16, torch.float32
DEV = "cuda:0"
POISON = 0xFF                  # a word of these bytes carries epoch 0xffffffff, which no reduce reaches
TIMEOUT_S = "10"               # a consumer that never sees its words traps after this, instead of after 600 s
PULL_THREADS, CONSUME_THREADS = 256, 512
# output modes: (h, y, q)
MODES = {"h": (1, 0, 0), "y": (0, 1, 0), "h+y": (1, 1, 0), "h+y+q": (1, 1, 1), "q": (0, 0, 1)}


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------- references and checks
def h_ref(parts, res=None):
    """bf16(bf16(fp32 sum of parts in list order) + res) (no res: the first rounding only)"""
    s = torch.zeros(parts[0].shape, dtype=F32, device=parts[0].device)
    for p in parts:
        s = s + p.float()
    h = s.to(BF)
    return h if res is None else (h.float() + res.float()).to(BF)


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16).cpu(), b.contiguous().view(torch.int16).cpu())


def rms_terms(dim, threads):
    """levels of fp32 additions in a reduce kernel's sum of squares"""
    return 8 * _cdiv(dim, 8 * threads) + 5 + threads // 32


def y_ratio(y, h, w, threads):
    ref, acc = rms_ref(h.double(), w.double().to(h.device), EPS, rms_terms(h.shape[-1], threads))
    return ratio(y, ref, bound(ref, acc, BF))


def q_matches(q, qs, y):
    """q (uint8) / qs == act_quant_deepseek_v3 of y, bit for bit"""
    qo, so = O.act_quant_deepseek_v3(y.cpu())
    return torch.equal(qs.cpu(), so) and torch.equal(q.cpu(), qo.view(torch.uint8))


def words_ready(words, slot, world, n, epoch):
    """words: int32 [2 slots, sources, 2 * words] of a push area; the first n words of every source in `slot` carry
    `epoch`"""
    return bool((words[slot, :world, 1:2 * n:2] == epoch).all())


def order_rows(world, dim, g, device="cpu"):
    """[world, dim] bf16 partial rows: column r - 1 (1 <= r <= world - 2) holds 1, 2^24, -2^24 at ranks r - 1, r, r + 1
    and 0 elsewhere, the remaining columns random"""
    p = torch.randn(world, dim, generator=g).to(BF)
    for r in range(1, world - 1):
        p[:, r - 1] = 0
        p[r - 1, r - 1], p[r, r - 1], p[r + 1, r - 1] = 1.0, 2.0 ** 24, -2.0 ** 24
    return p.to(device)


def sources(world, rows, dim, seed, device="cpu"):
    """W partials [rows, dim] and a residual; rows of three magnitudes (the smallest makes eps matter), row 0 pinning
    the rank order"""
    g = torch.Generator().manual_seed(seed)
    sc = torch.tensor((1e-3, 1.0, 30.0)).repeat(_cdiv(rows, 3))[:rows, None]
    parts = [(torch.randn(rows, dim, generator=g) * sc).to(BF) for _ in range(world)]
    res = (torch.randn(rows, dim, generator=g) * sc).to(BF)
    o = order_rows(world, dim, g)
    for r in range(world):
        parts[r][0] = o[r]
    return [p.to(device) for p in parts], res.to(device)


# ------------------------------------------------------------------------- injected-error self-test of the checks
def test_bound_rejects_injected_errors():
    """The checks admit the reference and reject each injected error."""
    names = set()
    for world in (3, 5, 8):
        parts, res = sources(world, 6, 512, seed=world)
        want = h_ref(parts, res)
        assert same_bits(want, h_ref(parts, res))
        assert not same_bits(want, h_ref(parts[:-1], res))
        names.add("a dropped source")
        assert not same_bits(want, h_ref(parts[::-1], res))
        names.add("sources in reverse order")
        for r in range(1, world - 1):                                   # every adjacent swap but ranks 0 and 1
            swapped = parts[:r] + [parts[r + 1], parts[r]] + parts[r + 2:]
            assert not same_bits(want, h_ref(swapped, res)), r
        s = torch.zeros(6, 512)
        for p in parts:
            s = s + p.float()
        assert not same_bits(want, (s + res.float()).to(BF))
        names.add("residual before the first rounding")
        # RMSNorm of h: the correctly rounded y passes, y without eps does not
        w = (torch.rand(512, generator=torch.Generator().manual_seed(world)) + 0.5).to(BF)
        hd = want.double()
        ref, _ = rms_ref(hd, w.double(), EPS, 0)
        for threads in (PULL_THREADS, CONSUME_THREADS):
            assert y_ratio(ref.to(BF), want, w, threads) <= 1.0
            no_eps = hd / torch.sqrt((hd * hd).mean(-1, keepdim=True)) * w.double()
            assert y_ratio(no_eps.to(BF), want, w, threads) > 1.0
        names.add("eps dropped")
        y = ref.to(BF)
        qo, so = O.act_quant_deepseek_v3(y)
        q = qo.view(torch.uint8)
        assert q_matches(q, so, y)
        assert not q_matches(q, torch.roll(so, 1, dims=1), y)
        names.add("scales of the neighbouring group")
    # the words of a push area: the right slot and epoch pass, the other slot or epoch - 1 do not
    n, calls = 100, 6
    slot = calls & 1
    for world in (1, 4):
        area = torch.full((2, world, 2 * n + 8), -1, dtype=torch.int32)
        area[slot, :, 1:2 * n:2] = calls + 1
        assert words_ready(area, slot, world, n, calls + 1)
        other = torch.full_like(area, -1)
        other[1 - slot, :, 1:2 * n:2] = calls + 1
        assert not words_ready(other, slot, world, n, calls + 1)
        names.add("the wrong slot")
        stale = area.clone()
        stale[slot, :, 1:2 * n:2] = calls
        assert not words_ready(stale, slot, world, n, calls + 1)
        names.add("the wrong epoch")
        short = area.clone()
        short[slot, world - 1, 2 * n - 1] = -1                          # the last word of the last source missing
        assert not words_ready(short, slot, world, n, calls + 1)
    assert names == {"a dropped source", "sources in reverse order", "residual before the first rounding",
                     "eps dropped", "scales of the neighbouring group", "the wrong slot", "the wrong epoch"}


# ---------------------------------------------------------------------------------------------------- GPU calls
def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def _last_error():
    return _lib().chitu_b200_last_error().decode(errors="replace")


def _ok(rc, what):
    assert rc == 0, (what, rc, _last_error())


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class _DeviceMemory:
    """a device allocation the library owns, as a torch tensor (no copy)"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3,
                                         "strides": None}


class Comm:
    """A communicator; `area` is its push area as bytes [2 slots, world sources, source bytes], `words` the same as
    int32 [2, world, 2 * words per source] (data, epoch)."""

    def __init__(self, rank, world, slot_bytes):
        lib = _lib()
        h = ctypes.c_void_p()
        self.ipc = (ctypes.c_uint8 * 128)()
        old = os.environ.get("CHITU_B200_COMM_TIMEOUT_S")
        os.environ["CHITU_B200_COMM_TIMEOUT_S"] = TIMEOUT_S
        try:
            _ok(lib.chitu_b200_comm_create(rank, world, slot_bytes, ctypes.byref(h), self.ipc), "comm_create")
        finally:
            if old is None:
                del os.environ["CHITU_B200_COMM_TIMEOUT_S"]
            else:
                os.environ["CHITU_B200_COMM_TIMEOUT_S"] = old
        self.h, self.world = h.value, world
        area, nb, calls = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_void_p()
        _ok(lib.chitu_b200_debug_comm_push_area(self.h, ctypes.byref(area), ctypes.byref(nb), ctypes.byref(calls)),
            "debug_comm_push_area")
        assert nb.value >= 2 * slot_bytes
        self.source_bytes = nb.value
        self.area = torch.as_tensor(_DeviceMemory(area.value, 2 * world * nb.value), device=DEV).view(2, world, -1)
        self.words = self.area.view(torch.int32)
        self.calls_t = torch.as_tensor(_DeviceMemory(calls.value, 4), device=DEV).view(torch.int32)

    def calls(self):
        return int(self.calls_t.item())

    def status(self):
        return int(_lib().chitu_b200_comm_status(self.h))

    def write(self, slot, src, part, epoch):
        """the words of a bf16 partial [rows, dim] as source `src` of `slot`"""
        n = part.numel() // 2
        w = self.words[slot, src, :2 * n].view(n, 2)
        w[:, 0] = part.to(DEV).contiguous().view(torch.int32).view(-1)
        w[:, 1] = epoch

    def pushed(self, calls, rows, dim):
        """the partial a producer pushed for the reduce after `calls`: all rows * dim / 2 words of source 0 in slot
        calls & 1 carry the epoch, nothing else of the (poisoned) area was written"""
        n, slot = rows * dim // 2, calls & 1
        assert words_ready(self.words, slot, 1, n, calls + 1), "a pushed word is missing or has the wrong epoch"
        assert bool((self.area[slot, 0, 8 * n:] == POISON).all()), "written past the partial"
        assert bool((self.area[1 - slot] == POISON).all()), "written into the other slot"
        return self.words[slot, 0, 0:2 * n:2].contiguous().view(BF).view(rows, dim)

    def consume(self, res, outs, w, rows, dim):
        return _lib().chitu_b200_allreduce_consume(self.h, _ptr(res), *outs.ptrs(w), rows, dim, EPS, _stream())

    def close(self):
        if self.h:
            _lib().chitu_b200_comm_destroy(self.h)
            self.h = None


def _out(shape, dtype):
    return Padded(torch.empty(shape, dtype=dtype), pad=SENTINEL, fill=SENTINEL)


class Outs:
    """the outputs of one reduce in sentinel-padded buffers (None where the mode leaves them out)"""

    def __init__(self, rows, dim, mode):
        h, y, q = MODES[mode]
        self.mode = mode
        self.h = _out((rows, dim), BF) if h else None
        self.y = _out((rows, dim), BF) if y else None
        self.q = _out((rows, dim), torch.uint8) if q else None
        self.qs = _out((rows, dim // 128), F32) if q else None

    def ptrs(self, w):
        v = lambda P: None if P is None else _ptr(P.view)        # noqa: E731
        return v(self.h), (None if self.y is None and self.q is None else _ptr(w)), v(self.y), v(self.q), v(self.qs)

    def check(self, want_h, w, threads, what, with_y=None):
        """pads intact, h bit exact, y inside the bound, q / qs those of act_quant of y (of `with_y`'s y for q only)"""
        for P in (self.h, self.y, self.q, self.qs):
            assert P is None or P.pads_intact(), ("pad overwritten",) + what
        if self.h is not None:
            assert same_bits(self.h.view, want_h), ("h differs",) + what
        if self.y is not None:
            r = y_ratio(self.y.view, want_h, w, threads)
            assert r <= 1.0, ("y outside the bound", r) + what
        if self.q is not None and self.y is not None:
            assert q_matches(self.q.view, self.qs.view, self.y.view), ("q / qs differ",) + what
        if self.q is not None and self.y is None:
            assert torch.equal(self.q.view, with_y.q.view) and torch.equal(self.qs.view, with_y.qs.view), \
                ("q-only run differs from the run with y",) + what


def _norm_w(dim, seed):
    g = torch.Generator().manual_seed(seed)
    return Padded((torch.rand(dim, generator=g) + 0.5).to(BF)).view


# ------------------------------------------------------------------------------------------ pull kernel, W = 1
PULL_DIMS = (8, 264, 512, 4096, 7168, 8192)
PULL_ROWS = (1, 2, 17, 255, 256)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", PULL_DIMS)
def test_pull_kernel_world1(dim):
    """chitu_b200_allreduce_residual_rmsnorm at W = 1 in every output mode, with and without a residual; each mode is
    five back-to-back calls of different row counts, so the per-row call counters diverge and rows of one call use
    different slots."""
    lib = _lib()
    comm = Comm(0, 1, max(PULL_ROWS) * dim * 2)
    try:
        w = _norm_w(dim, dim)
        modes = [m for m in MODES if dim % 256 == 0 or not MODES[m][2]]
        for residual in (False, True):
            inputs = {}
            for rows in PULL_ROWS:
                parts, res = sources(1, rows, dim, seed=rows * 31 + dim, device=DEV)
                inputs[rows] = (Padded(parts[0]), Padded(res) if residual else None)
            runs = {}
            for mode in modes:
                for rows in PULL_ROWS:
                    P, R = inputs[rows]
                    outs = Outs(rows, dim, mode)
                    _ok(lib.chitu_b200_allreduce_residual_rmsnorm(comm.h, _ptr(P.view), R and _ptr(R.view),
                                                                  *outs.ptrs(w), rows, dim, EPS, _stream()),
                        "allreduce_residual_rmsnorm")
                    runs[(mode, rows)] = outs
            torch.cuda.synchronize()
            for (mode, rows), outs in runs.items():
                P, R = inputs[rows]
                assert P.pads_intact()
                want = h_ref([P.view], None if R is None else R.view)
                outs.check(want, w, PULL_THREADS, ("pull", dim, rows, mode, residual), runs.get(("h+y+q", rows)))
            assert comm.status() == 0
        assert comm.status() == 0
    finally:
        comm.close()


# ------------------------------------------------------------------------------ consumer on W sources the test wrote
# (rows, dim, mode, residual); a q-only step follows the step with y on the same inputs
CONSUME_SEQ = ((1, 8, "h", False), (3, 264, "h+y", True), (2, 512, "h+y+q", False), (2, 512, "q", False),
               (17, 4096, "y", True), (255, 8192, "h+y+q", True), (255, 8192, "q", True), (256, 7168, "h+y+q", False),
               (256, 7168, "h", True))


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8])
def test_consumer_sums_the_sources_in_rank_order(world):
    """chitu_b200_allreduce_consume on an unconnected (0, W) communicator whose area the test filled: the slot the
    reduce reads holds the W partials with its epoch, the other slot different data with the previous epoch.  h is the
    rank-ordered sum bit for bit (row 0 pins the order across the 4-source batches at W = 5 and 8), the call counter
    advances by one per consume whatever the grid, and rows = 0 launches nothing."""
    from chitu_b200._lib import launch_count
    comm = Comm(0, world, 256 * 8192 * 2)
    try:
        last = None
        for i, (rows, dim, mode, residual) in enumerate(CONSUME_SEQ):
            parts, res = sources(world, rows, dim, seed=rows * 7 + dim + world, device=DEV)
            decoy, _ = sources(world, rows, dim, seed=rows * 7 + dim + world + 1, device=DEV)
            R = Padded(res) if residual else None
            w = _norm_w(dim, dim + 1)
            n0 = comm.calls()
            slot = n0 & 1
            for r in range(world):
                comm.write(slot, r, parts[r], n0 + 1)
                comm.write(1 - slot, r, decoy[r], n0)
            torch.cuda.synchronize()
            assert words_ready(comm.words, slot, world, rows * dim // 2, n0 + 1)
            outs = Outs(rows, dim, mode)
            _ok(comm.consume(R and R.view, outs, w, rows, dim), "allreduce_consume")
            torch.cuda.synchronize()
            assert comm.calls() == n0 + 1, (rows, dim, mode)
            outs.check(h_ref(parts, res if residual else None), w, CONSUME_THREADS, ("consume", world, i, rows, dim,
                                                                                     mode, residual), last)
            assert comm.status() == 0
            last = outs
        n0, before = comm.calls(), launch_count()
        outs = Outs(1, 512, "h")
        assert comm.consume(None, outs, None, 0, 512) == 0
        torch.cuda.synchronize()
        assert comm.calls() == n0 and launch_count() == before and bool((outs.h.buf == SENTINEL).all())
        assert comm.status() == 0
    finally:
        comm.close()


# ------------------------------------------------------------------------------------------ refusals of both reduces
SHAPE_CHECK = "rows >= 0 && rows <= kMaxRows && dim > 0 && dim % 8 == 0 && dim <= 8192"
# entry -> (its C name, its first check)
REDUCE_ENTRIES = {"pull": ("chitu_b200_allreduce_residual_rmsnorm", "handle && partial && " + SHAPE_CHECK),
                  "consume": ("chitu_b200_allreduce_consume", "handle && " + SHAPE_CHECK)}
# (arguments changed from a valid 16 x 512 call with every output, the failed check; None: the entry's first check)
REDUCE_REFUSALS = (
    (dict(handle=None), None), (dict(partial=None), None), (dict(rows=-1), None), (dict(rows=257), None),
    (dict(dim=0), None), (dict(dim=12), None), (dict(dim=8200), None),
    (dict(h=None, norm_w=None, y=None, q=None, qs=None), "h_out || norm_w"),
    (dict(qs=None), "(q == nullptr) == (q_scales == nullptr)"),
    (dict(q=None), "(q == nullptr) == (q_scales == nullptr)"),
    (dict(dim=264), "q == nullptr || (norm_w && dim % 256 == 0)"),
    (dict(norm_w=None, y=None), "q == nullptr || (norm_w && dim % 256 == 0)"),
    (dict(rows=17), "(int64_t)rows * dim * 2 <= c->slot_bytes"),
)


@pytest.mark.gpu
def test_reduce_refusals_launch_nothing():
    """Both reduce entries refuse each bad argument with -1 and the message of the check that failed, under the entry's
    own name; nothing is launched or written, and the call counter stays.  rows = 0 returns 0 and launches nothing."""
    from chitu_b200._lib import launch_count
    lib = _lib()
    comm = Comm(0, 1, 16 * 512 * 2)
    try:
        n = 257 * 8200                                           # elements of the widest refused shape
        bufs = {k: torch.full((n,), -1, dtype=torch.int32, device=DEV) for k in ("partial", "res", "h", "norm_w", "y",
                                                                                   "q", "qs")}
        comm.area.fill_(POISON)
        torch.cuda.synchronize()
        before = launch_count()
        for entry, (name, first) in REDUCE_ENTRIES.items():
            for change, check in REDUCE_REFUSALS + ((dict(rows=0), 0),):
                if entry == "consume" and "partial" in change:
                    continue
                a = dict(handle=comm.h, rows=16, dim=512, **{k: _ptr(t) for k, t in bufs.items()})
                a.update(change)
                if entry == "pull":
                    rc = lib.chitu_b200_allreduce_residual_rmsnorm(a["handle"], a["partial"], a["res"], a["h"],
                                                                   a["norm_w"], a["y"], a["q"], a["qs"], a["rows"],
                                                                   a["dim"], EPS, _stream())
                else:
                    rc = lib.chitu_b200_allreduce_consume(a["handle"], a["res"], a["h"], a["norm_w"], a["y"], a["q"],
                                                          a["qs"], a["rows"], a["dim"], EPS, _stream())
                if check == 0:
                    assert rc == 0, (entry, change, _last_error())
                else:
                    assert rc == -1, (entry, change, rc)
                    want = f"{name}: argument check failed: {first if check is None else check}"
                    assert _last_error() == want, (entry, change, _last_error())
        torch.cuda.synchronize()
        assert launch_count() == before
        assert all(bool((t == -1).all()) for t in bufs.values())
        assert bool((comm.area == POISON).all()) and comm.calls() == 0 and comm.status() == 0
    finally:
        comm.close()


# --------------------------------------------------------------------------------------- GEMM push epilogues, W = 1
def _push_gemm(call, comm, ws, nbytes=None):
    """the _ar entry of a G Call's operands (no bias, no residual)"""
    lib = _lib()
    nb = ws.numel() if nbytes is None else nbytes
    if call.kind == "16":
        return lib.chitu_b200_linear_bf16_ar(_ptr(call.x.view), _ptr(call.w.view), call.M, call.N, call.K, comm.h,
                                             _ptr(ws), nb, _stream())
    return lib.chitu_b200_fp8_gemm_ar(_ptr(call.x.view), _ptr(call.a_s), _ptr(call.w.view), _ptr(call.b_s), call.M,
                                      call.N, call.K, comm.h, _ptr(ws), nb, _stream())


def _gemm_push_cases(kind, sms):
    cases = [(M, N, K) for k, M, N, K, _ in _case_table(sms) if k == kind]
    return cases + [(M, N, {"16": 1024, "fp8": 512}[kind]) for N in (8, 200, 1000) for M in (1, 33, 129)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["16", "fp8"])
def test_gemm_push_epilogue_world1(kind):
    """Every (BN x stream-K regime) case of the GEMM case table and N tails through linear_bf16_ar / fp8_gemm_ar at
    W = 1: exactly the M * N / 2 words of one slot are written, with the epoch, inside the fp64 GEMM bound; consumed with
    a residual, h equals the plain entry's output with that residual bit for bit."""
    sms = _sms()
    comm = Comm(0, 1, 256 * 8192 * 2)
    cells, worst = set(), 0.0
    try:
        for M, N, K in _gemm_push_cases(kind, sms):
            sc = _schedule(kind, M, N, K, sms)
            cells |= {(sc["BN"], r) for r in sc["regimes"]}
            op = _gemm_operands(kind, M, N, K, seed=M * 7919 + N + K)
            ref, rss = _reference(_to_device(op), bias=False)
            call = Call(op)
            ws = _workspace(M, N)
            comm.area.fill_(POISON)
            n0 = comm.calls()
            _ok(_push_gemm(call, comm, ws), (kind, M, N, K))
            torch.cuda.synchronize()
            what = (kind, M, N, K)
            assert call.x.pads_intact() and call.w.pads_intact(), what
            assert int(ws[:TICKET_BYTES].count_nonzero()) == 0, ("tickets left non-zero",) + what
            got = comm.pushed(n0, M, N)
            r = _ratio(got, ref, rss, U_OUT[BF], _tau(kind, 2))
            assert r <= 1.0, ("pushed partial outside the bound", r) + what
            worst = max(worst, r)
            res = torch.randn(M, N, generator=torch.Generator().manual_seed(N + M)).to(BF)
            R, outs = Padded(res), Outs(M, N, "h")
            _ok(comm.consume(R.view, outs, None, M, N), "allreduce_consume")
            torch.cuda.synchronize()
            assert comm.calls() == n0 + 1, what
            plain = Call(op, residual=res).run(2, ws)
            torch.cuda.synchronize()
            assert outs.h.pads_intact() and same_bits(outs.h.view, plain), ("TP h differs from the plain entry",) + what
            assert comm.status() == 0, what
        assert comm.status() == 0
    finally:
        comm.close()
    assert cells == {(bn, r) for k, _, _, _, cs in _case_table(sms) if k == kind for bn, r in cs}
    print(f"[comm bound] push kind={kind} max|y-ref|/bound={worst:.3f}")


@pytest.mark.gpu
def test_push_refusals_launch_nothing():
    """SIMT-only shapes and a workspace one byte short return -2 from the path choice; odd N, M * N * 2 past the slot
    and an expert shape off the grouped path are refused too.  Nothing is launched, the areas and the call counters
    stay as they were."""
    from chitu_b200._lib import launch_count
    lib = _lib()
    comm, small = Comm(0, 1, 1 << 20), Comm(0, 1, 256)
    try:
        for c in (comm, small):
            c.area.fill_(POISON)
        torch.cuda.synchronize()
        before = launch_count()
        k16 = Call(_gemm_operands("16", 4, 128, 16, seed=1))
        k16.K = 12                                               # rows of 24 bytes: no TMA
        fp8_tail = Call(_gemm_operands("fp8", 16, 300, 400, seed=2))
        fine = Call(_gemm_operands("16", 17, 384, 1024, seed=3))
        ws = _workspace(17, 384)
        need = _lib().chitu_b200_linear_workspace_bytes(17, 384)
        assert _push_gemm(k16, comm, ws) == -2
        assert _push_gemm(fp8_tail, comm, ws) == -2
        assert _push_gemm(fine, comm, ws, need - 1) == -2 and "wgmma path unavailable" in _last_error()
        assert _push_gemm(fine, small, ws) == -1 and "argument check" in _last_error()       # 17 * 384 * 2 > 256
        odd = Call(_gemm_operands("16", 1, 129, 256, seed=4))
        assert _push_gemm(odd, comm, ws) == -1
        for N1, T in ((384, 6), (256, 200)):                     # off the grouped path; T * K1 * 2 past the slot
            case = dict(wmode="bf16", T=T, topk=2, E=4, N1=N1, K1=256, routing="random", na=None,
                        ids_dtype=torch.int32, tw_dtype=BF, residual=False, seed=5, cell=None)
            f = FusedCall(_moe_operands(case))
            mws = _fresh_ws(lib.chitu_b200_moe_workspace_bytes(T, 2, 4, N1, 256))
            target = comm if T == 6 else small
            rc = _experts_ar(f, target, mws)
            assert rc == (-2 if T == 6 else -1), (N1, T, rc, _last_error())
        torch.cuda.synchronize()
        assert launch_count() == before
        for c in (comm, small):
            assert bool((c.area == POISON).all()) and c.calls() == 0
    finally:
        comm.close()
        small.close()


# ------------------------------------------------------------------------------------ expert-combine push, W = 1
def _experts_ar(f, comm, ws):
    c = f.c
    from chitu_b200._lib import dtype_code
    return _lib().chitu_b200_fused_experts_ar(
        _ptr(f.x.view), _ptr(f.w1), _ptr(f.w2), _ptr(f.w1_s), _ptr(f.w2_s), _ptr(f.tw), dtype_code(f.tw.dtype),
        _ptr(f.ids), dtype_code(f.ids.dtype), c["T"], c["topk"], c["E"], c["N1"], c["K1"], WCODE[c["wmode"]], comm.h,
        _ptr(ws), ws.numel(), _stream())


MOE_T = (1, 3, 16, 64, 200)


def _moe_case(wmode, T, i, seed):
    return dict(wmode=wmode, T=T, topk=3, E=8, N1=256, K1=256, routing="random", na=None,
                ids_dtype=(torch.int32, torch.int64)[i % 2], tw_dtype=(BF, F32)[i % 2], residual=True, seed=seed,
                cell=None)


@pytest.mark.gpu
@pytest.mark.parametrize("wmode", WMODES)
def test_expert_combine_push_world1(wmode):
    """fused_experts_ar at W = 1, with dropped pairs (pos < 0): the pushed words equal fused_experts without a residual,
    and after a consume with a residual h equals fused_experts with it, bit for bit."""
    lib = _lib()
    comm = Comm(0, 1, max(MOE_T) * 256 * 2)
    try:
        for i, T in enumerate(MOE_T):
            case = _moe_case(wmode, T, i, seed=7000 + 10 * i + WCODE[wmode])
            assert _moe_path(T, 3, 8, 256, 256, wmode) == "grouped"
            op = _moe_operands(case)
            assert T == 1 or bool((op["ids"] < 0).any())
            with_res, plain = FusedCall(op), FusedCall(dict(op, res=None))
            nbytes = lib.chitu_b200_moe_workspace_bytes(T, 3, 8, 256, 256)
            want_h = with_res.run(_fresh_ws(nbytes)).clone()
            want_p = plain.run(_fresh_ws(nbytes)).clone()
            comm.area.fill_(POISON)
            plain.out.view.view(torch.uint8).fill_(0xFF)
            n0 = comm.calls()
            _ok(_experts_ar(plain, comm, _fresh_ws(nbytes)), ("fused_experts_ar", wmode, T))
            torch.cuda.synchronize()
            assert same_bits(comm.pushed(n0, T, 256), want_p), ("pushed partial differs", wmode, T)
            assert bool((plain.out.view.view(torch.int16) == -1).all())          # `out` is not written
            outs = Outs(T, 256, "h")
            _ok(comm.consume(with_res.res.view, outs, None, T, 256), "allreduce_consume")
            torch.cuda.synchronize()
            assert comm.calls() == n0 + 1
            assert outs.h.pads_intact() and same_bits(outs.h.view, want_h), ("TP h differs", wmode, T)
            assert comm.status() == 0
        assert comm.status() == 0
    finally:
        comm.close()


# ------------------------------------------------------------------------------------------------ CUDA graph replay
@pytest.mark.gpu
def test_two_layers_in_a_cuda_graph():
    """linear_bf16_ar -> consume -> fp8_gemm_ar -> consume captured once and replayed three times with new inputs:
    every replay equals the eager calls bit for bit (h also equals the plain entries), and the call counter advances by
    two per replay."""
    sms = _sms()
    shapes = [("16",) + _split_case("16", sms, "slot1", 64), ("fp8",) + _split_case("fp8", sms, "slot1", 64)]
    comm = Comm(0, 1, max(M * N for _, M, N, _ in shapes) * 2)
    try:
        layers = []
        for j, (kind, M, N, K) in enumerate(shapes):
            call = Call(_gemm_operands(kind, M, N, K, seed=50 + j))
            res = Padded(torch.zeros(M, N, dtype=BF))
            outs = Outs(M, N, "h+y+q" if N % 256 == 0 else "h+y")
            layers.append((call, res, outs, _norm_w(N, 60 + j)))
        ws = torch.zeros(max(_lib().chitu_b200_linear_workspace_bytes(M, N) for _, M, N, _ in shapes),
                         dtype=torch.uint8, device=DEV)

        def step(check=False):
            """both layers; with `check` (eager only) the host sees every pushed word before the consume"""
            for call, res, outs, w in layers:
                n0 = comm.calls() if check else None
                _ok(_push_gemm(call, comm, ws), "push")
                if check:
                    torch.cuda.synchronize()
                    assert words_ready(comm.words, n0 & 1, 1, call.M * call.N // 2, n0 + 1), ("words missing", call.kind)
                _ok(comm.consume(res.view, outs, w, call.M, call.N), "consume")

        ops = {}

        def load(i):
            for j, (call, res, outs, _) in enumerate(layers):
                op = ops[j] = _gemm_operands(call.kind, call.M, call.N, call.K, seed=100 * i + j)
                call.x.view.copy_(op["x"].to(DEV))
                call.w.view.copy_(op["w"].to(DEV))
                for name in ("a_s", "b_s"):
                    if getattr(call, name) is not None:
                        getattr(call, name).copy_(op[name].to(DEV))
                res.view.copy_(torch.randn(call.M, call.N, generator=torch.Generator().manual_seed(i + j)).to(BF))

        def snapshot():
            return [[P.view.clone() for P in (outs.h, outs.y, outs.q, outs.qs) if P is not None]
                    for _, _, outs, _ in layers]

        eager = []
        for i in range(1, 4):
            load(i)
            step(check=True)
            torch.cuda.synchronize()
            eager.append(snapshot())
            for j, ((call, res, outs, w), got) in enumerate(zip(layers, eager[-1])):
                plain = Call(ops[j], residual=res.view).run(2, ws)
                torch.cuda.synchronize()
                assert same_bits(got[0], plain), call.kind
                outs.check(got[0], w, CONSUME_THREADS, ("graph eager", call.kind, i))
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step()                                               # warm-up off the capture
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        for i, want in zip(range(1, 4), eager):
            load(i)
            for _, _, outs, _ in layers:
                for P in (outs.h, outs.y, outs.q, outs.qs):
                    if P is not None:
                        P.view.view(torch.uint8).fill_(0xFF)
            torch.cuda.synchronize()
            n0 = comm.calls()
            graph.replay()
            torch.cuda.synchronize()
            assert comm.calls() == n0 + 2
            for (call, _, outs, _), ref in zip(layers, want):
                got = [P.view for P in (outs.h, outs.y, outs.q, outs.qs) if P is not None]
                assert all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(got, ref)), \
                    ("replay differs from the eager calls", call.kind, i)
                assert all(P is None or P.pads_intact() for P in (outs.h, outs.y, outs.q, outs.qs))
        assert comm.status() == 0 and int(ws[:TICKET_BYTES].count_nonzero()) == 0
    finally:
        comm.close()


# ------------------------------------------------------------------------- producers of W ranks on one GPU, over IPC
MP_LINEAR = (33, 1024, 512)          # M, N, K of every rank's row-parallel linear
MP_EXPERTS_T = 16


def _mp_worker(rank, world, store_path, out_dir):
    """One rank: connect over IPC, push a linear (and at W = 2 an expert block), check that every source's words are
    present, consume, and save h beside the plain-entry partials.  Host barriers separate produce and consume."""
    import torch.distributed as dist
    out = os.path.join(out_dir, f"rank{rank}.pt")
    comm = None
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", store=dist.FileStore(store_path, world), rank=rank, world_size=world)
        lib = _lib()
        M, N, K = MP_LINEAR
        comm = Comm(rank, world, max(M * N, MP_EXPERTS_T * 256) * 2)
        blobs = [None] * world
        dist.all_gather_object(blobs, bytes(comm.ipc))
        blob = b"".join(blobs)
        rc = lib.chitu_b200_comm_connect(comm.h, (ctypes.c_uint8 * len(blob)).from_buffer_copy(blob))
        errs = [None] * world
        dist.all_gather_object(errs, "" if rc == 0 else _last_error())
        if any(errs):
            torch.save({"ipc_refused": [e for e in errs if e]}, out)
            return
        dist.barrier()
        result = {}

        def reduce(name, produce, rows, dim, seed):
            n0 = comm.calls()
            _ok(produce(), name)
            torch.cuda.synchronize()
            dist.barrier()                                       # every rank's words have landed
            ready = [None] * world
            dist.all_gather_object(ready, words_ready(comm.words, n0 & 1, world, rows * dim // 2, n0 + 1))
            result[name + "_ready"] = ready
            if not all(ready):
                return
            res = torch.randn(rows, dim, generator=torch.Generator().manual_seed(seed)).to(BF)
            outs = Outs(rows, dim, "h")
            _ok(comm.consume(Padded(res).view, outs, None, rows, dim), "consume")
            torch.cuda.synchronize()
            result[name + "_calls"] = comm.calls() - n0
            result[name + "_h"] = outs.h.view.cpu()
            result[name + "_res"] = res

        call = Call(_gemm_operands("16", M, N, K, seed=300 + rank))
        ws = _workspace(M, N)
        reduce("linear", lambda: _push_gemm(call, comm, ws), M, N, 11)
        result["linear_part"] = call.run(2, ws).cpu()
        dist.barrier()
        if world == 2:
            T = MP_EXPERTS_T
            case = _moe_case("fp8", T, rank, seed=400 + rank)
            f = FusedCall(dict(_moe_operands(case), res=None))
            nbytes = lib.chitu_b200_moe_workspace_bytes(T, 3, 8, 256, 256)
            reduce("experts", lambda: _experts_ar(f, comm, _fresh_ws(nbytes)), T, 256, 12)
            result["experts_part"] = f.run(_fresh_ws(nbytes)).cpu()
            dist.barrier()
        result["status"] = comm.status()
        torch.save(result, out)
        dist.barrier()                                           # no rank frees its area while a peer still reads it
    except Exception:
        torch.save({"error": traceback.format_exc()}, out)
        raise
    finally:
        if comm is not None:
            comm.close()
        if dist.is_initialized():
            dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_producers_across_processes(world):
    """W processes on one GPU connected over CUDA IPC, each pushing its partial into every rank's area: every source is
    present with the epoch before the consume, h is byte-identical on every rank and equals the rank-ordered sum of
    the ranks' plain-entry partials plus the residual."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_mp_worker, args=(r, world, os.path.join(tmp, "store"), tmp)) for r in range(world)]
        try:
            for p in procs:
                p.start()
            for p in procs:
                p.join(300)
            results = []
            for r in range(world):
                path = os.path.join(tmp, f"rank{r}.pt")
                assert os.path.exists(path), (f"rank {r} wrote no result", [p.exitcode for p in procs])
                results.append(torch.load(path))
        finally:
            for p in procs:
                if p.is_alive():
                    p.kill()
                p.join(10)
    for r, res in enumerate(results):
        assert "error" not in res, (r, res.get("error"))
    if "ipc_refused" in results[0]:
        pytest.skip("cudaIpcOpenMemHandle refused a handle of the same device: " + results[0]["ipc_refused"][0])
    assert [p.exitcode for p in procs] == [0] * world
    for name in ("linear", "experts") if world == 2 else ("linear",):
        for r, res in enumerate(results):
            assert res[name + "_ready"] == [True] * world, (name, r, res[name + "_ready"])
            assert res[name + "_calls"] == 1, (name, r)
        want = h_ref([res[name + "_part"] for res in results], results[0][name + "_res"])
        for r, res in enumerate(results):
            assert same_bits(res[name + "_h"], results[0][name + "_h"]), (name, "h differs between ranks", r)
            assert same_bits(res[name + "_h"], want), (name, "h differs from the rank-ordered sum", r)
    assert all(res["status"] == 0 for res in results)
