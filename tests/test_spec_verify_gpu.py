"""The speculative verify step of the LLaMA engine on the GPU.

1. The greedy acceptance kernel, bit exact against the Python rule, eager and replayed from a graph.
2. PDL ordering: a decode step launched directly after the acceptance kernel (which writes seq_lens, read by the decode
   kernels before their griddepcontrol.wait) equals the same step after a synchronise.
3. The verify step against fp64, teacher-forced per layer with the method and bound of test_engine_steps_gpu: the layer
   is recomputed over the B * (k + 1) rows from the engine's own input to it and the cache as it was, with causal
   attention over the cache and the k + 1 new rows; exactly the rows seq_len .. seq_len + k of each request change in
   every layer, each within one storage rounding of the reference's; graph replay equals eager, and rewinding seq_lens
   and replaying reproduces the step.
4. Agreement with sequential greedy decode, and a wrong draft is rejected at its position with the rejected rows
   invisible to the next decode step.
"""
import dataclasses

import pytest
import torch
import torch.nn.functional as Fn

import test_engine_steps_gpu as ES
import torch_ref as R
from test_fp8_rowwise_cpu import quant_rowwise

BF, F8, F64 = torch.bfloat16, torch.float8_e4m3fn, torch.float64
DEV = "cuda:0"
K = 3
BATCH = 5
PAGE = 256
MAX_SEQ = 4 * PAGE + 4
# length 0 and 1; a page boundary inside the k + 1 rows; mid-page; the last k + 1 positions of max_seq_len
STARTS = [0, 1, PAGE - 2, 2 * PAGE + 7, MAX_SEQ - (K + 1)]


# ----------------------------------------------------------------------------------------------- acceptance kernel
def accept_rule(target, drafts, n_draft, seq_lens):
    B, k1 = target.shape
    out = torch.full((B, k1), -1, dtype=torch.int64)
    acc = torch.zeros(B, dtype=torch.int32)
    nxt = torch.zeros(B, dtype=torch.int64)
    lens = seq_lens.clone()
    for b in range(B):
        a = 0
        while a < int(n_draft[b]) and int(drafts[b, a]) == int(target[b, a]):
            a += 1
        out[b, :a + 1] = target[b, :a + 1]
        acc[b], nxt[b] = a, target[b, a]
        lens[b] += a + 1
    return out, acc, nxt, lens


def accept_case(B, k, seed):
    """Targets and drafts whose first mismatch runs over every position 0..k (k: all match), and n_draft over 0..k,
    with rows of all-accepted (n_draft = k, no mismatch) and none-accepted (mismatch at 0) included."""
    g = torch.Generator().manual_seed(seed)
    target = torch.randint(0, 128256, (B, k + 1), generator=g)
    drafts = target[:, :k].clone()
    first_bad = torch.arange(B) % (k + 1)
    n_draft = (torch.arange(B) // (k + 1)) % (k + 1)
    n_draft[0], first_bad[0] = k, k                  # all accepted
    if B > 1:
        n_draft[1], first_bad[1] = k, 0              # none accepted
    for b in range(B):
        if first_bad[b] < k:
            # the drafts after the first mismatch still match: they must not count
            drafts[b, first_bad[b]] = (target[b, first_bad[b]] + 1 + b) % 128256
    seq_lens = torch.randint(0, 4096, (B,), generator=g, dtype=torch.int32)
    return target, drafts, n_draft.to(torch.int32), seq_lens


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 7, 64, 129, 256])
@pytest.mark.parametrize("k", [1, 2, 4, 7, 15])
def test_acceptance_bit_exact(B, k):
    from chitu_b200.ops import accept_draft_tokens_greedy as acc
    target, drafts, n_draft, seq_lens = accept_case(B, k, seed=B * 31 + k)
    want = accept_rule(target, drafts, n_draft, seq_lens)
    t, d, n, s = (x.to(DEV) for x in (target, drafts, n_draft, seq_lens))
    got = acc(t, d, n, s)
    torch.cuda.synchronize()
    for gv, wv, name in zip(got + (s,), want, ("out_tokens", "accepted", "next_tokens", "seq_lens")):
        assert torch.equal(gv.cpu(), wv), name
    # graph replay equals eager
    s.copy_(seq_lens.to(DEV))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = acc(t, d, n, s)
    s.copy_(seq_lens.to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    for gv, wv in zip(static + (s,), want):
        assert torch.equal(gv.cpu(), wv)


# ------------------------------------------------------------------------------------------------------- engines
@dataclasses.dataclass(frozen=True)
class Variant:
    engine_kw: tuple = ()

    @property
    def kw(self):
        return dict(self.engine_kw)

    @property
    def fp8_weights(self):
        return self.kw.get("weight_format") == "fp8"


VARIANTS = {
    "bf16": Variant(),
    "e4m3_kv": Variant((("kv_dtype", F8),)),
    "w4a16": Variant((("weight_format", "w4a16"),)),
    "fp8": Variant((("weight_format", "fp8"),)),
    "fp8_e4m3_kv": Variant((("weight_format", "fp8"), ("kv_dtype", F8))),
    "tp2_shard": Variant((("tp_size", 2),)),
}


def make_engine(kw, batch=BATCH, starts=STARTS, max_draft=K):
    from chitu_b200.engine import LlamaConfig, LlamaDecodeEngine
    cfg = LlamaConfig(dim=512, n_layers=3, n_heads=4, n_kv_heads=2, vocab_size=1024, multiple_of=256,
                      ffn_dim_multiplier=None)
    eng = LlamaDecodeEngine(cfg, max_reqs=batch, max_seq_len=MAX_SEQ, device=DEV, page_size=PAGE, max_draft=max_draft,
                            **kw)
    g = torch.Generator(device=eng.device).manual_seed(5)
    for w in [L[k] for L in eng.layers for k in ("attn_norm", "ffn_norm")] + [eng.norm]:
        w.copy_(0.5 + torch.rand(w.shape, generator=g, device=eng.device))
    eng.set_synthetic_context(0)
    eng.seq_lens.copy_(torch.tensor(starts, dtype=torch.int32))
    return eng


def verify_inputs(eng, seed):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(0, eng.cfg.vocab_size, (eng.B,), generator=g)
    drafts = torch.randint(0, eng.cfg.vocab_size, (eng.B, eng.max_draft), generator=g)
    n = torch.arange(eng.B, dtype=torch.int32) % (eng.max_draft + 1)
    return tok.pin_memory(), drafts.pin_memory(), n.pin_memory()


def fp8_lin(x, w, cd):
    q, s = quant_rowwise(x)
    return ((q.to(cd) * s.to(cd)[:, None]) @ w.to(cd).T).to(x.dtype)


def ref_verify_layer(eng, lw, h, k_cache, v_cache, lens, cos, sin, sq, cd=F64, fp8=False):
    """One LLaMA layer over B * sq rows (row b * sq + i at position lens[b] + i), in `cd`, rounding where the engine
    stores: the k / v rows are appended to the caches (cloned by the caller) and each query i of request b attends the
    keys 0 .. lens[b] + i."""
    lin = (lambda x, w: fp8_lin(x, w, cd)) if fp8 else (lambda x, w: R._lin(x, w, cd))
    Hq, Hkv, eps, page = eng.Hq, eng.Hkv, eng.cfg.norm_eps, eng.page
    M = h.shape[0]
    B = M // sq
    D = lw["wqkv"].shape[0] // (Hq + 2 * Hkv)
    g = Hq // Hkv
    qkv = lin(R.rms_norm(h, lw["attn_norm"], eps, cd), lw["wqkv"])
    q = qkv[:, :Hq * D].reshape(M, Hq, D)
    k = qkv[:, Hq * D:(Hq + Hkv) * D].reshape(M, Hkv, D)
    v = qkv[:, (Hq + Hkv) * D:].reshape(M, Hkv, D)
    q, k = R.rotary_interleaved(q, k, cos, sin, cd)
    o = torch.empty(M, Hq * D, dtype=h.dtype, device=h.device)
    table = eng.block_table
    for b, L in enumerate(lens.tolist()):
        for i in range(sq):
            p, r = L + i, b * sq + i
            blk = table[b, p // page].long()
            k_cache[blk, p % page] = R.store_rows(k[r], k_cache.dtype)
            v_cache[blk, p % page] = R.store_rows(v[r], v_cache.dtype)
        n = L + sq
        n_pages = (n + page - 1) // page
        kk = k_cache[table[b, :n_pages].long()].reshape(n_pages * page, Hkv, D)[:n].to(cd)
        vv = v_cache[table[b, :n_pages].long()].reshape(n_pages * page, Hkv, D)[:n].to(cd)
        qb = (q[b * sq:(b + 1) * sq].to(cd) / D ** 0.5).view(sq, Hkv, g, D)
        s = torch.einsum("ikgd,skd->ikgs", qb, kk)
        mask = torch.arange(n, device=h.device)[None, :] > (L + torch.arange(sq, device=h.device))[:, None]
        s = s.masked_fill(mask[:, None, None, :], float("-inf"))
        out = torch.einsum("ikgs,skd->ikgd", torch.softmax(s, dim=-1), vv)
        o[b * sq:(b + 1) * sq] = out.reshape(sq, Hq * D).to(h.dtype)
    h = h + lin(o, lw["wo"])
    gu = lin(R.rms_norm(h, lw["ffn_norm"], eps, cd), lw["w13"])
    F = gu.shape[1] // 2
    return h + lin(Fn.silu(gu[:, :F]) * gu[:, F:], lw["w2"])


def verify_mask(cache, table, lens, sq, page):
    mask = torch.zeros(cache.shape[0], cache.shape[1], dtype=torch.bool, device=cache.device)
    for b, L in enumerate(lens.tolist()):
        for p in range(L, L + sq):
            mask[int(table[b, p // page]), p % page] = True
    return mask


def check_rows(after, before, ref_after, table, lens, sq, page, upstream=2.0 ** -8):
    """Exactly the rows seq_len .. seq_len + sq - 1 of every request changed; the largest distance of a written value
    from the reference's, in units of one storage rounding (test_engine_steps_gpu.check_append's measure)."""
    mask = verify_mask(after, table, lens, sq, page)
    nb, pg = after.shape[0], after.shape[1]
    a, b = after.view(torch.uint8).reshape(nb, pg, -1), before.view(torch.uint8).reshape(nb, pg, -1)
    assert torch.equal(a[~mask], b[~mask]), "a cache row outside seq_len .. seq_len + k changed"
    got = after.reshape(nb, pg, -1)[mask].double()
    want = ref_after.reshape(nb, pg, -1)[mask].double()
    rel = 2.0 ** -3 if after.dtype == F8 else 2.0 ** -8
    tol = rel * torch.maximum(got.abs(), want.abs()) + upstream * want.abs().amax(dim=-1, keepdim=True) + 2.0 ** -9
    return ((got - want).abs() / tol).max().item()


def same_state(a, b, what):
    for name in ("logits", "target", "out_tokens", "accepted", "next_tokens", "seq_lens"):
        x, y = getattr(a, name), getattr(b, name)
        assert torch.equal(x.view(torch.int16) if x.dtype == BF else x, y.view(torch.int16) if y.dtype == BF else y), \
            f"{what}: {name} differs"
    for ca, cb in zip(a.caches, b.caches):
        assert torch.equal(ca.view(torch.uint8), cb.view(torch.uint8)), f"{what}: KV cache bytes differ"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VARIANTS))
def test_verify_step(name):
    v = VARIANTS[name]
    A, G = make_engine(v.kw), make_engine(v.kw)
    G.capture_verify()
    for ca, cg in zip(A.caches, G.caches):         # capture_verify()'s warm-up steps wrote cache rows
        ca.copy_(cg)
    sq, n_layers = K + 1, len(A.layers)
    layers = A.ref_layers()
    gen = torch.Generator(device=DEV).manual_seed(9)
    tok, drafts, n = verify_inputs(A, seed=1)
    lens = A.seq_lens.clone()
    before = [[c[li].clone() for c in A.caches] for li in range(n_layers)]
    A.capture_h = []
    out_a, acc_a = A.verify(tok, drafts, n)
    hs, A.capture_h = A.capture_h, None
    out_g, acc_g = G.verify(tok, drafts, n)
    torch.cuda.synchronize()
    same_state(A, G, "graph vs eager")
    # rewind and replay
    first = (G.logits.clone(), [c.clone() for c in G.caches], out_g.clone())
    G.seq_lens.copy_(lens)
    again, _ = G.verify(tok, drafts, n)
    torch.cuda.synchronize()
    assert torch.equal(again, first[2]) and torch.equal(G.logits.view(torch.int16), first[0].view(torch.int16))
    assert all(torch.equal(c.view(torch.uint8), f.view(torch.uint8)) for c, f in zip(G.caches, first[1]))
    # acceptance of the engine's own argmax
    M = A.B * sq
    assert torch.equal(A.target.view(-1), A.logits[:M].float().argmax(dim=-1)), "target is not the first maximal index"
    want = accept_rule(A.target.cpu(), drafts, n, lens.cpu())
    assert torch.equal(out_a, want[0]) and torch.equal(acc_a, want[1]) and torch.equal(A.seq_lens.cpu(), want[3])
    # every layer, teacher-forced, against fp64; the written KV rows
    pos = (lens.long()[:, None] + torch.arange(sq, device=DEV)).view(-1)
    cos, sin = A.cos_table[pos], A.sin_table[pos]
    worst_kv, worst = 0.0, (0.0, 0.0)
    failures = []
    for li in range(n_layers):
        h = hs[li][:M]
        caches = [c.clone() for c in before[li]]
        ref = ref_verify_layer(A, layers[li], h, *caches, lens, cos, sin, sq, fp8=v.fp8_weights)
        for after, b4, r in zip((c[li] for c in A.caches), before[li], caches):
            worst_kv = max(worst_kv, check_rows(after, b4, r, A.block_table, lens, sq, A.page))
        floor = 0.0
        d_ref = ref.double() - h.double()
        for _ in range(ES.FLOOR_SEEDS):
            hp = ES.ulp_perturb(h, gen)
            outp = ref_verify_layer(A, layers[li], hp, *[c.clone() for c in before[li]], lens, cos, sin, sq,
                                    fp8=v.fp8_weights)
            floor = max(floor, ES.rel_err(outp.double() - hp.double(), d_ref))
        err = ES.rel_err(hs[li + 1][:M].double() - h.double(), d_ref)
        worst = max(worst, (err, floor))
        if err > ES.bound(floor):
            failures.append(f"layer {li}: err {err:.3e} > bound {ES.bound(floor):.3e} (floor {floor:.3e})")
    ref = R.final_logits(hs[-1][:M], A.norm, A.head, A.cfg.norm_eps, F64)
    err = ES.rel_err(A.logits[:M].double(), ref)
    floor = max(ES.rel_err(R.final_logits(ES.ulp_perturb(hs[-1][:M], gen), A.norm, A.head, A.cfg.norm_eps, F64), ref)
                for _ in range(ES.FLOOR_SEEDS))
    if err > ES.bound(floor):
        failures.append(f"logits: err {err:.3e} > bound {ES.bound(floor):.3e} (floor {floor:.3e})")
    print(f"{name}: worst layer err {worst[0]:.3e} (floor {worst[1]:.3e})  logits err {err:.3e} (floor {floor:.3e})"
          f"  written KV {worst_kv:.2f} roundings  launches {G.launches_per_verify}")
    assert worst_kv <= 1.0, f"a written KV value is {worst_kv:.2f} roundings from the reference's"
    assert not failures, "\n".join(failures)


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True])
def test_decode_directly_after_acceptance(graph):
    """The acceptance kernel writes seq_lens; the decode step launched right behind it equals the same step after a
    synchronise, bit for bit."""
    from chitu_b200.ops import accept_draft_tokens_greedy as acc
    engs = [make_engine({}), make_engine({})]
    if graph:
        for e in engs:
            e.capture()
    for ca, cb in zip(*(e.caches for e in engs)):
        cb.copy_(ca)
    engs[1].seq_lens.copy_(engs[0].seq_lens)
    target, drafts, n_draft, _ = accept_case(BATCH, K, seed=3)
    target, drafts, n_draft = (x.to(DEV) for x in (target, drafts, n_draft))
    tok = torch.randint(0, 1024, (BATCH,), generator=torch.Generator().manual_seed(4)).pin_memory()
    for i, e in enumerate(engs):
        torch.cuda.synchronize()
        e.tokens.copy_(tok)
        acc(target, drafts, n_draft, e.seq_lens)
        if i == 1:
            torch.cuda.synchronize()
        e.step()
    torch.cuda.synchronize()
    a, b = engs
    assert torch.equal(a.seq_lens, b.seq_lens)
    assert torch.equal(a.next_tokens, b.next_tokens)
    assert torch.equal(a.logits.view(torch.int16), b.logits.view(torch.int16))
    for ca, cb in zip(a.caches, b.caches):
        assert torch.equal(ca.view(torch.uint8), cb.view(torch.uint8))


# ------------------------------------------------------------------------------------ agreement with greedy decode
AGREE_B = 16
AGREE_STARTS = [0, 1, PAGE - 2, PAGE + 3, 2 * PAGE - 1, 300, 600, 17, 5, 700, 900, 2 * PAGE + 100, 64, 128, 450,
                MAX_SEQ - (K + 2)]
MARGIN = 2 * ES.C_MIN        # a top-2 logit gap, relative to the row's largest |logit|, no rounding difference can flip


def snapshot(e):
    return e.seq_lens.clone(), [c.clone() for c in e.caches]


def restore(e, snap):
    e.seq_lens.copy_(snap[0])
    for c, s in zip(e.caches, snap[1]):
        c.copy_(s)


def greedy_run(e, tok, steps):
    """`steps` greedy decode steps from tok: the tokens emitted, and each step's relative top-2 margin per request."""
    toks, margins = [], []
    for _ in range(steps):
        tok = e.decode(tok.pin_memory())
        lg = e.logits[:e.B].double()
        top = lg.topk(2, dim=-1)[0]
        margins.append(((top[:, 0] - top[:, 1]) / lg.abs().amax(dim=-1)).cpu())
        toks.append(tok)
    return torch.stack(toks, dim=1), torch.stack(margins, dim=1)


@pytest.mark.gpu
@pytest.mark.parametrize("kv", ["bf16", "e4m3"])
def test_agreement_with_sequential_decode(kv):
    kw = dict(kv_dtype=F8) if kv == "e4m3" else {}
    e = make_engine(kw, batch=AGREE_B, starts=AGREE_STARTS)
    snap = snapshot(e)
    t0 = torch.randint(0, 1024, (AGREE_B,), generator=torch.Generator().manual_seed(7))
    seq, margins = greedy_run(e, t0, K + 1)                    # s_1 .. s_{k+1}
    restore(e, snap)
    n_all = torch.full((AGREE_B,), K, dtype=torch.int32)
    out, acc = e.verify(t0.pin_memory(), seq[:, :K].pin_memory(), n_all.pin_memory())
    sure = (margins > MARGIN).all(dim=1)
    assert int(sure.sum()) >= 1, "no request has a clear greedy path: the test checks nothing"
    assert bool((acc[sure] == K).all()), acc
    assert torch.equal(out[sure], seq[sure])
    assert torch.equal(e.seq_lens.cpu()[sure], snap[0].cpu()[sure] + K + 1)
    for b in range(AGREE_B):                                   # every request: a prefix of the greedy path
        a = int(acc[b])
        assert torch.equal(out[b, :a], seq[b, :a]) and bool((out[b, a + 1:] == -1).all())
    # a wrong draft at position j: j accepted; the next decode step sees only the accepted tokens
    s_eng = make_engine(kw, batch=AGREE_B, starts=AGREE_STARTS, max_draft=0)
    for j in range(K):
        restore(e, snap)
        restore(s_eng, snap)
        drafts = seq[:, :K].clone()
        drafts[:, j] = (drafts[:, j] + 1) % 1024
        out, acc = e.verify(t0.pin_memory(), drafts.pin_memory(), n_all.pin_memory())
        sure_j = (margins[:, :j + 1] > MARGIN).all(dim=1)
        assert bool((acc[sure_j] == j).all()), (j, acc)
        assert torch.equal(out[sure_j, :j + 1], seq[sure_j, :j + 1])
        assert torch.equal(e.seq_lens.cpu()[sure_j], snap[0].cpu()[sure_j] + j + 1)
        nxt = e.next_tokens.cpu()
        e.decode(nxt.pin_memory())
        # the engine that was only ever given the accepted tokens: t0, s_1 .. s_{j+1}
        tok = t0
        for i in range(j + 2):
            s_eng.decode(tok.pin_memory())
            tok = seq[:, i] if i <= j else tok
        torch.cuda.synchronize()
        rows = sure_j.to(DEV)
        assert torch.equal(e.seq_lens[rows], s_eng.seq_lens[rows])
        err = ES.rel_err(e.logits[:AGREE_B].double()[rows], s_eng.logits[:AGREE_B].double()[rows])
        print(f"{kv}: wrong draft at {j}: {int(sure_j.sum())} requests checked, next-step logits err {err:.3e}")
        assert err <= ES.C_MIN, f"wrong draft at {j}: the next decode step differs by {err:.3e}"
