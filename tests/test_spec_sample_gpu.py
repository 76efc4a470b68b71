"""Sampled verification of speculative drafts on the GPU.

1. chitu_b200_spec_accept_sampled against the fp64 rule of test_spec_sample_cpu, with the slack of
   test_step_ops_dispatch_gpu's sample_rule / check_draw: every acceptance decision that clears its slack equals the
   rule's, every draw lies in its CDF interval, greedy requests equal the greedy rule exactly.
2. The same two chi-square properties as the CPU test, on 2^16 requests with identical rows and device uniforms.
3. With no drafts, the drawn token equals chitu_b200_sample_top_k_top_p's, bit for bit.
4. The engine: an all-greedy batch equals the greedy verify step bit for bit (outputs, seq_lens, logits, KV bytes), a
   mixed batch on its greedy requests; the engine's tail against the rule; graph replay and rewound replay.
5. PDL ordering: the entry directly after the kernel that writes its logits, and a decode step directly after the entry,
   equal the same launches with a synchronise between them.
"""
import math

import pytest
import torch

import test_spec_verify_gpu as SV
from test_spec_sample_cpu import V_STAT, stat_check, stat_rows
from test_step_ops_dispatch_gpu import check_draw, sample_rule

DEV = "cuda:0"
F32 = torch.float32
U_TOP = 0.99999994                  # the largest float below 1


def _dtype(name):
    return {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}[name]


def make_case(B, k, V, dtype, dense, seed):
    """Requests cycling through T in {0, 0.05, 1}, top_k in {0, 1, 50, -3}, top_p in {0.3, 1}, uniforms including 0
    and the largest float below 1, rows with -inf logits, drafts at the argmax, at random and outside the kept set, and
    (dense) q(d) = 0 and q >= p (a residual of zero mass).  Logits have a padded row stride."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    gc = torch.Generator().manual_seed(seed)
    R = B * (k + 1)
    base = torch.randn(R, V + 5, generator=g, device=DEV) * 3
    for r in range(0, R, 3):                                     # -inf on every third row, never on its maximum
        m = torch.rand(V, generator=g, device=DEV) < 0.4
        m[int(torch.argmax(base[r, :V]))] = False
        base[r, :V][m] = -math.inf
    logits = base.to(dtype)[:, :V]
    Ts, tks, tps = [0.0, 0.05, 1.0], [0, 1, 50, -3], [0.3, 1.0]
    T = torch.tensor([Ts[b % 3] for b in range(B)], dtype=F32)
    top_k = torch.tensor([min(tks[(b // 3) % 4], V) for b in range(B)], dtype=torch.int32)
    top_p = torch.tensor([tps[(b // 2) % 2] for b in range(B)], dtype=F32)
    n = torch.tensor([(b * 7 + 3) % (k + 1) for b in range(B)], dtype=torch.int32)
    n[0] = k
    am = logits.float().argmax(dim=1).view(B, k + 1).cpu()
    drafts = torch.randint(0, V, (B, k), generator=gc)
    use_am = torch.rand(B, k, generator=gc) < 0.6
    drafts = torch.where(use_am, am[:, :k], drafts)
    ua = torch.rand(B, k, generator=gc)
    ud = torch.rand(B, generator=gc)
    ua.view(-1)[::5], ua.view(-1)[1::7], ud[::4], ud[1::5] = 0.0, U_TOP, 0.0, U_TOP
    q = None
    if dense:
        q = torch.softmax(torch.randn(B, k, V, generator=g, device=DEV), dim=-1)
        for b in range(B):
            if b % 4 == 1:                                       # q(d) = 0
                q[b, 0, int(drafts[b, 0])] = 0.0
            if b % 4 == 2:          # q = p / max p >= the renormalised p: a residual of zero mass when rejected
                p = torch.softmax(logits[b * (k + 1)].float() / max(float(T[b]), 1e-3), dim=0)
                q[b, 0] = p / p.max()
                ua[b, 0] = 0.75
    return dict(logits=logits, drafts=drafts.to(DEV), n_draft=n.to(DEV), temperatures=T.to(DEV),
                top_ks=top_k.to(DEV), top_ps=top_p.to(DEV), u_accept=ua.to(DEV), u_draw=ud.to(DEV), draft_probs=q)


def check_against_rule(case, seq_before, out, acc, nxt, seq_after):
    """(checked acceptance decisions, checked draws); asserts on every clear disagreement"""
    lg = case["logits"].double().cpu()
    B, k = case["drafts"].shape
    V = lg.shape[1]
    drafts, n_draft = case["drafts"].cpu(), case["n_draft"].cpu()
    T, tk, tp = case["temperatures"].cpu(), case["top_ks"].cpu(), case["top_ps"].cpu()
    ua, ud = case["u_accept"].cpu(), case["u_draw"].cpu()
    q = None if case["draft_probs"] is None else case["draft_probs"].cpu()
    out, acc, nxt = out.cpu(), acc.cpu(), nxt.cpu()
    assert torch.equal(seq_after.cpu(), seq_before.cpu() + acc + 1)
    n_dec = n_draw = 0
    for b in range(B):
        n, a = int(n_draft[b]), int(acc[b])
        assert 0 <= a <= n
        assert torch.equal(out[b, :a], drafts[b, :a]) and int(out[b, a]) == int(nxt[b])
        assert bool((out[b, a + 1:] == -1).all())
        rows = lg[b * (k + 1): (b + 1) * (k + 1)]
        if float(T[b]) <= 0:                                     # greedy: exact
            am = [int(torch.argmax(rows[i].float())) for i in range(k + 1)]
            want = 0
            while want < n and int(drafts[b, want]) == am[want]:
                want += 1
            assert a == want and int(nxt[b]) == am[a], (b, a, want)
            n_dec += 1
            continue
        top_k = int(tk[b]) if int(tk[b]) > 0 else V
        rules = [sample_rule(rows[i], float(T[b]), top_k, float(tp[b]), V) for i in range(n + 1)]
        sure = True
        for i in range(n + 1):
            p, must, may, _, _ = rules[i]
            z_lo, z_hi = float(p[must].sum()), float(p[may].sum())
            if i == n:
                break
            d = int(drafts[b, i])
            qd = 1.0 if q is None else float(q[b, i, d])
            x = float(ua[b, i]) * qd
            lo = float(p[d]) / z_hi if bool(must[d]) else 0.0
            hi = float(p[d]) / z_lo if bool(may[d]) else 0.0
            if x < lo * (1 - 1e-5) - 1e-30 and lo > 0:
                clear = "accept"
            elif x >= hi * (1 + 1e-5) or hi == 0:
                clear = "reject"
            else:
                sure = False
                break
            n_dec += 1
            if clear == "reject":
                assert a == i, (b, i, a, "rule rejects")
                break
            assert a > i, (b, i, a, "rule accepts")
        if not sure:
            continue
        p, must, may, _, delta_d = rules[a]
        u = float(ud[b])
        tok = int(nxt[b])
        if a == n:
            check_draw(p, must, may, tok, u, delta_d)
            n_draw += 1
            continue
        if not bool((must == may).all()):
            continue                                             # the kept set itself is uncertain: no residual check
        pk = torch.where(must, p, 0.0) / float(p[must].sum())
        if q is None:
            qa = torch.zeros(V, dtype=torch.float64)
            qa[int(drafts[b, a])] = 1.0
        else:
            qa = q[b, a].double()
        r = (pk - qa).clamp(min=0)
        zr = float(r.sum())
        if zr == 0:
            check_draw(p, must, may, tok, u, delta_d)
        elif zr > 1e-3:
            c = torch.cumsum(r, 0)
            before, upto = float(c[tok] - r[tok]), float(c[tok])
            slack = 1e-4 * zr
            assert before <= u * zr + slack and upto >= u * zr - slack, (b, tok, before, upto, u * zr)
        else:
            continue
        n_draw += 1
    return n_dec, n_draw


def run_entry(case, seq_lens):
    from chitu_b200.ops import accept_draft_tokens_sampled as acc
    return acc(case["logits"], case["drafts"], case["n_draft"], seq_lens, case["temperatures"], case["top_ks"],
               case["top_ps"], case["u_accept"], case["u_draw"], draft_probs=case["draft_probs"])


CASES = [  # (B, k, V, dtype, dense)
    (1, 1, 7, "fp32", False), (1, 15, 1000, "bf16", True), (7, 3, 1025, "fp16", False), (16, 7, 1000, "fp32", True),
    (32, 7, 128256, "bf16", False), (12, 4, 128256, "bf16", True), (128, 1, 1025, "bf16", True),
    (256, 1, 7, "fp16", False), (16, 15, 1025, "bf16", False), (64, 3, 1000, "fp32", True)]


@pytest.mark.gpu
@pytest.mark.parametrize("case_id", range(len(CASES)))
def test_entry_against_rule(case_id):
    B, k, V, dt, dense = CASES[case_id]
    case = make_case(B, k, V, _dtype(dt), dense, seed=case_id + 1)
    seq0 = torch.randint(0, 4096, (B,), dtype=torch.int32, device=DEV)
    seq = seq0.clone()
    out, acc, nxt = run_entry(case, seq)
    torch.cuda.synchronize()
    n_dec, n_draw = check_against_rule(case, seq0, out, acc, nxt, seq)
    print(f"B {B} k {k} V {V} {dt} {'dense' if dense else 'token-only'}: {n_dec} decisions, {n_draw} draws checked")
    assert n_dec >= B // 2 and n_draw >= B // 4
    # graph replay equals eager
    seq2 = seq0.clone()
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        static = run_entry(case, seq2)
    seq2.copy_(seq0)
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(static + (seq2,), (out, acc, nxt, seq)):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_distribution_on_device(dense):
    """2^16 requests with the CPU test's rows: first tokens ~ p_0, second tokens after an accepted d_0 ~ p_1"""
    from chitu_b200.ops import accept_draft_tokens_sampled as acc
    p, q = stat_rows(dense)
    B, k = 1 << 16, 2
    g = torch.Generator(device=DEV).manual_seed(17)
    # logits log p (cut entries -inf): at T = 1 with no top-k / top-p the target is p
    lg = torch.where(p > 0, p.log(), torch.full_like(p, -math.inf)).float().to(DEV)
    logits = lg.repeat(B, 1)
    if dense:
        qd = q.float().to(DEV)
        drafts = torch.stack([torch.multinomial(qd[i], B, replacement=True, generator=g) for i in range(k)], dim=1)
        dp = qd[None].expand(B, k, V_STAT).contiguous()
    else:
        drafts = torch.randint(0, V_STAT, (B, k), generator=g, device=DEV)
        dp = None
    args = dict(temperatures=torch.ones(B, device=DEV), top_ks=torch.zeros(B, dtype=torch.int32, device=DEV),
                top_ps=torch.ones(B, device=DEV))
    seq = torch.zeros(B, dtype=torch.int32, device=DEV)
    out, a, _ = acc(logits, drafts, torch.full((B,), k, dtype=torch.int32, device=DEV), seq, args["temperatures"],
                    args["top_ks"], args["top_ps"], torch.rand(B, k, generator=g, device=DEV),
                    torch.rand(B, generator=g, device=DEV), draft_probs=dp)
    out, a = out.cpu().numpy(), a.cpu().numpy()
    emit = [(int(a[i]), list(out[i])) for i in range(B)]
    p0, p1 = stat_check(emit, p, B)
    print(f"{'dense' if dense else 'token-only'}: chi-square p-values {p0:.3g} {p1:.3g}")
    assert p0 > 1e-6 and p1 > 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("V,dt", [(128256, "bf16"), (1025, "fp32"), (7, "fp16")])
def test_no_drafts_equals_sampler(V, dt):
    from chitu_b200.ops import sample_top_k_top_p
    B, k = 48, 3
    case = make_case(B, k, V, _dtype(dt), False, seed=V)
    case["temperatures"] = torch.tensor([[0.05, 1.0, 0.7][b % 3] for b in range(B)], dtype=F32, device=DEV)
    case["n_draft"] = torch.zeros(B, dtype=torch.int32, device=DEV)
    _, acc, nxt = run_entry(case, torch.zeros(B, dtype=torch.int32, device=DEV))
    rows0 = case["logits"][::k + 1]
    want = sample_top_k_top_p(rows0, case["temperatures"], case["top_ks"], case["top_ps"], case["u_draw"])
    torch.cuda.synchronize()
    assert bool((acc == 0).all()) and torch.equal(nxt, want)


# -------------------------------------------------------------------------------------------------------- engine
ENGINE_VARIANTS = ["bf16", "e4m3_kv", "w4a16", "fp8", "fp8_e4m3_kv"]


def sampled_engine(name, **kw):
    return SV.make_engine(dict(SV.VARIANTS[name].kw, sampled_verify=True, **kw))


def sampling_args(B, T):
    return dict(temperature=torch.tensor(T, dtype=F32), top_k=torch.tensor([0, 50, 1, 0, 7][:B], dtype=torch.int32),
                top_p=torch.tensor([1.0, 0.9, 1.0, 0.3, 0.8][:B], dtype=F32))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ENGINE_VARIANTS)
def test_greedy_equivalence(name):
    G = SV.make_engine(SV.VARIANTS[name].kw)
    S = sampled_engine(name)
    tok, drafts, n = SV.verify_inputs(G, seed=1)
    B = G.B
    lens = G.seq_lens.clone()
    out_g, acc_g = G.verify(tok, drafts, n)
    out_s, acc_s = S.verify(tok, drafts, n, **sampling_args(B, [0.0] * B))
    torch.cuda.synchronize()
    assert torch.equal(out_g, out_s) and torch.equal(acc_g, acc_s)
    assert torch.equal(G.next_tokens, S.next_tokens) and torch.equal(G.seq_lens, S.seq_lens)
    assert torch.equal(G.logits.view(torch.int16), S.logits.view(torch.int16))
    for cg, cs in zip(G.caches, S.caches):
        assert torch.equal(cg.view(torch.uint8), cs.view(torch.uint8))
    # a mixed batch: its greedy requests as the greedy step's
    S.seq_lens.copy_(lens)
    T = [0.0, 1.0, 0.0, 0.7, 0.0][:B]
    out_m, acc_m = S.verify(tok, drafts, n, **sampling_args(B, T))
    greedy = torch.tensor(T) == 0
    assert torch.equal(out_m[greedy], out_g[greedy]) and torch.equal(acc_m[greedy], acc_g[greedy])


def engine_case(e, dense):
    B, k = e.B, e.max_draft
    return dict(logits=e.logits[:B * (k + 1)], drafts=e.draft_tokens, n_draft=e.n_draft, temperatures=e.temperatures,
                top_ks=e.top_ks, top_ps=e.top_ps, u_accept=e.u_accept, u_draw=e.u_draw,
                draft_probs=e.draft_probs if dense else None)


def dense_inputs(e, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.softmax(torch.randn(e.B, e.max_draft, e.cfg.vocab_size, generator=g), dim=-1)


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_engine_tail_against_rule(dense):
    e = sampled_engine("bf16", draft_probs=dense)
    tok, drafts, n = SV.verify_inputs(e, seed=2)
    # drafts at the model's greedy choice would be accepted too often to test rejection; random ones rarely: mix them
    lens = e.seq_lens.clone()
    kw = sampling_args(e.B, [1.0, 0.05, 0.0, 1.0, 0.7])
    out, acc = e.verify(tok, drafts, n, draft_probs=dense_inputs(e, 3) if dense else None, **kw)
    torch.cuda.synchronize()
    n_dec, n_draw = check_against_rule(engine_case(e, dense), lens, out, acc, e.next_tokens, e.seq_lens)
    assert n_dec >= 3 and n_draw >= 2


def snapshot(e):
    return e.seq_lens.clone(), [c.clone() for c in e.caches], e.sample_generator.get_state()


def restore(e, snap):
    e.seq_lens.copy_(snap[0])
    for c, s in zip(e.caches, snap[1]):
        c.copy_(s)
    e.sample_generator.set_state(snap[2])


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
def test_graph_replay(dense):
    A, G = sampled_engine("bf16", draft_probs=dense), sampled_engine("bf16", draft_probs=dense)
    G.capture_verify()
    for ca, cg in zip(A.caches, G.caches):
        ca.copy_(cg)
    A.sample_generator.set_state(G.sample_generator.get_state())
    tok, drafts, n = SV.verify_inputs(A, seed=4)
    kw = sampling_args(A.B, [1.0, 1.0, 0.0, 0.7, 1.0])
    dp = dense_inputs(A, 5) if dense else None
    snap = snapshot(G)
    out_a, acc_a = A.verify(tok, drafts, n, draft_probs=dp, **kw)
    out_g, acc_g = G.verify(tok, drafts, n, draft_probs=dp, **kw)
    torch.cuda.synchronize()
    assert torch.equal(A.uniforms, G.uniforms)
    assert torch.equal(out_a, out_g) and torch.equal(acc_a, acc_g)
    SV.same_state(A, G, "graph vs eager")
    first = (out_g.clone(), G.uniforms.clone(), [c.clone() for c in G.caches], G.seq_lens.clone())
    # the next replay draws fresh uniforms
    G.verify(tok, drafts, n, draft_probs=dp, **kw)
    torch.cuda.synchronize()
    assert not torch.equal(G.uniforms, first[1])
    # rewound: generator state, seq_lens and caches restored -> the same step
    restore(G, snap)
    again, _ = G.verify(tok, drafts, n, draft_probs=dp, **kw)
    torch.cuda.synchronize()
    assert torch.equal(again, first[0]) and torch.equal(G.uniforms, first[1]) and torch.equal(G.seq_lens, first[3])
    assert all(torch.equal(c.view(torch.uint8), f.view(torch.uint8)) for c, f in zip(G.caches, first[2]))


@pytest.mark.gpu
def test_pdl_ordering():
    """The entry launched right behind the GEMM that writes its logits, and a decode step right behind the entry (which
    writes seq_lens), equal the same launches with a synchronise between them."""
    from chitu_b200.ops import linear
    B, k, V = 5, 3, 1024
    case = make_case(B, k, V, torch.bfloat16, True, seed=9)
    g = torch.Generator(device=DEV).manual_seed(10)
    x = torch.randn(B * (k + 1), 4096, generator=g, device=DEV).to(torch.bfloat16)
    w = (torch.randn(V, 4096, generator=g, device=DEV) * 0.05).to(torch.bfloat16)
    engs = [SV.make_engine({}), SV.make_engine({})]
    for ca, cb in zip(*(e.caches for e in engs)):
        cb.copy_(ca)
    engs[1].seq_lens.copy_(engs[0].seq_lens)
    tok = torch.randint(0, 1024, (B,), generator=torch.Generator().manual_seed(4)).pin_memory()
    results = []
    for i, e in enumerate(engs):
        torch.cuda.synchronize()
        e.tokens.copy_(tok)
        case["logits"] = linear(x, w)
        if i == 1:
            torch.cuda.synchronize()
        out = run_entry(case, e.seq_lens)
        if i == 1:
            torch.cuda.synchronize()
        e.step()
        torch.cuda.synchronize()
        results.append(out)
    a, b = engs
    for x1, x2 in zip(*results):
        assert torch.equal(x1, x2)
    assert torch.equal(a.seq_lens, b.seq_lens) and torch.equal(a.next_tokens, b.next_tokens)
    assert torch.equal(a.logits.view(torch.int16), b.logits.view(torch.int16))
    for ca, cb in zip(a.caches, b.caches):
        assert torch.equal(ca.view(torch.uint8), cb.view(torch.uint8))
