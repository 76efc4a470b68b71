"""Sampled verification of speculative drafts without a GPU: the refusals of chitu_b200_spec_accept_sampled, its
Python wrapper and the LLaMA engine's sampled verify step; the verify step's library calls, recorded with
test_engine_calls_cpu's stand-ins; and the fp64 reference of the rule (`spec_rule`), checked statistically: the first
emitted token is distributed as p_0, and after an accepted d_0 the second as p_1."""
import contextlib
import json
from unittest import mock

import numpy as np
import pytest
import torch
from scipy.stats import chisquare

import test_engine_calls_cpu as EC

K = 3
SAMPLED = dict(max_draft=K, sampled_verify=True)


# -------------------------------------------------------------------------------------------------- the fp64 rule
def target_probs(l, T, top_k, top_p, kept=None):
    """p of one row (fp64 logits l [V], as stored): softmax(l / T), renormalised over the kept set (an entry is kept
    when the mass of strictly larger entries is <= top_p and fewer than top_k entries are strictly larger).  `kept`
    overrides the kept mask."""
    l = torch.as_tensor(l, dtype=torch.float64)
    V = l.numel()
    p = torch.softmax(l / T, dim=0)
    if kept is None:
        asc, _ = p.sort()
        cs = torch.cumsum(asc.flip(0), 0)
        n_gt = V - torch.searchsorted(asc, p, right=True)
        m_gt = torch.where(n_gt > 0, cs[(n_gt - 1).clamp(min=0)], torch.zeros((), dtype=p.dtype))
        kept = (p > 0) & (m_gt <= top_p) & (n_gt < (top_k if top_k > 0 else V))
    pk = torch.where(kept, p, 0.0)
    return pk / pk.sum()


def draw(w, u):
    """Inverse CDF in vocabulary order at u * sum(w); past the end: the last positive entry."""
    w = torch.as_tensor(w, dtype=torch.float64)
    c = torch.cumsum(w, 0)
    idx = torch.nonzero(c > u * float(c[-1]))
    return int(idx[0]) if idx.numel() else int(torch.nonzero(w > 0)[-1])


def spec_rule(p, q, drafts, n, u_accept, u_draw):
    """One request: p [n + 1, V] the target rows, q [n, V] the drafter's (None: one-hot at the drafts), drafts [n],
    u_accept [n], u_draw.  Returns (accepted count a, emitted tokens [a + 1])."""
    a = 0
    while a < n:
        d = int(drafts[a])
        qd = 1.0 if q is None else float(q[a][d])
        if not (p[a][d] > 0 and u_accept[a] * qd < p[a][d]):
            break
        a += 1
    if a < n:
        qa = torch.zeros_like(p[a]) if q is None else torch.as_tensor(q[a], dtype=torch.float64)
        if q is None:
            qa[int(drafts[a])] = 1.0
        r = (p[a] - qa).clamp(min=0)
        tok = draw(r if float(r.sum()) > 0 else p[a], u_draw)
    else:
        tok = draw(p[a], u_draw)
    return a, [int(x) for x in drafts[:a]] + [tok]


def _chi2(counts, p, N):
    p = np.asarray(p, dtype=np.float64)
    counts = np.asarray(counts, dtype=np.float64)
    assert counts[p == 0].sum() == 0, "a token outside the kept set was emitted"
    sel = p > 0
    return chisquare(counts[sel], p[sel] / p[sel].sum() * counts.sum()).pvalue


V_STAT = 8


def stat_rows(dense):
    """Three target rows for two drafts (T 0.8, top_k 6, top_p 0.95: some entries cut) and the drafter's two rows
    (dense, or one-hot)."""
    g = torch.Generator().manual_seed(11)
    l = torch.randn(3, V_STAT, generator=g, dtype=torch.float64) * 1.5
    p = torch.stack([target_probs(l[i], 0.8, 6, 0.95) for i in range(3)])
    q = torch.softmax(torch.randn(2, V_STAT, generator=g, dtype=torch.float64) * 1.5, dim=1) if dense else None
    return p, q


def stat_check(emit, p, N):
    """first tokens ~ p_0; second tokens after an accepted d_0 ~ p_1 (chi-square p-values)"""
    first = np.bincount([e[1][0] for e in emit], minlength=V_STAT)
    second = np.bincount([e[1][1] for e in emit if e[0] >= 1], minlength=V_STAT)
    assert second.sum() > N // 10, "too few accepted first drafts to test the second token"
    return _chi2(first, p[0], N), _chi2(second, p[1], N)


@pytest.mark.parametrize("dense", [False, True])
def test_rule_is_distribution_preserving(dense):
    p, q = stat_rows(dense)
    N = 20000
    rng = np.random.default_rng(3)
    emit = []
    for _ in range(N):
        if dense:        # draft-model drafts are drawn from the drafter's rows
            d = [int(rng.choice(V_STAT, p=q[i].numpy() / q[i].sum().item())) for i in range(2)]
        else:            # token-only drafts: any proposal, here random tokens (some outside the kept set)
            d = [int(x) for x in rng.integers(0, V_STAT, 2)]
        emit.append(spec_rule(p, q, d, 2, rng.random(2), rng.random()))
    p0, p1 = stat_check(emit, p, N)
    assert p0 > 1e-6 and p1 > 1e-6, (p0, p1)


# ------------------------------------------------------------------------------------------------------- refusals
def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def test_c_entry_refuses_bad_arguments_and_launches_nothing():
    from chitu_b200 import _lib as L
    lib = _lib()
    A = 1 << 20                              # stand-ins: every case is refused before a dereference
    names = ("logits", "temps", "top_ks", "top_ps", "drafts", "n_draft", "u_accept", "u_draw", "seq_lens", "out",
             "accepted", "nxt", "ws")
    ptrs = {n: (i + 1) * A for i, n in enumerate(names)}
    need = lib.chitu_b200_spec_accept_sampled_workspace_bytes(4, 3)
    assert need >= 4 * 4 * 16

    def call(**kw):
        v = dict(ptrs, B=4, k=3, V=1000, stride=1000, dtype=L.CB_BF16, dp=None, dp_stride=0, ws_bytes=need)
        v.update(kw)
        return lib.chitu_b200_spec_accept_sampled(
            v["logits"], v["stride"], v["V"], v["dtype"], v["temps"], v["top_ks"], v["top_ps"], v["drafts"],
            v["n_draft"], v["dp"], v["dp_stride"], v["u_accept"], v["u_draw"], v["seq_lens"], v["out"], v["accepted"],
            v["nxt"], v["B"], v["k"], v["ws"], v["ws_bytes"], None)

    before = L.launch_count()
    bad = [{n: None} for n in names] + [dict(B=-1), dict(k=0), dict(k=-2), dict(V=0), dict(stride=999),
                                         dict(ws_bytes=need - 1), dict(dp=15 * A, dp_stride=999),
                                         dict(dtype=L.CB_FP8_E4M3), dict(dtype=L.CB_I32)]
    for kw in bad:
        assert call(**kw) < 0, kw
        assert "chitu_b200_spec_accept_sampled" in lib.chitu_b200_last_error().decode(), kw
    assert call(B=0) == 0                    # nothing to do
    assert L.launch_count() == before


def _ok_args(B=4, k=3, V=16, dtype=torch.bfloat16, dense=False):
    f32, i32 = torch.float32, torch.int32
    a = dict(logits=torch.zeros(B * (k + 1), V, dtype=dtype), drafts=torch.zeros(B, k, dtype=torch.int64),
             n_draft=torch.zeros(B, dtype=i32), seq_lens=torch.zeros(B, dtype=i32), temperatures=torch.ones(B),
             top_ks=torch.zeros(B, dtype=i32), top_ps=torch.ones(B), u_accept=torch.zeros(B, k, dtype=f32),
             u_draw=torch.zeros(B, dtype=f32))
    a["draft_probs"] = torch.zeros(B, k, V, dtype=f32) if dense else None
    return a


def test_wrapper_refusals():
    from chitu_b200._lib import launch_count
    from chitu_b200.ops import accept_draft_tokens_sampled as acc
    _lib()
    B, k, V = 4, 3, 16
    f32, i32, i64 = torch.float32, torch.int32, torch.int64
    bad = [dict(logits=None), dict(logits=torch.zeros(B * (k + 1), V, dtype=torch.int32)),
           dict(logits=torch.zeros(B * (k + 1), V, dtype=torch.float8_e4m3fn)),
           dict(logits=torch.zeros(B * k, V)), dict(logits=torch.zeros(V, B * (k + 1)).t()),
           dict(logits=torch.zeros(B * (k + 1) * V)), dict(drafts=torch.zeros(B, k, dtype=i32)),
           dict(drafts=torch.zeros(B, 0, dtype=i64)), dict(n_draft=torch.zeros(B, dtype=i64)),
           dict(seq_lens=torch.zeros(B + 1, dtype=i32)), dict(temperatures=torch.ones(B, dtype=torch.float64)),
           dict(top_ks=torch.zeros(B, dtype=i64)), dict(top_ps=torch.ones(B, 1)),
           dict(u_accept=torch.zeros(B, k + 1)), dict(u_accept=torch.zeros(B, k, dtype=torch.float16)),
           dict(u_draw=torch.zeros(B, 2)), dict(drafts=torch.zeros(k, B, dtype=i64).t()),
           dict(draft_probs=torch.zeros(B, k, V, dtype=torch.float16)), dict(draft_probs=torch.zeros(B, k, V + 1)),
           dict(draft_probs=torch.zeros(B, V, k).transpose(1, 2)), dict(draft_probs=torch.zeros(B, k + 1, V)[:, :k]),
           dict(draft_probs=torch.zeros(B * k * V))]
    before = launch_count()
    for kw in bad + [{}, dict(draft_probs=torch.zeros(B, k, V, dtype=f32))]:   # the last two: CPU tensors
        args = dict(_ok_args(B, k, V), **kw)
        with pytest.raises(ValueError):
            acc(**args)
    assert launch_count() == before


def test_engine_refusals():
    with pytest.raises(ValueError, match="max_draft"):
        EC._llama(128, sampled_verify=True)
    with pytest.raises(ValueError, match="sampled_verify"):
        EC._llama(128, max_draft=K, draft_probs=True)
    for tp in (dict(tp_size=2), EC._TP):
        with pytest.raises(ValueError, match="one GPU"):
            EC._llama(128, **tp, **SAMPLED)
    B = 3
    tok, drafts = torch.zeros(B, dtype=torch.int64), torch.zeros(B, K, dtype=torch.int64)
    nd = torch.full((B,), K, dtype=torch.int32)
    T, tk, tp = torch.ones(B), torch.zeros(B, dtype=torch.int32), torch.ones(B)
    # a greedy engine takes no sampling arguments
    greedy = EC._llama(128, max_draft=K)
    for kw in (dict(temperature=T), dict(top_k=tk), dict(top_p=tp), dict(temperature=T, top_k=tk, top_p=tp),
               dict(draft_probs=torch.zeros(B, K, 1024))):
        with pytest.raises(ValueError, match="sampled_verify"):
            greedy.verify(tok, drafts, nd, **kw)
    eng = EC._llama(128, **SAMPLED)
    bad = [dict(), dict(top_k=tk, top_p=tp), dict(temperature=T, top_p=tp), dict(temperature=T, top_k=tk),
           dict(temperature=torch.ones(B + 1), top_k=tk, top_p=tp),
           dict(temperature=T, top_k=torch.zeros(B, 1, dtype=torch.int32), top_p=tp),
           dict(temperature=torch.tensor([1.0, float("inf"), 1.0]), top_k=tk, top_p=tp),
           dict(temperature=torch.tensor([1.0, float("nan"), 1.0]), top_k=tk, top_p=tp),
           dict(temperature=T, top_k=tk, top_p=torch.tensor([1.0, 0.0, 0.5])),
           dict(temperature=T, top_k=tk, top_p=torch.tensor([1.0, 1.5, 0.5])),
           dict(temperature=T, top_k=tk, top_p=tp, draft_probs=torch.zeros(B, K, 1024))]     # token-only engine
    for kw in bad:
        with pytest.raises(ValueError):
            eng.verify(tok, drafts, nd, **kw)
    dense = EC._llama(128, draft_probs=True, **SAMPLED)
    assert tuple(dense.draft_probs.shape) == (B, K, 1024) and dense.draft_probs.dtype == torch.float32
    for dp in (None, torch.zeros(B, K, 1023), torch.zeros(B, K - 1, 1024), torch.zeros(B, K, 1024, dtype=torch.float64)):
        with pytest.raises(ValueError, match="draft_probs"):
            dense.verify(tok, drafts, nd, temperature=T, top_k=tk, top_p=tp, draft_probs=dp)


# ---------------------------------------------------------------------------------------------------- call lists
@contextlib.contextmanager
def _rand_recorded(rec):
    real = torch.rand

    def rand(*args, out=None, **kw):
        rec.record("torch.rand", (out,))
        return real(*args, out=out, **kw)

    with mock.patch.object(torch, "rand", rand):
        yield


def _trace(kw, body):
    rec = EC.Recorder()
    with EC._patched(rec), _rand_recorded(rec):
        eng = EC._llama(128, **kw)
        rec.watch(eng)
        getattr(eng, body)()
    return eng, rec


MODES = {"single": dict(), "single_e4m3_kv": dict(kv_dtype=torch.float8_e4m3fn), "single_w4a16": dict(weight_format="w4a16"),
         "single_fp8": dict(weight_format="fp8")}


@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("mode", list(MODES))
def test_sampled_verify_step_calls(mode, dense):
    """The greedy verify step's calls up to the head, then the uniforms, then the sampled acceptance: no argmax and no
    greedy acceptance."""
    _, greedy = _trace(dict(MODES[mode], max_draft=K), "_verify_body")
    eng, rec = _trace(dict(MODES[mode], draft_probs=dense, **SAMPLED), "_verify_body")
    assert [c[0] for c in greedy.calls[-2:]] == ["chitu_b200_argmax", "chitu_b200_spec_accept_greedy"]
    assert rec.calls[:-2] == greedy.calls[:-2]
    p = lambda t: rec.pointer(t.data_ptr())                         # noqa: E731
    B, V = eng.B, eng.cfg.vocab_size
    assert rec.calls[-2] == ["torch.rand", p(eng.uniforms)]
    assert eng.uniforms.numel() == B * (K + 1)
    assert p(eng.u_accept) == p(eng.uniforms) and p(eng.u_draw)[1] == B * K * 4
    dp = [None, 0] if not dense else [p(eng.draft_probs), V]
    assert rec.calls[-1] == ["chitu_b200_spec_accept_sampled", p(eng.logits), V, V, 0, p(eng.temperatures),
                             p(eng.top_ks), p(eng.top_ps), p(eng.draft_tokens), p(eng.n_draft)] + dp + \
        [p(eng.u_accept), p(eng.u_draw), p(eng.seq_lens), p(eng.out_tokens), p(eng.accepted), p(eng.next_tokens), B, K,
         p(eng.spec_ws), eng.spec_ws.numel(), 0]
    assert eng.logits.shape[0] == B * (K + 1)


def test_decode_step_unchanged_with_sampled_verify():
    """An engine built for sampled verification runs exactly the golden decode step."""
    with open(EC.GOLDEN) as f:
        want = json.load(f)["llama_single_rope"]
    _, rec = _trace(dict(draft_probs=True, **SAMPLED), "_step_body")
    assert json.loads(json.dumps(rec.calls)) == want
