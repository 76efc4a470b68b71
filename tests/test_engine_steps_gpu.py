"""Each decode engine's production step, replayed as a CUDA graph over a run of decode steps, pinned step by step.

Every variant builds two engines from the same seed and context at toy widths (dim 512, 3 layers, vocabulary 1024), with
every RMSNorm weight overwritten by distinct random values in [0.5, 1.5): engine A runs eager and records the residual
stream entering every layer (`capture_h`); engine B is captured and stepped with `decode()`, as `bench.py` does.  Over
`STEPS` teacher-forced steps (a different seeded token vector each step) the batch holds a request starting at length
0, requests that cross a page boundary (255 -> 256, or 63 -> 64 for the 64-token MLA pages) during the run, and a long
request whose keys the decode kernel splits and which attends exactly `max_seq_len` keys in the last step.  At every
step:

1. graph = eager, bit for bit: logits, next tokens, `seq_lens` and every byte of every layer's cache; once per
   variant, `seq_lens` is rewound and the graph replayed, which must reproduce the step bit for bit;
2. KV bookkeeping: in every layer exactly one row per request changed (page `block_table[b, L // page]`, slot
   `L % page`), and each appended value is within one storage rounding (bf16, or e4m3 after a clamp to +-448) of the
   reference's row;
3. every layer, teacher-forced: the layer is recomputed in fp64 (tests/torch_ref.py) from A's own input to it and A's
   cache as it was before the step, and the layer's increment Δ = h_out - h_in is compared, so the residual stream
   cannot hide an error in the update; then the final norm + head from A's last residual, and `next_tokens` must be the
   first maximal index of the engine's own logits.  MoE routing must be identical, except on rows where the reference's
   own k-th and (k+1)-th scores are within one bf16 ulp; those rows are left out of the numeric check.

Bound: err = max|Δ_engine - Δ_ref| / max|Δ_ref|; floor = the largest err between the reference and itself with its input
moved by one bf16 ulp (`FLOOR_SEEDS` seeds, rows whose routing the perturbation flips left out).  Each layer needs
err <= max(3 floor, C_MIN) and err <= CAP.  `test_bound_rejects_injected_wiring_errors` (CPU) shows, at the same shapes
and lengths, that the bound rejects the wiring errors that are easiest to make in these engines.

DeepSeek's routing rule also excuses rows whose expert-group choice is a near tie, or whose k-th / (k+1)-th margin is
within three times the reference's own score movement under that perturbation: its fp8 GEMMs re-quantise their inputs,
so the gate inputs of two correct implementations differ by more than an ulp.

Measured on one H100 80GB HBM3 at a 700 W power limit, worst layer err (its floor) over the run: LLaMA head-dim 128
1.09e-2 (1.64e-2), head-dim 64 4.9e-3 (9.9e-3), linear_impl=1 1.10e-2 (1.37e-2), e4m3 KV 1.09e-2 (1.37e-2), tp=2 shard
1.11e-2 (1.11e-2); Mixtral 1.44e-2 (1.08e-2); DeepSeek 3.5e-2 (6.5e-2), e4m3 latent 5.2e-2 (5.8e-2).  Logits err
<= 4.2e-3 everywhere (floors 6e-3 to 1e-2).  So C_MIN = 1e-2 (below every LLaMA / Mixtral floor x 3) and CAP = 8e-2
(DeepSeek's floors x 3 exceed it).  With these, the CPU self-test rejects every injected error by a factor of at least 2
at some step; a cos / sin gather at seq_lens + 1, the previous layer's ffn_norm, seq_lens - 1 handed to the fused
rope attention and a dropped DeepSeek attention residual each fail `test_engine_steps` for every variant they reach.
"""
import dataclasses

import pytest
import torch

import torch_ref as R

BF, F8, F64 = torch.bfloat16, torch.float8_e4m3fn, torch.float64
STEPS = 8
BATCH = 5
REWIND_STEP = 3
FLOOR_SEEDS = 3
C_MIN = 1e-2
CAP = 8e-2
NORM_KEYS = ("attn_norm", "ffn_norm", "q_norm", "kv_norm")


@dataclasses.dataclass(frozen=True)
class Variant:
    family: str                  # "llama" | "mixtral" | "deepseek"
    engine_kw: tuple = ()        # extra engine keyword arguments
    head_dim: int = 128          # LLaMA only

    @property
    def page(self):
        return 64 if self.family == "deepseek" else 256

    @property
    def max_seq_len(self):
        # not a multiple of the page: the longest request crosses a page boundary in its last steps and attends exactly
        # max_seq_len keys in the last one
        return 4 * self.page + 4 if self.family != "deepseek" else 8 * self.page + 4

    @property
    def starts(self):
        # length 0 and 1 (the new key is most of what they attend); across a page boundary; across another; the
        # longest (split keys, ends at max_seq_len)
        p = self.page
        if self.family == "deepseek":
            return [0, 1, p - 4, 4 * p - 6, self.max_seq_len - STEPS]
        return [0, 1, p - 6, 2 * p - 4, self.max_seq_len - STEPS]


VARIANTS = {
    "llama_d128": Variant("llama"),                                           # fused-rope GQA, SiLU-pairs epilogue
    "llama_d64": Variant("llama", head_dim=64),                               # rotary_interleaved + SIMT attention
    "llama_linear_impl1": Variant("llama", (("linear_impl", 1),)),            # SIMT GEMV, unfused silu_and_mul
    "llama_e4m3_kv": Variant("llama", (("kv_dtype", F8),)),                   # gqa_paged_attn_fp8kv
    "llama_tp2_shard": Variant("llama", (("tp_size", 2),)),                   # per-rank heads, vocabulary shard
    "mixtral_tp2_shard": Variant("mixtral", (("tp_size", 2),)),               # rotary_half_strided, bf16 experts
    "deepseek_tp2_shard": Variant("deepseek", (("tp_size", 2),)),             # mla_decode over a bf16 latent cache
    "deepseek_tp2_e4m3": Variant("deepseek", (("tp_size", 2), ("kv_dtype", F8))),   # mla_attn_fp8kv
}


def make_engine(v: Variant, device):
    """The variant's engine with distinct random norm weights, a synthetic context and the variant's start lengths."""
    kw = dict(v.engine_kw)
    if v.family == "llama":
        from chitu_b200.engine import LlamaConfig, LlamaDecodeEngine
        cfg = LlamaConfig(dim=512, n_layers=3, n_heads=512 // v.head_dim, n_kv_heads=2, vocab_size=1024, multiple_of=256,
                          ffn_dim_multiplier=None)
        eng = LlamaDecodeEngine(cfg, max_reqs=BATCH, max_seq_len=v.max_seq_len, device=device, page_size=v.page, **kw)
    elif v.family == "mixtral":
        from chitu_b200.engine_mixtral import MixtralConfig, MixtralDecodeEngine
        cfg = MixtralConfig(dim=512, n_layers=3, n_heads=4, n_kv_heads=2, vocab_size=1024, intermediate_dim=512,
                            num_local_experts=4, num_experts_per_tok=2)
        eng = MixtralDecodeEngine(cfg, max_reqs=BATCH, max_seq_len=v.max_seq_len, device=device, page_size=v.page, **kw)
    else:
        from chitu_b200.engine_deepseek import DeepSeekConfig, DeepSeekDecodeEngine
        cfg = DeepSeekConfig(vocab_size=1024, dim=512, inter_dim=1024, moe_inter_dim=256, n_layers=3, n_dense_layers=1,
                             n_heads=8, n_routed_experts=16, n_activated_experts=4, n_expert_groups=4, n_limited_groups=2,
                             q_lora_rank=256)
        eng = DeepSeekDecodeEngine(cfg, max_reqs=BATCH, max_seq_len=v.max_seq_len, device=device, page_size=v.page, **kw)
    g = torch.Generator(device=eng.device).manual_seed(5)
    for w in [L[k] for L in eng.layers for k in NORM_KEYS if k in L] + [eng.norm]:
        w.copy_(0.5 + torch.rand(w.shape, generator=g, device=eng.device))
    eng.set_synthetic_context(0)
    eng.seq_lens.copy_(torch.tensor(v.starts, dtype=torch.int32))
    return eng


def step_tokens(t, vocab):
    return torch.randint(0, vocab, (BATCH,), generator=torch.Generator().manual_seed(100 + t))


class Model:
    """The fp64 reference of one engine's layers, reading the engine's weights, tables and block table."""

    def __init__(self, v: Variant, eng):
        self.v, self.eng = v, eng
        self.layers = eng.ref_layers() if v.family == "llama" else eng.layers
        self.k = None if v.family == "llama" else (eng.topk if v.family == "mixtral" else eng.cfg.n_activated_experts)

    def layer(self, li, h, caches, lens, cd=F64, fault=None, lw=None, pos_shift=0, routes=None):
        """h_out of layer li from h; `caches` (this layer's, cloned by the caller) get the appended rows."""
        e, lw = self.eng, lw or self.layers[li]
        pos = (lens + pos_shift).long().to(e.cos_table.device)
        cos, sin = e.cos_table[pos], e.sin_table[pos]
        eps = e.cfg.norm_eps
        if self.v.family == "llama":
            return R.llama_layer(lw, h, caches[0], caches[1], lens, e.block_table, cos, sin, e.Hq, e.Hkv, eps,
                                 compute_dtype=cd, fault=fault)
        if self.v.family == "mixtral":
            return R.mixtral_layer(lw, h, caches[0], caches[1], lens, e.block_table, cos, sin, e.Hq, e.Hkv, e.topk, eps,
                                   compute_dtype=cd, fault=fault, route_out=routes)
        return R.deepseek_layer(lw, h, caches[0], lens, e.block_table, cos, sin, e.cfg, e.H, routes, compute_dtype=cd,
                                fault=fault)

    def logits(self, h, cd=F64, norm=None):
        e = self.eng
        return R.final_logits(h, e.norm if norm is None else norm, e.head, e.cfg.norm_eps, cd)


def ulp_perturb(x, gen):
    """x (bf16) moved by about one ulp with a random sign on every element."""
    sign = torch.randint(0, 2, x.shape, generator=gen, device=x.device).float() * 2 - 1
    return (x.float() * (1 + sign * 2.0 ** -8)).to(BF)


def kept_rows(got_ids, routes, k, score_noise=None):
    """Rows whose routing agrees with the reference's.  A row may differ only where the reference's own k-th and
    (k+1)-th scores (or, for a grouped router, its last selected and best unselected group scores) are within one bf16 ulp (a tie two correct roundings may break either way), or, given
    `score_noise` (per row: how far the reference's own scores move, relative to the k-th, when its input moves by one
    bf16 ulp), within three times that noise: DeepSeek's fp8 GEMMs re-quantise their inputs, so the gate inputs of two
    correct implementations differ by more than an ulp."""
    if got_ids is None or not routes:
        return None
    idx, sc = routes[0][:2]
    diff = (got_ids[:, :k].sort(dim=-1)[0] != idx.to(got_ids.device).sort(dim=-1)[0]).any(dim=-1)
    if bool(diff.any()):
        top = sc.double().topk(k + 1, dim=-1)[0]
        margin = (top[:, k - 1] - top[:, k]) / top[:, k - 1].abs().clamp(min=1e-12)
        tie = torch.full_like(margin, 2.0 ** -7)
        if score_noise is not None:
            tie = torch.maximum(tie, 3 * score_noise.to(tie.device))
        excused = margin < tie
        if len(routes[0]) > 2:            # a grouped router: the group choice is a second selection
            excused |= routes[0][2].to(tie.device) < tie
        excused = excused.to(diff.device)
        assert bool(excused[diff].all()), "routing differs on a row that is neither a tie nor within the reference's noise"
    return ~diff


def rel_err(d_got, d_ref, rows=None):
    d_got, d_ref = d_got.double(), d_ref.double()
    if rows is not None:
        rows = rows.to(d_got.device)
        d_got, d_ref = d_got[rows], d_ref[rows]
    if d_ref.numel() == 0:
        return 0.0
    if not bool(d_got.isfinite().all()):
        return float("inf")
    return ((d_got - d_ref).abs().max() / d_ref.abs().max().clamp(min=1e-30)).item()


def bound(floor):
    return min(max(3 * floor, C_MIN), CAP)


def layer_floor(m, li, h, caches, lens, ref_out, ref_routes, gen):
    """(the largest err between the reference and itself with its input moved by one bf16 ulp, the largest move of each
    row's routing scores under that perturbation relative to its k-th score, or None)."""
    d_ref = ref_out.double() - h.double()
    floor, noise = 0.0, None
    for _ in range(FLOOR_SEEDS):
        hp, routes = ulp_perturb(h, gen), []
        out = m.layer(li, hp, [c.clone() for c in caches], lens, routes=routes)
        rows = None
        if routes:
            rows = (routes[0][0].sort(dim=-1)[0] == ref_routes[0][0].sort(dim=-1)[0]).all(dim=-1)
            sc, sc_p = ref_routes[0][1].double(), routes[0][1].double()
            kth = sc.topk(m.k, dim=-1)[0][:, -1].abs().clamp(min=1e-12)
            move = (sc_p - sc).abs().amax(dim=-1) / kth
            noise = move if noise is None else torch.maximum(noise, move)
        floor = max(floor, rel_err(out.double() - hp.double(), d_ref, rows))
    return floor, noise


def append_mask(cache, table, lens, page):
    mask = torch.zeros(cache.shape[0], cache.shape[1], dtype=torch.bool, device=cache.device)
    for b, L in enumerate(lens.tolist()):
        mask[int(table[b, L // page]), L % page] = True
    return mask


def check_append(after, before, ref_after, table, lens, page, upstream=2.0 ** -8):
    """Exactly the row (table[b, L // page], L % page) of every request changed; returns the largest distance of an
    appended value from the reference's, in units of one rounding of the cache's element type plus `upstream` of the
    row's range (the GEMM output the row was computed from: two accumulation orders may round it differently, and an
    fp8 GEMM re-quantises its input, which moved DeepSeek's latent rows by up to 1.8 % of the range on the H100)."""
    mask = append_mask(after, table, lens, page)
    nb, pg = after.shape[0], after.shape[1]
    a, b = after.view(torch.uint8).reshape(nb, pg, -1), before.view(torch.uint8).reshape(nb, pg, -1)
    assert torch.equal(a[~mask], b[~mask]), "a cache row other than the appended ones changed"
    got = after.reshape(nb, pg, -1)[mask].double()
    want = ref_after.to(after.device).reshape(nb, pg, -1)[mask].double()
    rel = 2.0 ** -3 if after.dtype == F8 else 2.0 ** -8
    tol = rel * torch.maximum(got.abs(), want.abs()) + upstream * want.abs().amax(dim=-1, keepdim=True) + 2.0 ** -9
    return ((got - want).abs() / tol).max().item()


def assert_same_state(a, b, na, nb, what):
    assert torch.equal(na, nb), f"{what}: next tokens differ"
    assert torch.equal(a.logits.view(torch.int16), b.logits.view(torch.int16)), f"{what}: logits differ"
    assert torch.equal(a.seq_lens, b.seq_lens), f"{what}: seq_lens differ"
    for ca, cb in zip(a.caches, b.caches):
        assert torch.equal(ca.view(torch.uint8), cb.view(torch.uint8)), f"{what}: KV cache bytes differ"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VARIANTS))
def test_engine_steps(name):
    v = VARIANTS[name]
    dev = "cuda:0"
    A, G = make_engine(v, dev), make_engine(v, dev)
    G.capture()
    for ca, cg in zip(A.caches, G.caches):         # capture()'s warm-up steps wrote cache rows
        ca.copy_(cg)
    m = Model(v, A)
    n_layers = len(A.layers)
    gen = torch.Generator(device=dev).manual_seed(9)
    worst = dict(kv=0.0, layer=(0.0, 0.0, None), logits=(0.0, 0.0, None))
    failures = []
    for t in range(STEPS):
        tok = step_tokens(t, A.cfg.vocab_size).pin_memory()
        lens = A.seq_lens.clone()
        before = [[c[li].clone() for c in A.caches] for li in range(n_layers)]
        A.capture_h = []
        na = A.decode(tok)
        hs, A.capture_h = A.capture_h, None
        ng = G.decode(tok)
        torch.cuda.synchronize()
        assert len(hs) == n_layers + 1
        assert_same_state(A, G, na, ng, f"step {t}: graph vs eager")
        if t == REWIND_STEP:
            first = (G.logits.clone(), ng.clone(), [c.clone() for c in G.caches])
            G.seq_lens.copy_(lens)
            again = G.decode(tok)
            torch.cuda.synchronize()
            assert torch.equal(again, first[1]) and torch.equal(G.logits.view(torch.int16), first[0].view(torch.int16))
            assert all(torch.equal(c.view(torch.uint8), f.view(torch.uint8)) for c, f in zip(G.caches, first[2])), \
                "rewound replay changed the caches"
        assert torch.equal(A.seq_lens, lens + 1)
        assert torch.equal(A.next_tokens, A.logits.float().argmax(dim=-1)), "next token is not the first maximal index"
        if v.family == "deepseek":        # the shared expert: the last routing slot of every MoE token, weight 1
            nd = A.cfg.n_dense_layers
            assert bool((A.gate_i_all[nd:, :, -1] == A.cfg.n_routed_experts).all())
            assert bool((A.gate_w_all[nd:, :, -1] == 1).all())
        for li in range(n_layers):
            caches, routes = [c.clone() for c in before[li]], []
            ref = m.layer(li, hs[li], caches, lens, routes=routes)
            for after, b4, r in zip((c[li] for c in A.caches), before[li], caches):
                worst["kv"] = max(worst["kv"], check_append(after, b4, r, A.block_table, lens, A.page,
                                                            2.0 ** -5 if v.family == "deepseek" else 2.0 ** -8))
            floor, noise = layer_floor(m, li, hs[li], before[li], lens, ref, routes, gen)
            got_ids = A.gate_i_all[li] if m.k is not None and (v.family == "mixtral" or li >= A.cfg.n_dense_layers) else None
            rows = kept_rows(got_ids, routes, m.k, noise if v.family == "deepseek" else None)
            err = rel_err(hs[li + 1].double() - hs[li].double(), ref.double() - hs[li].double(), rows)
            if err > worst["layer"][0]:
                worst["layer"] = (err, floor, (t, li))
            if err > bound(floor):
                failures.append(f"step {t} layer {li}: err {err:.3e} > bound {bound(floor):.3e} (floor {floor:.3e})")
        ref = m.logits(hs[-1])
        err = rel_err(A.logits.double(), ref)
        floor = max(rel_err(m.logits(ulp_perturb(hs[-1], gen)), ref) for _ in range(FLOOR_SEEDS))
        if err > worst["logits"][0]:
            worst["logits"] = (err, floor, t)
        if err > bound(floor):
            failures.append(f"step {t} logits: err {err:.3e} > bound {bound(floor):.3e} (floor {floor:.3e})")
    print(f"{name}: worst layer err {worst['layer'][0]:.3e} (floor {worst['layer'][1]:.3e}, step/layer {worst['layer'][2]})"
          f"  worst logits err {worst['logits'][0]:.3e} (floor {worst['logits'][1]:.3e})"
          f"  appended KV {worst['kv']:.2f} roundings")
    assert worst["kv"] <= 1.0, f"an appended KV value is {worst['kv']:.2f} roundings from the reference's"
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------ the bound bites (CPU)
def _cpu_engine(v):
    """The variant's engine built on the CPU (weights, caches, tables; no kernel runs)."""
    from test_engine_calls_cpu import Recorder, _patched
    with _patched(Recorder()):
        return make_engine(v, "cpu")


def _faults(v, m, li):
    """(name, keyword arguments of Model.layer) for every injected wiring error that applies to layer li."""
    L = m.layers[li]
    out = [("rotary at L + 1", dict(pos_shift=1)),
           ("new key / value not attended", dict(fault="new_kv_dropped")),
           ("ffn_norm and attn_norm swapped", dict(lw=dict(L, attn_norm=L["ffn_norm"], ffn_norm=L["attn_norm"]))),
           ("residual added twice", dict(fault="residual_twice")),
           ("residual dropped", dict(fault="residual_dropped"))]
    if li > 0:
        out += [("previous layer's cache", dict(prev_cache=True)),
                ("next_norm from the wrong layer", dict(lw=dict(L, attn_norm=m.layers[li - 1]["attn_norm"])))]
    if v.family == "mixtral":
        F = L["w1"].shape[1] // 2
        out += [("gate / up halves swapped", dict(lw=dict(L, w1=torch.cat([L["w1"][:, F:], L["w1"][:, :F]], dim=1)))),
                ("routing weights not renormalised", dict(fault="no_renorm"))]
    if v.family == "deepseek":
        out += [("one absorbed head off by one", dict(fault="head_off_by_one"))]
        if li >= m.eng.cfg.n_dense_layers:
            out += [("shared expert weight 0.5", dict(fault="shared_weight"))]
    return out


@pytest.mark.parametrize("name", list(VARIANTS))
def test_bound_rejects_injected_wiring_errors(name):
    """At the variant's shapes and at every step's lengths, the layer bound of `test_engine_steps` passes a correct
    implementation (the fp32 reference stands in for the engine) and rejects every injected wiring error: each must
    push some layer of the run over its bound, as `test_engine_steps` would then fail."""
    v = VARIANTS[name]
    eng = _cpu_engine(v)
    m = Model(v, eng)
    n_layers = len(eng.layers)
    gen = torch.Generator().manual_seed(9)
    caches0 = [[c[li].clone() for c in eng.caches] for li in range(n_layers)]
    rejected = {}
    for t in range(STEPS):
        lens = torch.tensor(v.starts, dtype=torch.int32) + t
        h = eng.embed[step_tokens(t, eng.cfg.vocab_size)]
        for li in range(n_layers):
            routes, r32 = [], []
            ref = m.layer(li, h, [c.clone() for c in caches0[li]], lens, routes=routes)
            floor, _ = layer_floor(m, li, h, caches0[li], lens, ref, routes, gen)
            d_ref = ref.double() - h.double()
            ok = m.layer(li, h, [c.clone() for c in caches0[li]], lens, cd=torch.float32, routes=r32)
            err = rel_err(ok.double() - h.double(), d_ref, kept_rows(r32[0][0] if r32 else None, routes, m.k))
            assert err <= bound(floor), f"step {t} layer {li}: the fp32 reference fails the bound ({err:.3e})"
            for fname, kw in _faults(v, m, li):
                src = caches0[li - 1] if kw.pop("prev_cache", False) else caches0[li]
                bad = m.layer(li, h, [c.clone() for c in src], lens, **kw)
                ratio = rel_err(bad.double() - h.double(), d_ref) / bound(floor)
                r = rejected.setdefault(fname, [0.0] * STEPS)
                r[t] = max(r[t], ratio)
            h = ref
    for fname, r in rejected.items():
        print(f"{name}: {fname}: err / bound per step " + " ".join(f"{x:.1f}" for x in r))
    missed = [f for f, r in rejected.items() if max(r) <= 1.0]
    assert not missed, f"the bound does not reject {missed}"
