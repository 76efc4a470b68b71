"""The tensor-parallel decode engines at W = 2 and 4, as W processes on one GPU, pinned to the fp64 reference of the
model their shards assemble.

Each rank draws its own random shards (seed + 1000 * rank), so the model of a tensor-parallel engine is defined only
as the assembly of its W shards.  `assemble` states that sharding map once per family: q / k / v heads rank-major in
`wqkv`; `wo` and `w2` concatenated along K; each rank's `w13` ([gate ; up] after un-interleaving) concatenated as
[gate_0 .. gate_{W-1} ; up_0 .. up_{W-1}], per expert the same for `w1` / `we1` along N1 and `w2` / `we2` along K;
DeepSeek's `wq_b`, `wkv_b` and `wo` following their heads, with the fp8 block-scale rows beside them; the head
concatenated along the vocabulary.  The KV caches assemble the same way (the concatenation of the ranks' KV heads;
DeepSeek's latent cache is replicated and must be identical on every rank).  Each rank's caches are filled with its
heads' slice of one seeded full-width cache, so that the assembled cache holds distinct heads.

`test_tp_engine_steps` spawns W worker processes on cuda:0 (gloo over a FileStore, a short timeout), builds every
variant of that W with `tp_rank=r, tp_size=W, process_group=group, use_fused_allreduce=False` and runs `STEPS` eager
teacher-forced decode steps at the start lengths of `test_engine_steps_gpu.Variant.starts`: the engine's
`torch.distributed` path (`_allreduce` -> `dist.all_reduce` and `global_argmax` -> `dist.all_gather_into_tensor`), with
gloo standing in for NCCL, which refuses two ranks on one device.  Every wait is a host-side collective; no kernel
spins on another process's memory.  This torch's gloo takes the CUDA tensors of both collectives; where a gloo build
refuses them, the worker stages the two calls through host copies in its own process (`_stage_collectives`) and the
test prints which path ran.  The parent then checks:

1. replicated state is identical on every rank, bit for bit: embedding, norms, router weights, DeepSeek's `wqkv_a`,
   block table, rotary tables, the residual stream entering every layer, routing, next tokens, `seq_lens`, DeepSeek's
   latent cache, and the verify outputs;
2. every layer, teacher-forced from the ranks' common input, against `torch_ref.*_layer` of the assembled model with
   the full head counts, with the bound, floor and routing rule of `test_engine_steps_gpu`; then the final norm + the
   assembled head against the concatenated logits;
3. KV bookkeeping in the assembled caches: exactly one row per request per layer changed, within one storage rounding
   of the reference's (so no rank writes outside its heads' rows);
4. next tokens are the first maximal index of the concatenated logits; in step `TIE_STEP` every rank's head shard is
   the same seeded matrix, so every row's maximum ties across all W shards and the lowest global index must win;
5. verify (`max_draft=3`, greedy): `max_draft + 1` passes over the same positions, each pass's drafts extending the
   greedy chain of the last, so that every acceptance count 0 .. n_draft occurs; `target` is the first maximal index
   of the concatenated verify logits, and `out_tokens`, `accepted` and `seq_lens` are greedy acceptance over it.

A TP step rounds each rank's partial to bf16 before the sum, one rounding more than the full model; the bound of
`test_engine_steps_gpu` absorbs it unchanged (below).

`test_rank_by_rank_equals_assembled_model` (CPU) pins the sharding map without a GPU: an fp64 computation that applies
each rank's own shards and head slice and sums the partials agrees with the assembled model's reference to 1e-12 (it
is bit-identical at these shapes), and so do the appended cache rows and the logits.
`test_bound_rejects_assembly_faults` (CPU) shows that each assembly fault a shared sharding error would make pushes
some layer (or the logits) past its bound at some step, by a factor of at least 2.3 (DeepSeek's gate / up swap on one
rank; the others by 3 to 100).

Measured on one H100 80GB HBM3 at a 700 W power limit, worst layer err (its floor), worst logits err (its floor),
appended KV distance in storage roundings:
  W = 2  LLaMA d128       1.13e-2 (7.0e-3)   4.5e-3 (6.8e-3)   0.67
         LLaMA e4m3 KV    1.32e-2 (9.9e-3)   2.5e-3 (9.9e-3)   0.27
         Mixtral          1.27e-2 (1.43e-2)  2.3e-3 (7.0e-3)   0.44
         DeepSeek         3.60e-2 (5.21e-2)  2.5e-4 (6.0e-3)   0.61
         DeepSeek e4m3    4.34e-2 (5.27e-2)  3.1e-4 (9.8e-3)   0.65
         LLaMA verify     (decode steps as LLaMA d128)          0.43
  W = 4  LLaMA d128       1.95e-2 (1.40e-2)  2.6e-3 (1.05e-2)  0.65
         Mixtral          1.27e-2 (1.11e-2)  4.3e-3 (8.6e-3)   0.65
gloo ran both collectives on the CUDA tensors (no host staging).  The whole GPU test took 47 s (W = 2: 15 s in the
ranks, 11 s of checks; W = 4: 15 s and 4 s).  Making `global_argmax` add (rank ^ 1) * vocab_local fails check 4 at
step 0; letting rank 1 read its interleaved w13 rows as [gate ; up] halves fails every layer by 10x to 20x its bound.
"""
import dataclasses
import datetime
import os
import tempfile
import time
import traceback

import pytest
import torch

import test_engine_steps_gpu as ES
import torch_ref as R
from test_spec_verify_gpu import accept_rule

BF, F8, F64 = torch.bfloat16, torch.float8_e4m3fn, torch.float64
STEPS = ES.STEPS
BATCH = ES.BATCH
TIE_STEP = 5
VERIFY_N_DRAFT = [3, 3, 2, 1, 0]          # per request
GLOO_TIMEOUT_S = 120
JOIN_S = 900
REPLICATED = ("attn_norm", "ffn_norm", "q_norm", "kv_norm", "gate_w", "gate_b", "wqkv_a", "wqkv_a_s")
# engine entries the reference does not read: DeepSeek's dequantised wkv_b and the shared expert's views into we1 / we2
NOT_SAVED = ("wkv_b_bf16", "ws13", "ws13_s", "ws2", "ws2_s")


@dataclasses.dataclass(frozen=True)
class TPVariant:
    family: str                  # "llama" | "mixtral" | "deepseek"
    world: int
    engine_kw: tuple = ()

    @property
    def es(self):
        """test_engine_steps_gpu's variant of the family: page, max_seq_len and start lengths."""
        return ES.Variant(self.family)

    @property
    def max_draft(self):
        return dict(self.engine_kw).get("max_draft", 0)

    @property
    def starts(self):
        s = list(self.es.starts)
        # the verify passes after the decode steps write max_draft + 1 rows: the longest request ends at max_seq_len
        s[-1] -= self.max_draft + 1 if self.max_draft else 0
        return s


VARIANTS = {
    "llama_d128_w2": TPVariant("llama", 2),                                     # fused-rope GQA, SiLU-pairs epilogue
    "llama_e4m3_kv_w2": TPVariant("llama", 2, (("kv_dtype", F8),)),             # gqa_paged_attn_fp8kv
    "mixtral_w2": TPVariant("mixtral", 2),                                      # bf16 experts, one reduce per layer
    "deepseek_w2": TPVariant("deepseek", 2),                                    # bf16 latent cache
    "deepseek_e4m3_w2": TPVariant("deepseek", 2, (("kv_dtype", F8),)),          # e4m3 latent cache
    "llama_verify_w2": TPVariant("llama", 2, (("max_draft", 3),)),              # greedy verify, max_draft = 3
    "llama_d128_w4": TPVariant("llama", 4),
    "mixtral_w4": TPVariant("mixtral", 4),
}
CPU_VARIANTS = [n for n, v in VARIANTS.items() if not v.max_draft]      # the verify engine's layers are llama_d128's

# assembly faults a sharding error shared by every reduction path would make (`assemble`'s `fault`)
FAULTS = {
    "llama": ("q shards swapped, KV not", "wo in reverse rank order", "rank 1's gate / up swapped",
              "head offset by one rank"),
    "mixtral": ("q shards swapped, KV not", "wo in reverse rank order", "rank 1's gate / up swapped",
                "experts' halves in reverse rank order", "head offset by one rank"),
    "deepseek": ("wo in reverse rank order", "rank 1's gate / up swapped", "experts' halves in reverse rank order",
                 "rank 1's wkv_b with rank 0's heads", "head offset by one rank"),
}


def config(family, W):
    """test_engine_steps_gpu's toy widths, scaled so that every shard stays a multiple of 128 where an fp8 block
    scale or a wgmma tile needs it, and every rank holds at least one KV head."""
    if family == "llama":
        from chitu_b200.engine import LlamaConfig
        return LlamaConfig(dim=512, n_layers=3, n_heads=4, n_kv_heads=max(2, W), vocab_size=1024, multiple_of=256 * W,
                           ffn_dim_multiplier=None)
    if family == "mixtral":
        from chitu_b200.engine_mixtral import MixtralConfig
        return MixtralConfig(dim=512, n_layers=3, n_heads=4, n_kv_heads=max(2, W), vocab_size=1024,
                             intermediate_dim=512, num_local_experts=4, num_experts_per_tok=2)
    from chitu_b200.engine_deepseek import DeepSeekConfig
    return DeepSeekConfig(vocab_size=1024, dim=512, inter_dim=512 * W, moe_inter_dim=128 * W, n_layers=3,
                          n_dense_layers=1, n_heads=4 * W, n_routed_experts=16, n_activated_experts=4,
                          n_expert_groups=4, n_limited_groups=2, q_lora_rank=256)


def build(v: TPVariant, rank, group, device):
    """Rank `rank`'s engine of the variant: the same seeded norm weights on every rank, the synthetic context, this
    rank's heads of one seeded full-width KV cache, and the variant's start lengths."""
    W, ev = v.world, v.es
    kw = dict(v.engine_kw, max_reqs=BATCH, max_seq_len=ev.max_seq_len, device=device, page_size=ev.page, tp_rank=rank,
              tp_size=W, process_group=group, use_fused_allreduce=False)
    cfg = config(v.family, W)
    if v.family == "llama":
        from chitu_b200.engine import LlamaDecodeEngine as E
    elif v.family == "mixtral":
        from chitu_b200.engine_mixtral import MixtralDecodeEngine as E
    else:
        from chitu_b200.engine_deepseek import DeepSeekDecodeEngine as E
    eng = E(cfg, **kw)
    g = torch.Generator(device=eng.device).manual_seed(5)
    for w in [L[k] for L in eng.layers for k in ES.NORM_KEYS if k in L] + [eng.norm]:
        w.copy_(0.5 + torch.rand(w.shape, generator=g, device=eng.device))
    eng.set_synthetic_context(0)
    if v.family != "deepseek":
        for li in range(cfg.n_layers):
            for ci, cache in enumerate(eng.caches):
                nb, pg, hkv, D = cache.shape[1:]
                gen = torch.Generator(device=eng.device).manual_seed(1000 + 2 * li + ci)
                full = torch.empty(nb, pg, hkv * W, D, device=eng.device).normal_(0, 1, generator=gen)
                cache[li].copy_(full[:, :, rank * hkv:(rank + 1) * hkv].clamp(-448.0, 448.0))
    eng.seq_lens.copy_(torch.tensor(v.starts, dtype=torch.int32))
    return eng


def to(obj, device):
    """obj with every tensor inside it (dicts, lists, tuples) moved to `device`."""
    if isinstance(obj, torch.Tensor):
        return obj.to(device)
    if isinstance(obj, dict):
        return {k: to(x, device) for k, x in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(to(x, device) for x in obj)
    return obj


def shard_state(eng, family):
    """One rank's weights in the reference's layout (LLaMA's w13 un-interleaved), its tables and its caches."""
    layers = (eng.ref_layers() if family == "llama" else
              [{k: t for k, t in L.items() if k not in NOT_SAVED} for L in eng.layers])
    return dict(layers=layers, embed=eng.embed, norm=eng.norm, head=eng.head, block_table=eng.block_table,
                cos=eng.cos_table, sin=eng.sin_table, caches=tuple(c.clone() for c in eng.caches))


# ------------------------------------------------------------------ the sharding map
def _pairs(ws, dim, swap=None):
    """[gate ; up] halves of every rank's tensor along `dim`, concatenated as [gate_0 .. gate_{W-1} ; up_0 ..];
    `swap`: the rank whose gate and up are exchanged (a fault)."""
    n = ws[0].shape[dim] // 2
    gates, ups = [w.narrow(dim, 0, n) for w in ws], [w.narrow(dim, n, n) for w in ws]
    if swap is not None:
        gates[swap], ups[swap] = ups[swap], gates[swap]
    return torch.cat(gates + ups, dim)


def assemble(v: TPVariant, cfg, shards, fault=None):
    """(layers, head) of the full-width model the W ranks' shards assemble, or of a wrong assembly (`fault`, one of
    FAULTS[family])."""
    assert fault is None or fault in FAULTS[v.family], fault
    rev = (lambda xs: xs[::-1])
    keep = (lambda xs: xs)
    swap = 1 if fault == "rank 1's gate / up swapped" else None
    experts = rev if fault == "experts' halves in reverse rank order" else keep
    wo_order = rev if fault == "wo in reverse rank order" else keep
    W = len(shards)
    layers = []
    for li in range(cfg.n_layers):
        Ls = [s["layers"][li] for s in shards]
        full = {k: Ls[0][k] for k in REPLICATED if k in Ls[0]}

        def cat(key, dim, order=keep):
            return torch.cat(order([L[key] for L in Ls]), dim)

        if v.family in ("llama", "mixtral"):
            D, Hq, Hkv = cfg.head_dim, cfg.n_heads // W, cfg.n_kv_heads // W
            q = [L["wqkv"][:Hq * D] for L in Ls]
            k = [L["wqkv"][Hq * D:(Hq + Hkv) * D] for L in Ls]
            val = [L["wqkv"][(Hq + Hkv) * D:] for L in Ls]
            if fault == "q shards swapped, KV not":
                q = q[::-1]
            full["wqkv"] = torch.cat(q + k + val)
            full["wo"] = cat("wo", 1, wo_order)
        if v.family == "llama":
            full["w13"] = _pairs([L["w13"] for L in Ls], 0, swap)
            full["w2"] = cat("w2", 1)
        elif v.family == "mixtral":
            full["w1"] = _pairs(experts([L["w1"] for L in Ls]), 1, swap)
            full["w2"] = cat("w2", 2)
        elif v.family == "deepseek":
            full["wq_b"], full["wq_b_s"] = cat("wq_b", 0), cat("wq_b_s", 0)
            kv_order = rev if fault == "rank 1's wkv_b with rank 0's heads" else keep
            full["wkv_b"], full["wkv_b_s"] = cat("wkv_b", 0, kv_order), cat("wkv_b_s", 0, kv_order)
            full["wo"], full["wo_s"] = cat("wo", 1, wo_order), cat("wo_s", 1, wo_order)
            if "w13" in Ls[0]:
                full["w13"], full["w13_s"] = (_pairs([L[n] for L in Ls], 0, swap) for n in ("w13", "w13_s"))
                full["w2"], full["w2_s"] = cat("w2", 1), cat("w2_s", 1)
            else:
                full["we1"], full["we1_s"] = (_pairs(experts([L[n] for L in Ls]), 1) for n in ("we1", "we1_s"))
                full["we2"], full["we2_s"] = cat("we2", 2), cat("we2_s", 2)
        layers.append(full)
    heads = [s["head"] for s in shards]
    if fault == "head offset by one rank":
        heads = heads[1:] + heads[:1]
    return layers, torch.cat(heads)


def assemble_caches(v: TPVariant, rank_caches):
    """The full caches: the concatenation of the ranks' KV heads, or DeepSeek's replicated latent cache."""
    if v.family == "deepseek":
        return tuple(rank_caches[0])
    return tuple(torch.cat([rc[i] for rc in rank_caches], dim=-2) for i in range(len(rank_caches[0])))


class Assembled:
    """The full-width model, with the attributes `test_engine_steps_gpu.Model` reads from an engine."""

    def __init__(self, v: TPVariant, cfg, shards, fault=None):
        s0 = shards[0]
        self.cfg = cfg
        self.layers, self.head = assemble(v, cfg, shards, fault)
        self.embed, self.norm, self.block_table = s0["embed"], s0["norm"], s0["block_table"]
        self.cos_table, self.sin_table = s0["cos"], s0["sin"]
        if v.family == "deepseek":
            self.H = cfg.n_heads
        else:
            self.Hq, self.Hkv = cfg.n_heads, cfg.n_kv_heads
        if v.family == "mixtral":
            self.topk = cfg.num_experts_per_tok

    def ref_layers(self):
        return self.layers


# ------------------------------------------------------------------ rank by rank, fp64
def _tp_experts(x, w1s, w2s, topk_w, topk_ids, w1_ss=None, w2_ss=None):
    """torch_ref.fused_experts with each expert's intermediate split over the ranks: every rank's down-projection
    partial (fp64, unrounded) is summed before the slot's bf16 rounding, where the full model rounds its whole sum.
    fp8 block-scaled (w8a8) when the scales are given, bf16 otherwise."""
    cd = F64
    T, K1 = x.shape
    c3 = torch.zeros(T, topk_ids.shape[1], K1, dtype=x.dtype, device=x.device)
    fp8 = w1_ss is not None
    if fp8:
        xq, xs = R.group_quant(x)
    for e in torch.unique(topk_ids).tolist():
        tok, slot = (topk_ids == e).nonzero(as_tuple=True)
        y = 0
        for r in range(len(w1s)):
            if fp8:
                a2 = R.silu_and_mul(R.fp8_gemm(xq[tok], xs[tok], w1s[r][e], w1_ss[r][e], x.dtype, cd))
                aq, a_s = R.group_quant(a2)
                y = y + R.fp8_gemm(aq, a_s, w2s[r][e], w2_ss[r][e], cd, cd)
            else:
                a2 = R.silu_and_mul((x[tok].to(cd) @ w1s[r][e].to(cd).T).to(x.dtype))
                y = y + a2.to(cd) @ w2s[r][e].to(cd).T
        c3[tok, slot] = (y * topk_w[tok, slot].to(cd)[:, None]).to(x.dtype)
    return c3.to(cd).sum(dim=1).to(x.dtype)


def _tp_deepseek(cfg, Ls, h, rcaches, lens, table, cos, sin):
    cd, B, eps = F64, h.shape[0], cfg.norm_eps
    C, Rr, dn, dv = cfg.kv_lora_rank, cfg.qk_rope_head_dim, cfg.qk_nope_head_dim, cfg.v_head_dim
    L0 = Ls[0]
    xn = R.rms_norm(h, L0["attn_norm"], eps, cd)
    q_a, kv, k_pe = torch.split(R.fp8_linear(xn, L0["wqkv_a"], L0["wqkv_a_s"], cd), [cfg.q_lora_rank, C, Rr], dim=-1)
    qn = R.rms_norm(q_a.contiguous(), L0["q_norm"], eps, cd)
    part = 0
    for L, (kc,) in zip(Ls, rcaches):
        Hr = L["wq_b"].shape[0] // (dn + Rr)
        q_nope, q_pe = torch.split(R.fp8_linear(qn, L["wq_b"], L["wq_b_s"], cd).view(B, Hr, dn + Rr), [dn, Rr], dim=-1)
        q_pe, k_rot = R.rotary_interleaved(q_pe, k_pe, cos, sin, cd)
        wkv_b = R.weight_dequant(L["wkv_b"], L["wkv_b_s"]).view(Hr, dn + dv, C)
        q_abs = torch.einsum("shd,hdc->shc", q_nope.to(cd), wkv_b[:, :dn].to(cd)).to(BF)
        this_kv = torch.cat([R.rms_norm(kv.contiguous(), L["kv_norm"], eps, cd), k_rot], dim=-1)
        x = R.mla_attn_with_kvcache(q_abs, q_pe.contiguous(), kc, this_kv, lens, table, cfg.softmax_scale, cd)
        o = torch.einsum("bhc,hdc->bhd", x.to(cd), wkv_b[:, -dv:].to(cd)).to(BF)
        oq, o_s = R.act_quant(o.reshape(B, Hr * dv))
        part = part + R.fp8_gemm(oq, o_s, L["wo"], L["wo_s"], cd, cd)
    h = h + part.to(h.dtype)
    xn = R.rms_norm(h, L0["ffn_norm"], eps, cd)
    if "w13" in L0:
        part = 0
        for L in Ls:
            aq, a_s = R.act_quant(R.silu_and_mul(R.fp8_linear(xn, L["w13"], L["w13_s"], cd)))
            part = part + R.fp8_gemm(aq, a_s, L["w2"], L["w2_s"], cd, cd)
        return h + part.to(h.dtype)
    w, idx, _ = R.moe_gate(xn, L0["gate_w"], L0["gate_b"], cfg.n_activated_experts, cfg.n_expert_groups,
                           cfg.n_limited_groups, cfg.score_func, cfg.route_scale)
    w = torch.cat([w, torch.ones_like(w[:, :1])], dim=1)                     # the shared expert, weight 1
    idx = torch.cat([idx, torch.full_like(idx[:, :1], cfg.n_routed_experts)], dim=1)
    return h + _tp_experts(xn, *([L[n] for L in Ls] for n in ("we1", "we2")), w, idx,
                           *([L[n] for L in Ls] for n in ("we1_s", "we2_s")))


def tp_layer(v: TPVariant, cfg, Ls, h, rcaches, lens, full):
    """One layer computed rank by rank in fp64: each rank applies its own shards `Ls[r]` to the common input h and
    appends to its own caches `rcaches[r]`; the row-parallel partials are summed unrounded and rounded where the full
    model rounds its product.  Same roundings as torch_ref's layer of the assembled model otherwise."""
    pos = lens.long().to(full.cos_table.device)
    cos, sin = full.cos_table[pos], full.sin_table[pos]
    if v.family == "deepseek":
        return _tp_deepseek(cfg, Ls, h, rcaches, lens, full.block_table, cos, sin)
    cd, B, eps, W = F64, h.shape[0], cfg.norm_eps, len(Ls)
    D, Hq, Hkv = cfg.head_dim, cfg.n_heads // W, cfg.n_kv_heads // W
    L0 = Ls[0]
    xn = R.rms_norm(h, L0["attn_norm"], eps, cd)
    part = 0
    for L, (kc, vc) in zip(Ls, rcaches):
        qkv = R._lin(xn, L["wqkv"], cd)
        q, k = qkv[:, :Hq * D].reshape(B, Hq, D), qkv[:, Hq * D:(Hq + Hkv) * D].reshape(B, Hkv, D)
        val = qkv[:, (Hq + Hkv) * D:].reshape(B, 1, Hkv, D)
        q, k = R.rotary_interleaved(q, k, cos, sin, cd) if v.family == "llama" else R.rotary_half(q, k, cos, sin)
        o = R.gqa_paged_decode(q.view(B, 1, Hq, D), kc, vc, k.view(B, 1, Hkv, D), val, lens, full.block_table,
                               compute_dtype=cd)
        part = part + o.reshape(B, Hq * D).to(cd) @ L["wo"].to(cd).T
    h = h + part.to(h.dtype)
    xn = R.rms_norm(h, L0["ffn_norm"], eps, cd)
    if v.family == "llama":
        part = 0
        for L in Ls:
            F = L["w13"].shape[0] // 2
            gu = R._lin(xn, L["w13"], cd)
            part = part + (torch.nn.functional.silu(gu[:, :F]) * gu[:, F:]).to(cd) @ L["w2"].to(cd).T
        return h + part.to(h.dtype)
    probs = torch.softmax(R._lin(xn, L0["gate_w"], cd), dim=-1, dtype=cd)
    w, idx = torch.topk(probs, cfg.num_experts_per_tok, dim=-1)
    w = w / w.sum(dim=-1, keepdim=True)
    return h + _tp_experts(xn, [L["w1"] for L in Ls], [L["w2"] for L in Ls], w.to(xn.dtype), idx)


# ------------------------------------------------------------------ the CPU tests
def cpu_shards(v: TPVariant):
    """The W ranks' shard states, built on the CPU (weights, caches, tables; no kernel runs)."""
    from test_engine_calls_cpu import Recorder, _patched
    with _patched(Recorder()):
        return [shard_state(build(v, r, None, "cpu"), v.family) for r in range(v.world)]


@pytest.mark.parametrize("name", CPU_VARIANTS)
def test_rank_by_rank_equals_assembled_model(name):
    """At every step's lengths, every layer and the logits computed rank by rank from each rank's own shards agree
    with the reference of the assembled model to 1e-12, and so do the rows each rank appends to its caches."""
    v = VARIANTS[name]
    cfg = config(v.family, v.world)
    shards = cpu_shards(v)
    full = Assembled(v, cfg, shards)
    m = ES.Model(v.es, full)
    caches0 = assemble_caches(v, [s["caches"] for s in shards])
    worst = 0.0
    for t in range(STEPS):
        lens = torch.tensor(v.starts, dtype=torch.int32) + t
        h = full.embed[ES.step_tokens(t, cfg.vocab_size)]
        for li in range(cfg.n_layers):
            fc = [c[li].clone() for c in caches0]
            ref = m.layer(li, h, fc, lens)
            rc = [[c[li].clone() for c in s["caches"]] for s in shards]
            got = tp_layer(v, cfg, [s["layers"][li] for s in shards], h, rc, lens, full)
            worst = max(worst, ES.rel_err(got.double() - h.double(), ref.double() - h.double()))
            if v.family == "deepseek":
                assert all(torch.equal(r[0].view(torch.uint8), fc[0].view(torch.uint8)) for r in rc), (t, li)
            else:
                for i, c in enumerate(assemble_caches(v, rc)):
                    assert torch.equal(c.view(torch.uint8), fc[i].view(torch.uint8)), (t, li)
            h = ref
        tp_logits = torch.cat([R.final_logits(h, full.norm, s["head"], cfg.norm_eps, F64) for s in shards], dim=1)
        assert torch.equal(tp_logits, m.logits(h)), t
    print(f"{name}: rank by rank vs assembled, worst layer err {worst:.1e}")
    assert worst <= 1e-12


@pytest.mark.parametrize("name", CPU_VARIANTS)
def test_bound_rejects_assembly_faults(name):
    """Each assembly fault of FAULTS pushes some layer (the head's: the logits) of the run past the bound of
    `test_tp_engine_steps`, as that test would then fail if the engines computed the faulty assembly."""
    v = VARIANTS[name]
    cfg = config(v.family, v.world)
    shards = cpu_shards(v)
    full = Assembled(v, cfg, shards)
    m = ES.Model(v.es, full)
    bad = {f: ES.Model(v.es, Assembled(v, cfg, shards, f)) for f in FAULTS[v.family]}
    caches0 = assemble_caches(v, [s["caches"] for s in shards])
    gen = torch.Generator().manual_seed(9)
    ratio = {f: [0.0] * STEPS for f in bad}
    for t in range(STEPS):
        lens = torch.tensor(v.starts, dtype=torch.int32) + t
        h = full.embed[ES.step_tokens(t, cfg.vocab_size)]
        for li in range(cfg.n_layers):
            caches, routes = [c[li].clone() for c in caches0], []
            ref = m.layer(li, h, caches, lens, routes=routes)
            floor, _ = ES.layer_floor(m, li, h, [c[li] for c in caches0], lens, ref, routes, gen)
            d_ref = ref.double() - h.double()
            for f, mb in bad.items():
                out = mb.layer(li, h, [c[li].clone() for c in caches0], lens)
                ratio[f][t] = max(ratio[f][t], ES.rel_err(out.double() - h.double(), d_ref) / ES.bound(floor))
            h = ref
        ref = m.logits(h)
        floor = max(ES.rel_err(m.logits(ES.ulp_perturb(h, gen)), ref) for _ in range(ES.FLOOR_SEEDS))
        for f, mb in bad.items():
            ratio[f][t] = max(ratio[f][t], ES.rel_err(mb.logits(h), ref) / ES.bound(floor))
    for f, r in ratio.items():
        print(f"{name}: {f}: err / bound per step " + " ".join(f"{x:.1f}" for x in r))
    missed = [f for f, r in ratio.items() if max(r) <= 1.0]
    assert not missed, f"the bound does not reject {missed}"


# ------------------------------------------------------------------ the GPU test: W ranks as processes on one GPU
def _stage_collectives(group, world):
    """'cuda' when this torch's gloo runs all_reduce and all_gather_into_tensor on CUDA tensors; otherwise both are
    replaced, in this process only, by calls that stage through host copies, and 'host'."""
    import torch.distributed as dist
    try:
        x = torch.ones(4, dtype=BF, device="cuda")
        dist.all_reduce(x, group=group)
        out = torch.empty(2 * world, device="cuda")
        dist.all_gather_into_tensor(out, torch.ones(2, device="cuda"), group=group)
        torch.cuda.synchronize()
        assert bool((x == world).all()) and bool((out == 1).all())
        return "cuda"
    except (RuntimeError, ValueError):
        pass
    all_reduce, all_gather = dist.all_reduce, dist.all_gather_into_tensor

    def staged_all_reduce(t, op=dist.ReduceOp.SUM, group=None, async_op=False):
        hst = t.cpu()
        all_reduce(hst, op=op, group=group)
        t.copy_(hst)

    def staged_all_gather(out, inp, group=None, async_op=False):
        hst = torch.empty(out.shape, dtype=out.dtype)
        all_gather(hst, inp.cpu(), group=group)
        out.copy_(hst)

    dist.all_reduce, dist.all_gather_into_tensor = staged_all_reduce, staged_all_gather
    return "host"


def _run_verify(eng):
    """max_draft + 1 verify passes over the same positions (seq_lens rewound between them): pass p's first p drafts
    are the greedy targets the earlier passes found, the rest seeded random tokens."""
    B, k, vocab = eng.B, eng.max_draft, eng.cfg.vocab_size
    tok = ES.step_tokens(STEPS, vocab)
    chain = torch.randint(0, vocab, (B, k), generator=torch.Generator().manual_seed(300))
    n_draft = torch.tensor(VERIFY_N_DRAFT[:B], dtype=torch.int32)
    recs = []
    for p in range(k + 1):
        lens = eng.seq_lens.clone()
        out, acc = eng.verify(tok.pin_memory(), chain.clone().pin_memory(), n_draft.pin_memory())
        torch.cuda.synchronize()
        target = eng.target.cpu()
        recs.append(dict(drafts=chain.clone(), n_draft=n_draft.clone(), lens=lens.cpu(), target=target, out_tokens=out,
                         accepted=acc, seq_lens=eng.seq_lens.cpu(), next_tokens=eng.next_tokens.cpu(),
                         logits=eng.logits[:B * (k + 1)].cpu()))
        if p < k:
            chain[:, p] = target[:, p]
            eng.seq_lens.copy_(lens)
    return recs


def _run_variant(v: TPVariant, rank, group):
    eng = build(v, rank, group, "cuda:0")
    out = dict(static=to(shard_state(eng, v.family), "cpu"), steps=[])
    B, vocab = eng.B, eng.cfg.vocab_size
    for t in range(STEPS):
        tok, lens, head, rec = ES.step_tokens(t, vocab), eng.seq_lens.clone(), eng.head, {}
        if t == TIE_STEP:            # the same head shard on every rank: every row's maximum ties across the shards
            g = torch.Generator(device=eng.device).manual_seed(77)
            eng.head = (torch.randn(head.shape, generator=g, device=eng.device) * 0.02).to(BF)
            rec["tie_head"] = eng.head.cpu()
        eng.capture_h = []
        eng.decode(tok.pin_memory())
        hs, eng.capture_h, eng.head = eng.capture_h, None, head
        torch.cuda.synchronize()
        # (a verify engine's residual stream holds B * (max_draft + 1) rows; a decode step uses the first B)
        rec.update(tokens=tok, lens=lens.cpu(), hs=[x[:B].cpu() for x in hs], caches=[c.cpu() for c in eng.caches],
                   logits=eng.logits[:B].cpu(), next_tokens=eng.next_tokens.cpu(), seq_lens=eng.seq_lens.cpu())
        if hasattr(eng, "gate_i_all"):
            rec.update(gate_i=eng.gate_i_all.cpu(), gate_w=eng.gate_w_all.cpu())
        out["steps"].append(rec)
    if v.max_draft:
        out["verify"] = _run_verify(eng)
    return out


def _worker(rank, world, names, tmp):
    """One rank: every variant in `names`, each saved to tmp/<name>.rank<r>.pt; a failure's traceback to
    tmp/error.rank<r>.txt.  The group is destroyed on every path."""
    import torch.distributed as dist
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", store=dist.FileStore(os.path.join(tmp, "store"), world), rank=rank,
                                world_size=world, timeout=datetime.timedelta(seconds=GLOO_TIMEOUT_S))
        path = _stage_collectives(dist.group.WORLD, world)
        for name in names:
            torch.save(_run_variant(VARIANTS[name], rank, dist.group.WORLD), os.path.join(tmp, f"{name}.rank{rank}.pt"))
        torch.save(dict(collectives=path), os.path.join(tmp, f"done.rank{rank}.pt"))
    except BaseException:
        with open(os.path.join(tmp, f"error.rank{rank}.txt"), "w") as f:
            f.write(traceback.format_exc())
        raise
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _same(ts, what):
    for r, t in enumerate(ts[1:], 1):
        a, b = ts[0], t
        if a.is_floating_point():
            a, b = a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8)
        assert torch.equal(a, b), f"{what}: rank {r} differs from rank 0"


def check_variant(name, rs, dev):
    """Checks 1-5 of the module docstring on the W ranks' results `rs` of one variant; returns the bound failures
    (the other checks assert)."""
    v = VARIANTS[name]
    W, ev, fam = v.world, v.es, v.family
    cfg = config(fam, W)
    st = [to(r["static"], dev) for r in rs]
    for key in ("embed", "norm", "block_table", "cos", "sin"):
        _same([s[key] for s in st], key)
    for li in range(cfg.n_layers):
        for key in REPLICATED:
            if key in st[0]["layers"][li]:
                _same([s["layers"][li][key] for s in st], f"layer {li} {key}")
    full = Assembled(v, cfg, st)
    m = ES.Model(ev, full)
    caches = assemble_caches(v, [s["caches"] for s in st])
    gen = torch.Generator(device=dev).manual_seed(9)
    worst = dict(kv=0.0, layer=(0.0, 0.0, None), logits=(0.0, 0.0, None))
    failures = []
    for t in range(STEPS):
        steps = [to(r["steps"][t], dev) for r in rs]
        s0 = steps[0]
        for key in ("lens", "next_tokens", "seq_lens", "gate_i", "gate_w"):
            if key in s0:
                _same([s[key] for s in steps], f"step {t} {key}")
        for li in range(cfg.n_layers + 1):
            _same([s["hs"][li] for s in steps], f"step {t} residual stream entering layer {li}")
        if fam == "deepseek":
            for i in range(len(s0["caches"])):
                _same([s["caches"][i] for s in steps], f"step {t} latent cache")
        hs, lens = s0["hs"], s0["lens"]
        assert torch.equal(s0["seq_lens"], lens + 1)
        after = assemble_caches(v, [s["caches"] for s in steps])
        if fam == "deepseek":           # the shared expert: the last routing slot of every MoE token, weight 1
            nd = cfg.n_dense_layers
            assert bool((s0["gate_i"][nd:, :, -1] == cfg.n_routed_experts).all())
            assert bool((s0["gate_w"][nd:, :, -1] == 1).all())
        for li in range(cfg.n_layers):
            before = [c[li] for c in caches]
            ref_c, routes = [c.clone() for c in before], []
            ref = m.layer(li, hs[li], ref_c, lens, routes=routes)
            for a, b4, rc in zip((c[li] for c in after), before, ref_c):
                worst["kv"] = max(worst["kv"], ES.check_append(a, b4, rc, full.block_table, lens, ev.page,
                                                               2.0 ** -5 if fam == "deepseek" else 2.0 ** -8))
            floor, noise = ES.layer_floor(m, li, hs[li], before, lens, ref, routes, gen)
            moe = m.k is not None and (fam == "mixtral" or li >= cfg.n_dense_layers)
            rows = ES.kept_rows(s0["gate_i"][li] if moe else None, routes, m.k, noise if fam == "deepseek" else None)
            err = ES.rel_err(hs[li + 1].double() - hs[li].double(), ref.double() - hs[li].double(), rows)
            if err > worst["layer"][0]:
                worst["layer"] = (err, floor, (t, li))
            if err > ES.bound(floor):
                failures.append(f"{name} step {t} layer {li}: err {err:.3e} > bound {ES.bound(floor):.3e} "
                                f"(floor {floor:.3e})")
        caches = after
        head = torch.cat([s["tie_head"] for s in steps]) if "tie_head" in s0 else full.head
        logits = torch.cat([s["logits"] for s in steps], dim=1)
        ref = R.final_logits(hs[-1], full.norm, head, cfg.norm_eps, F64)
        err = ES.rel_err(logits.double(), ref)
        floor = max(ES.rel_err(R.final_logits(ES.ulp_perturb(hs[-1], gen), full.norm, head, cfg.norm_eps, F64), ref)
                    for _ in range(ES.FLOOR_SEEDS))
        if err > worst["logits"][0]:
            worst["logits"] = (err, floor, t)
        if err > ES.bound(floor):
            failures.append(f"{name} step {t} logits: err {err:.3e} > bound {ES.bound(floor):.3e} (floor {floor:.3e})")
        lg = logits.float()
        assert torch.equal(s0["next_tokens"], lg.argmax(dim=-1)), \
            f"step {t}: next tokens are not the first maximal index of the concatenated logits"
        if "tie_head" in s0:
            top = lg.amax(dim=-1, keepdim=True)
            ranks_at_max = (lg == top).view(BATCH, W, -1).any(dim=-1).sum(dim=-1)
            assert bool((ranks_at_max == W).all()), f"step {t}: the maxima do not tie across the shards"
            assert bool((s0["next_tokens"] < cfg.vocab_size // W).all()), "a tie did not go to the lowest global index"
    if v.max_draft:
        k = v.max_draft
        for p, recs in enumerate(zip(*[r["verify"] for r in rs])):
            for key in ("drafts", "target", "out_tokens", "accepted", "seq_lens", "next_tokens"):
                _same([rec[key] for rec in recs], f"verify pass {p} {key}")
            r0 = recs[0]
            lg = torch.cat([rec["logits"] for rec in recs], dim=1).float()
            target = lg.argmax(dim=-1).view(BATCH, k + 1)
            assert torch.equal(r0["target"], target), f"verify pass {p}: target is not the argmax of the logits"
            want = accept_rule(target, r0["drafts"], r0["n_draft"], r0["lens"])
            for got, w, what in zip((r0["out_tokens"], r0["accepted"], r0["next_tokens"], r0["seq_lens"]), want,
                                    ("out_tokens", "accepted", "next_tokens", "seq_lens")):
                assert torch.equal(got, w), f"verify pass {p}: {what} is not greedy acceptance"
        assert torch.equal(recs[0]["accepted"], recs[0]["n_draft"]), "the last pass did not accept the greedy chain"
    print(f"{name}: worst layer err {worst['layer'][0]:.3e} (floor {worst['layer'][1]:.3e}, step/layer "
          f"{worst['layer'][2]})  worst logits err {worst['logits'][0]:.3e} (floor {worst['logits'][1]:.3e})  "
          f"appended KV {worst['kv']:.2f} roundings")
    assert worst["kv"] <= 1.0, f"{name}: an appended KV value is {worst['kv']:.2f} roundings from the reference's"
    return failures


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_tp_engine_steps(world):
    import torch.multiprocessing as mp
    names = [n for n, v in VARIANTS.items() if v.world == world]
    ctx = mp.get_context("spawn")
    t0 = time.monotonic()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_worker, args=(r, world, names, tmp)) for r in range(world)]
        try:
            for p in procs:
                p.start()
            deadline = time.monotonic() + JOIN_S
            # a rank that fails ends the run: its peers would otherwise wait in a collective until the gloo timeout
            while any(p.is_alive() for p in procs) and time.monotonic() < deadline:
                if any(p.exitcode not in (None, 0) for p in procs):
                    break
                time.sleep(0.2)
        finally:
            for p in procs:
                if p.is_alive():
                    p.kill()
                p.join(10)
        errors = [open(os.path.join(tmp, f)).read() for f in sorted(os.listdir(tmp)) if f.startswith("error.")]
        assert not errors, "\n".join(errors)
        assert [p.exitcode for p in procs] == [0] * world, [p.exitcode for p in procs]
        paths = {torch.load(os.path.join(tmp, f"done.rank{r}.pt"))["collectives"] for r in range(world)}
        t_run = time.monotonic() - t0
        failures = []
        for name in names:
            rs = [torch.load(os.path.join(tmp, f"{name}.rank{r}.pt")) for r in range(world)]
            failures += check_variant(name, rs, "cuda:0")
    print(f"W = {world}: gloo collectives on {paths} tensors; ranks {t_run:.0f} s, checks "
          f"{time.monotonic() - t0 - t_run:.0f} s")
    assert not failures, "\n".join(failures)
