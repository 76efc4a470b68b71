"""Mixtral-8x7B decode step (BASELINE.json configs[2]): hf-llama attention (models/model_hf_llama.py:139-252: merged qkv,
half-split rotary, paged GQA decode, o_proj) + the sparse-MoE block of models/model_hf_mixtral.py:51-96 routed through
the fused experts (SURVEY a21): softmax(fp32) -> top-2 -> renormalise -> grouped bf16 expert GEMMs, ONE reduce per layer
where the reference all-reduces once per expert (FeedForward.down, 8 per layer).

Tensor parallel where the reference shards (SURVEY §8e): heads (8 q / 2 kv heads per rank at tp=4), every expert's
intermediate dim (gate/up chunked separately then concatenated, models/model.py:344-350); the router is computed
replicated (the reference splits its K dim over the ranks and all-reduces 8 logits: same sum, different order).

weight_format="w4a16" holds qkv, o and the experts as 4-bit groups of 128 (quantize/w4a16.py's round-to-nearest rule
applied to the same synthetic weights, one layer at a time as it is generated, so the bf16 model never exists whole: at
tp_size=1 the full Mixtral-8x7B fits on one 80 GB GPU) and runs them through chitu_b200_w4a16_gemm and
chitu_b200_fused_experts_w4a16; router, embedding, head, norms, rotary and attention stay bf16.  The 4-bit GEMM has no
push epilogue, so it runs on one GPU or in shard mode.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from . import _lib
from ._lib import check, current_stream, ptr
from .engine import DecodeEngine

BF = torch.bfloat16


@dataclass
class MixtralConfig:
    """chitu/config/models/Mixtral-8x7B-Instruct-v0.1.yaml:6-17."""
    dim: int = 4096
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: int = 8
    vocab_size: int = 32000
    intermediate_dim: int = 14336
    norm_eps: float = 1e-5
    rope_theta: float = 1000000.0
    num_local_experts: int = 8
    num_experts_per_tok: int = 2

    @property
    def head_dim(self):
        return self.dim // self.n_heads


MIXTRAL_8X7B = MixtralConfig()


class MixtralDecodeEngine(DecodeEngine):
    WEIGHT_FORMATS = ("bf16", "w4a16")
    QUANT_LINEARS = ("wqkv", "wo", "w1", "w2")

    def __init__(self, cfg: MixtralConfig, max_reqs: int, max_seq_len: int, device="cuda:0", page_size: int = 256,
                 seed: int = 0, tp_rank: int = 0, tp_size: int = 4, process_group=None, use_fused_allreduce: bool = True,
                 weight_format: str = "bf16"):
        D = cfg.head_dim
        T = tp_size
        self._set_weight_format(weight_format, tp_size, process_group)
        assert cfg.n_heads % T == 0 and cfg.n_kv_heads % T == 0 and cfg.intermediate_dim % (128 * T) == 0
        self.Hq, self.Hkv, self.D = cfg.n_heads // T, cfg.n_kv_heads // T, D
        self.F = cfg.intermediate_dim // T
        self.E, self.topk = cfg.num_local_experts, cfg.num_experts_per_tok
        super().__init__(cfg, max_reqs, max_seq_len, device, page_size, seed, tp_rank, tp_size, process_group,
                         use_fused_allreduce, attn_ws=(self.Hq, D, 64), lin_n=max(cfg.vocab_size // T, cfg.dim))
        dev, g, g_rep, rnd = self.device, self.g, self.g_rep, self._rnd
        dim = cfg.dim
        self.embed = rnd(g_rep, cfg.vocab_size, dim)
        self.layers = []
        for _ in range(cfg.n_layers):
            lw = dict(
                attn_norm=torch.ones(dim, dtype=BF, device=dev), ffn_norm=torch.ones(dim, dtype=BF, device=dev),
                wqkv=rnd(g, (self.Hq + 2 * self.Hkv) * D, dim), wo=rnd(g, dim, self.Hq * D),
                gate_w=rnd(g_rep, self.E, dim, scale=0.05),
                # experts stacked like fused_experts expects: w1 = [gate ; up] (merge_gate_up), w2 = down
                w1=rnd(g, self.E, 2 * self.F, dim), w2=rnd(g, self.E, dim, self.F))
            self.layers.append(self._quantized(lw))
        self.norm = torch.ones(dim, dtype=BF, device=dev)
        self.head = rnd(g, cfg.vocab_size // T, dim)
        self._gqa_buffers(BF, max_reqs)
        # hf rotary: cos/sin [pos, D/2] in the model dtype, half-split layout (ops.py:243-308 "hf-llama")
        freqs = 1.0 / (cfg.rope_theta ** (torch.arange(0, D, 2).float() / D))
        self._rope_tables(torch.outer(torch.arange(max_seq_len * 2, dtype=torch.float32), freqs), BF)
        # softmax over the E experts -> top-2 -> renormalise (model_hf_mixtral.py:57-64)
        self._init_moe(n_routed=self.E, topk=self.topk, slots=self.topk, n_stacked=self.E, n1=2 * self.F, score_mode=2)

    def _decode_layers(self):
        lib, B, D = self.lib, self.B, self.D
        st = current_stream()
        h, h2 = self.h, self.h2
        qkv_w = (self.Hq + 2 * self.Hkv) * D
        n_layers = len(self.layers)
        self._norm(h, self.layers[0]["attn_norm"], self.xn)
        for li, lw in enumerate(self.layers):
            if self.capture_h is not None:
                self.capture_h.append(h.clone())
            next_norm = self.layers[li + 1]["attn_norm"] if li + 1 < n_layers else self.norm
            self._layer_linear(self.xn, lw, "wqkv", self.qkv, B)
            q = self.qkv[:, : self.Hq * D]
            k = self.qkv[:, self.Hq * D: (self.Hq + self.Hkv) * D]
            # apply_rotary_pos_emb(..., "hf-llama") on the q / k views of the merged qkv output
            check(lib.chitu_b200_rotary_half_strided(ptr(q), qkv_w, ptr(self.q_rot), ptr(self.cos), ptr(self.sin), B, self.Hq, D,
                                                     _lib.CB_BF16, st), "rotary_half q")
            check(lib.chitu_b200_rotary_half_strided(ptr(k), qkv_w, ptr(self.k_rot), ptr(self.cos), ptr(self.sin), B, self.Hkv, D,
                                                     _lib.CB_BF16, st), "rotary_half k")
            self._gqa_attention(li, self.q_rot, self.k_rot)
            self._row_parallel(lambda out, res: self._layer_linear(self.attn_out, lw, "wo", out, B, residual=res),
                               lambda: self.comm.linear_push(self.attn_out, lw["wo"], B, self.lin_ws),
                               h, h2, lw["ffn_norm"], y=self.xn)
            # ---- sparse MoE block (model_hf_mixtral.py:51-96) through the fused experts ----
            self._moe_block(li, h2, h, next_norm, y=self.xn)
        if self.capture_h is not None:
            self.capture_h.append(h.clone())

    def ref_layers(self):
        """The layer weights as the reference multiplies them (the 4-bit ones dequantised) for the oracle side of the
        tests."""
        return [self._dequantized(lw) for lw in self.layers]

    def algorithmic_bytes(self, seq_len: int, distinct: float) -> int:
        """SURVEY §8d: every attention weight byte once, each DISTINCT expert once, KV rows once, bf16 head + router.
        The weights count the bytes of the tensors the engine holds (4-bit ones: the packed weight, its bf16 scales and
        its uint8 zeros)."""
        c, D, lw = self.cfg, self.D, self.layers[0]

        def nbytes(name):
            w = lw[name]
            return sum(t.nbytes for t in w) if isinstance(w, tuple) else w.nbytes

        attn = nbytes("wqkv") + nbytes("wo")
        expert = (nbytes("w1") + nbytes("w2")) // self.E
        kv = self.B * (seq_len + 1) * 2 * self.Hkv * D * 2
        return int(c.n_layers * (attn + distinct * expert + kv + self.E * c.dim * 2) + self.head.numel() * 2)


def run_bench(args, time_engine, ClockSampler, peaks):
    """bench.py --workload mixtral: Mixtral-8x7B bf16 fused-MoE decode, tp = WORLD_SIZE ranks (BASELINE configs[2]: tp=4,
    bs=16); on one GPU: one rank's tp=4 shard without collectives."""
    import json
    import os

    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    pg = None
    tp = world if world > 1 else (args.tp or 4)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(dev))
        pg = dist.group.WORLD
    cfg = MIXTRAL_8X7B if args.layers <= 0 else MixtralConfig(n_layers=args.layers)
    S = args.seq
    peak, peak_src = peaks()
    out = {}
    for B in (args.bs, 1):
        eng = MixtralDecodeEngine(cfg, max_reqs=B, max_seq_len=S + max(512, args.steps + args.warmup + 128), device=dev,
                                  tp_rank=rank if world > 1 else 0, tp_size=tp, process_group=pg,
                                  use_fused_allreduce=not args.nccl_allreduce)
        eng.set_synthetic_context(S)
        eng.capture()
        sampler = ClockSampler(local) if rank == 0 else None
        ms, e2e_ms, clocks = time_engine(eng, B, S, args, world, dev, sampler, label=f"mixtral_bs{B}")
        distinct = eng.distinct_experts_per_layer()
        nbytes = eng.algorithmic_bytes(S, distinct)
        out[B] = dict(ms=ms, e2e_ms=e2e_ms, distinct=distinct, bytes=nbytes, launches=int(eng.launches_per_step), clocks=clocks)
        del eng
        torch.cuda.empty_cache()
    if rank != 0:
        return
    B = args.bs
    r = out[B]
    gbs = r["bytes"] / (r["ms"] * 1e-3) / 1e9
    line = {"metric": f"decode tokens/s at bs={B} (Mixtral-8x7B bf16 fused-MoE paged-KV decode, tp={tp}, seq={S})",
            "value": B / (r["ms"] * 1e-3), "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": r["ms"], "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "bf16",
            "data": "synthetic",
            "config": {"workload": f"Mixtral-8x7B bf16, softmax top-2 router -> grouped wgmma expert GEMMs, bs={B} seq={S} page=256, "
                                   f"{cfg.n_layers} layers, tp={tp}" + ("" if world > 1 else " (one rank's shard on 1 GPU, no collectives)"),
                       "global_batch": B, "seq_len": S, "parallelism": f"tp{tp}", "cuda_graph": True,
                       "distinct_experts_per_layer": r["distinct"],
                       "l2": "inputs larger than L2: %.1f GB streamed per step" % (r["bytes"] / 1e9)},
            "bs1": {"value": 1 / (out[1]["ms"] * 1e-3), "ms_per_step": out[1]["ms"], "distinct_experts_per_layer": out[1]["distinct"],
                    "hbm_frac_of_step_roofline": out[1]["bytes"] / (out[1]["ms"] * 1e-3) / 1e9 / peak},
            "e2e": {"value": B / (r["e2e_ms"] * 1e-3), "unit": "tokens/s", "h2d_bytes_per_step": B * 8, "d2h_bytes_per_step": B * 8},
            "gpu_launches": r["launches"] * args.steps, "launches_per_step": r["launches"], "clocks": r["clocks"],
            "roofline": {"bound": "hbm", "achieved": gbs, "peak": peak, "unit": "GB/s", "frac": gbs / peak, "traffic": None,
                         "kernel": "whole decode step (per-rank algorithmic bytes / step time)", "peak_source": peak_src,
                         "step_algorithmic_bytes": r["bytes"]}}
    print(json.dumps(line))
