"""Mixtral-8x7B decode step (BASELINE.json configs[2]): hf-llama attention (models/model_hf_llama.py:139-252: merged qkv,
half-split rotary, paged GQA decode, o_proj) + the sparse-MoE block of models/model_hf_mixtral.py:51-96 routed through
the fused experts (SURVEY a21): softmax(fp32) -> top-2 -> renormalise -> grouped bf16 expert GEMMs, ONE reduce per layer
where the reference all-reduces once per expert (FeedForward.down, 8 per layer).

Tensor parallel where the reference shards (SURVEY §8e): heads (8 q / 2 kv heads per rank at tp=4), every expert's
intermediate dim (gate/up chunked separately then concatenated, models/model.py:344-350); the router is computed
replicated (the reference splits its K dim over the ranks and all-reduces 8 logits: same sum, different order).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from . import _lib
from ._lib import check, current_stream, ptr
from .tensor_parallel import global_argmax

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


class MixtralDecodeEngine:
    def __init__(self, cfg: MixtralConfig, max_reqs: int, max_seq_len: int, device="cuda:0", page_size: int = 256,
                 seed: int = 0, tp_rank: int = 0, tp_size: int = 4, process_group=None, use_fused_allreduce: bool = True):
        self.cfg, self.B, self.device = cfg, max_reqs, torch.device(device)
        self.tp_rank, self.tp_size, self.pg = tp_rank, tp_size, process_group
        self.lib = _lib.load()
        D = cfg.head_dim
        T = tp_size
        assert cfg.n_heads % T == 0 and cfg.n_kv_heads % T == 0 and cfg.intermediate_dim % (128 * T) == 0
        self.Hq, self.Hkv, self.D = cfg.n_heads // T, cfg.n_kv_heads // T, D
        self.F = cfg.intermediate_dim // T
        self.E, self.topk = cfg.num_local_experts, cfg.num_experts_per_tok
        self.page = page_size
        self.max_blocks = max_seq_len // page_size + 1
        nblk = self.max_blocks * max_reqs
        dev = self.device
        g = torch.Generator(device=dev).manual_seed(seed + 1000 * tp_rank)
        g_rep = torch.Generator(device=dev).manual_seed(seed + 7)

        def rnd(gen, *shape, scale=0.02):
            return (torch.randn(*shape, generator=gen, dtype=torch.float32, device=dev) * scale).to(BF)

        dim = cfg.dim
        self.embed = rnd(g_rep, cfg.vocab_size, dim)
        self.layers = []
        for _ in range(cfg.n_layers):
            self.layers.append(dict(
                attn_norm=torch.ones(dim, dtype=BF, device=dev), ffn_norm=torch.ones(dim, dtype=BF, device=dev),
                wqkv=rnd(g, (self.Hq + 2 * self.Hkv) * D, dim), wo=rnd(g, dim, self.Hq * D),
                gate_w=rnd(g_rep, self.E, dim, scale=0.05),
                # experts stacked like fused_experts expects: w1 = [gate ; up] (merge_gate_up), w2 = down
                w1=rnd(g, self.E, 2 * self.F, dim), w2=rnd(g, self.E, dim, self.F)))
        self.norm = torch.ones(dim, dtype=BF, device=dev)
        self.head = rnd(g, cfg.vocab_size // T, dim)
        self.k_cache = torch.zeros(cfg.n_layers, nblk, page_size, self.Hkv, D, dtype=BF, device=dev)
        self.v_cache = torch.zeros_like(self.k_cache)
        self.block_table = torch.zeros(max_reqs, self.max_blocks, dtype=torch.int32, device=dev)
        self.seq_lens = torch.zeros(max_reqs, dtype=torch.int32, device=dev)
        # hf rotary: cos/sin [pos, D/2] in the model dtype, half-split layout (ops.py:243-308 "hf-llama")
        freqs = 1.0 / (cfg.rope_theta ** (torch.arange(0, D, 2).float() / D))
        ang = torch.outer(torch.arange(max_seq_len * 2, dtype=torch.float32), freqs)
        self.cos_table, self.sin_table = ang.cos().to(BF).to(dev), ang.sin().to(BF).to(dev)
        B = max_reqs
        z = lambda *s, dt=BF: torch.zeros(*s, dtype=dt, device=dev)
        self.tokens = torch.zeros(B, dtype=torch.int64, device=dev)
        self.cos, self.sin = z(B, D // 2), z(B, D // 2)
        self.h, self.h2, self.xn, self.y = z(B, dim), z(B, dim), z(B, dim), z(B, dim)
        self.qkv = z(B, (self.Hq + 2 * self.Hkv) * D)
        self.q_rot, self.k_rot = z(B, self.Hq, D), z(B, self.Hkv, D)
        self.attn_out = z(B, self.Hq * D)
        self.gate_w_all = z(cfg.n_layers, B, self.topk)
        self.gate_i_all = torch.zeros(cfg.n_layers, B, self.topk, dtype=torch.int64, device=dev)
        self.logits = z(B, cfg.vocab_size // T)
        self.next_tokens = torch.zeros(B, dtype=torch.int64, device=dev)
        self.tp_gather = (torch.empty(T, B, 2, dtype=torch.float32, device=dev) if (process_group is not None and T > 1) else None)
        lib = self.lib
        self.attn_ws = torch.zeros(lib.chitu_b200_attn_workspace_bytes(B, self.Hq, D, 64), dtype=torch.uint8, device=dev)
        self.lin_ws = torch.zeros(max(lib.chitu_b200_linear_workspace_bytes(B, max(cfg.vocab_size // T, dim)), 256),
                                  dtype=torch.uint8, device=dev)
        self.moe_ws = torch.zeros(lib.chitu_b200_moe_workspace_bytes(B, self.topk, self.E, 2 * self.F, dim), dtype=torch.uint8,
                                  device=dev)
        self.gate_ws = torch.zeros(lib.chitu_b200_moe_gate_workspace_bytes(B, self.E), dtype=torch.uint8, device=dev)
        self.max_seq_len = max_seq_len
        self.graph = None
        self.launches_per_step = 0
        self.comm = None
        if T > 1 and process_group is not None and use_fused_allreduce:
            from .comm import FusedAllReduce
            self.comm = FusedAllReduce(process_group, max_reqs, dim, self.device)
        import os
        # all-reduce started from the producing kernel's epilogue (csrc/comm.cu push mode); 0 = the pull kernel
        self.ar_push = os.environ.get("CHITU_B200_AR_PUSH", "1") != "0"

    def set_synthetic_context(self, seq_len: int, seed: int = 2):
        g = torch.Generator(device="cpu").manual_seed(seed)
        gd = torch.Generator(device=self.device).manual_seed(seed + 11)
        nblk = self.k_cache.shape[1]
        self.block_table.copy_(torch.randperm(nblk, generator=g).to(torch.int32).view(self.B, self.max_blocks))
        self.seq_lens.fill_(seq_len)
        for l in range(self.cfg.n_layers):
            self.k_cache[l].normal_(0, 1, generator=gd)
            self.v_cache[l].normal_(0, 1, generator=gd)

    def _linear(self, x, w, y, M, residual=None):
        N, K = w.shape
        check(self.lib.chitu_b200_linear_bf16(ptr(x), ptr(w), None, ptr(residual), ptr(y), M, N, K, _lib.CB_BF16,
                                              ptr(self.lin_ws), self.lin_ws.numel(), 0, current_stream()), "linear_bf16")

    def _rmsnorm(self, x, w, y, M):
        check(self.lib.chitu_b200_rmsnorm(ptr(x), ptr(w), ptr(y), M, self.cfg.dim, self.cfg.norm_eps, _lib.CB_BF16,
                                          current_stream()), "rmsnorm")

    def _step_body(self):
        lib, B, D, cfg = self.lib, self.B, self.D, self.cfg
        st = current_stream()
        tp_on = self.pg is not None and self.tp_size > 1
        torch.index_select(self.cos_table, 0, self.seq_lens, out=self.cos)
        torch.index_select(self.sin_table, 0, self.seq_lens, out=self.sin)
        check(lib.chitu_b200_embedding(ptr(self.tokens), ptr(self.embed), ptr(self.h), B, cfg.dim, 0, cfg.vocab_size,
                                       _lib.CB_BF16, st), "embedding")
        h, h2 = self.h, self.h2
        qkv_w = (self.Hq + 2 * self.Hkv) * D
        n_layers = len(self.layers)

        def reduce_add_norm(partial, residual, h_out, norm_w):
            if self.comm is not None:
                self.comm(partial, residual, h_out, norm_w, self.xn, None, None, B, cfg.dim, cfg.norm_eps)
            else:
                torch.distributed.all_reduce(partial, group=self.pg)
                check(lib.chitu_b200_add(ptr(partial), ptr(residual), ptr(h_out), B * cfg.dim, _lib.CB_BF16, st), "add")
                self._rmsnorm(h_out, norm_w, self.xn, B)

        self._rmsnorm(h, self.layers[0]["attn_norm"], self.xn, B)
        for li, lw in enumerate(self.layers):
            next_norm = self.layers[li + 1]["attn_norm"] if li + 1 < n_layers else self.norm
            self._linear(self.xn, lw["wqkv"], self.qkv, B)
            q = self.qkv[:, : self.Hq * D]
            k = self.qkv[:, self.Hq * D: (self.Hq + self.Hkv) * D]
            v_view = self.qkv[:, (self.Hq + self.Hkv) * D:]
            # apply_rotary_pos_emb(..., "hf-llama") on the q / k views of the merged qkv output
            check(lib.chitu_b200_rotary_half_strided(ptr(q), qkv_w, ptr(self.q_rot), ptr(self.cos), ptr(self.sin), B, self.Hq, D,
                                                     _lib.CB_BF16, st), "rotary_half q")
            check(lib.chitu_b200_rotary_half_strided(ptr(k), qkv_w, ptr(self.k_rot), ptr(self.cos), ptr(self.sin), B, self.Hkv, D,
                                                     _lib.CB_BF16, st), "rotary_half k")
            check(lib.chitu_b200_gqa_paged_decode(
                ptr(self.q_rot), ptr(self.k_cache[li]), ptr(self.v_cache[li]), ptr(self.k_rot), ptr(v_view),
                self.Hkv * D, qkv_w, ptr(self.seq_lens), ptr(self.block_table), self.max_blocks, B, self.Hq, self.Hkv, D,
                self.page, self.max_seq_len, 1.0 / math.sqrt(D), ptr(self.attn_out), ptr(self.attn_ws),
                self.attn_ws.numel(), _lib.CB_BF16, st), "gqa_paged_decode")
            push = tp_on and self.comm is not None and self.ar_push
            if push:
                self.comm.linear_push(self.attn_out, lw["wo"], B, self.lin_ws)
                self.comm.consume(h, h2, lw["ffn_norm"], self.xn, None, None, B, cfg.dim, cfg.norm_eps)
            elif tp_on:
                self._linear(self.attn_out, lw["wo"], h2, B)
                reduce_add_norm(h2, h, h2, lw["ffn_norm"])
            else:
                self._linear(self.attn_out, lw["wo"], h2, B, residual=h)
                self._rmsnorm(h2, lw["ffn_norm"], self.xn, B)
            # ---- sparse MoE block (model_hf_mixtral.py:51-96) through the fused experts ----
            check(lib.chitu_b200_moe_gate(ptr(self.xn), ptr(lw["gate_w"]), None, 0, B, cfg.dim, self.E, 1, 1, self.topk, 2,
                                          1.0, ptr(self.gate_w_all[li]), ptr(self.gate_i_all[li]), self.topk,
                                          ptr(self.gate_ws), self.gate_ws.numel(), st), "moe_gate")
            if push:
                self.comm.experts_push(self.xn, lw["w1"], lw["w2"], None, None, self.gate_w_all[li], _lib.CB_BF16,
                                       self.gate_i_all[li], _lib.CB_I64, B, self.topk, self.E, 2 * self.F, cfg.dim, 0, self.moe_ws)
                self.comm.consume(h2, h, next_norm, self.xn, None, None, B, cfg.dim, cfg.norm_eps)
                continue
            check(lib.chitu_b200_fused_experts(
                ptr(self.xn), ptr(lw["w1"]), ptr(lw["w2"]), None, None, ptr(self.gate_w_all[li]), _lib.CB_BF16,
                ptr(self.gate_i_all[li]), _lib.CB_I64, B, self.topk, self.E, 2 * self.F, cfg.dim, 0,
                ptr(self.y if tp_on else h), None if tp_on else ptr(h2), ptr(self.moe_ws), self.moe_ws.numel(), st),
                "fused_experts")
            if tp_on:
                reduce_add_norm(self.y, h2, h, next_norm)
            else:
                self._rmsnorm(h, next_norm, self.xn, B)
        self._linear(self.xn, self.head, self.logits, B)
        vocab_local = cfg.vocab_size // self.tp_size
        check(lib.chitu_b200_argmax(ptr(self.logits), ptr(self.next_tokens), B, vocab_local, _lib.CB_BF16, st), "argmax")
        if tp_on:
            self.next_tokens.copy_(global_argmax(self.logits, self.next_tokens, self.tp_rank, vocab_local, self.pg, self.tp_gather))
        self.seq_lens.add_(1)

    def capture(self):
        torch.cuda.synchronize(self.device)
        saved = self.seq_lens.clone()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(2):
                self._step_body()
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        self.seq_lens.copy_(saved)
        before = _lib.launch_count()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._step_body()
        self.launches_per_step = _lib.launch_count() - before
        self.seq_lens.copy_(saved)
        torch.cuda.synchronize(self.device)

    def step(self):
        if self.graph is not None:
            self.graph.replay()
        else:
            before = _lib.launch_count()
            self._step_body()
            self.launches_per_step = _lib.launch_count() - before

    def decode(self, tokens_host: torch.Tensor) -> torch.Tensor:
        self.tokens.copy_(tokens_host, non_blocking=True)
        self.step()
        return self.next_tokens.cpu()

    def distinct_experts_per_layer(self) -> float:
        ids = self.gate_i_all.cpu()
        return float(sum(len(torch.unique(ids[l])) for l in range(ids.shape[0])) / ids.shape[0])

    def algorithmic_bytes(self, seq_len: int, distinct: float) -> int:
        """SURVEY §8d: every attention weight byte once, each DISTINCT expert once, KV rows once, bf16 head + router."""
        c, D = self.cfg, self.D
        attn = ((self.Hq + 2 * self.Hkv) * D * c.dim + c.dim * self.Hq * D) * 2
        expert = 3 * self.F * c.dim * 2
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
