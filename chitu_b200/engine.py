"""Decode-step engine: the caller side of the hot path, wired exactly like the reference's
`Transformer.decode_single_device` (chitu/models/model.py:467-474) + `TransformerBlockLlama`
(models/model_llama.py:152-185) + `Attention.decode_forward_paged` (models/model.py:167-198),
but every operator is a libchitu_b200 kernel and the whole step is one CUDA graph
(reference: per-batch-size graph capture, models/model.py:537-622).

It exists so `bench.py` can measure BASELINE.json's metric (decode tokens/s) on synthetic
weights of the named architecture; it is not a re-implementation of the reference's model zoo
(checkpoint loading, prefill, PP stay in the reference).

`DecodeEngine` is the part every model shares; the LLaMA, DeepSeek (engine_deepseek.py) and
Mixtral (engine_mixtral.py) engines add their weights and their layers.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from ._lib import check, current_stream, ptr
from .attn_backend import gqa_paged_attention
from .quantize import fp8, w4a16
from .tensor_parallel import global_argmax

BF = torch.bfloat16

# quantised weight format -> (the quantiser of one float weight [N, K] into the tensors the format's GEMMs read, the
# dequantiser of those tensors into the values the GEMMs multiply: bf16 for 4-bit weights, fp32 q * s for fp8 ones)
QUANT_FORMATS = {
    "w4a16": (lambda w: w4a16.quantize_rtn(w, BF), w4a16.dequantize),
    "fp8": (fp8.quantize_weight, fp8.dequantize),
}


@dataclass
class LlamaConfig:
    """chitu/config/models/Meta-Llama-3-8B-Instruct-original.yaml:6-14."""
    dim: int = 4096
    n_layers: int = 32
    n_heads: int = 32
    n_kv_heads: int = 8
    vocab_size: int = 128256
    multiple_of: int = 1024
    ffn_dim_multiplier: Optional[float] = 1.3
    norm_eps: float = 1e-5
    rope_theta: float = 500000.0

    @property
    def head_dim(self):
        return self.dim // self.n_heads

    @property
    def ffn_dim(self):
        # FeedForwardLlama.__init__ (models/model_llama.py:131-137)
        hidden = int(2 * (4 * self.dim) / 3)
        if self.ffn_dim_multiplier is not None:
            hidden = int(self.ffn_dim_multiplier * hidden)
        return self.multiple_of * ((hidden + self.multiple_of - 1) // self.multiple_of)


LLAMA3_8B = LlamaConfig()
LLAMA2_7B = LlamaConfig(dim=4096, n_layers=32, n_heads=32, n_kv_heads=32, vocab_size=32000, multiple_of=256,
                        ffn_dim_multiplier=None, norm_eps=1e-5, rope_theta=10000.0)


class DecodeEngine:
    """Greedy decode over persistent buffers, eager or replayed as one CUDA graph: embedding + rotary-position gather,
    the model's layers, then the vocab-parallel head and argmax.

    A subclass builds its weights, its KV caches (listed in `self.caches`) and its rotary tables (`_rope_tables`),
    and runs its layers in `_decode_layers`: from the embedded tokens in `self.h` to the final norm in `self.xn`.
    `_norm` is the RMSNorm the row-parallel reduce ends with (bf16 here).

    Tensor parallel when a process group is given and tp_size > 1 (`tp_on`).  With tp_size > 1 and no group the engine
    runs ONE rank's shard without collectives ("shard mode": the per-rank kernel time of a tensor-parallel
    configuration measured on one GPU)."""

    linear_impl = 0          # `impl` of the bf16 linear entries: 0 = auto
    # "w4a16": the subclass's QUANT_LINEARS hold (qweight, scales, zeros) in quantize/w4a16.py's layout (stacked per
    # expert for the MoE weights) and run on the 4-bit GEMMs; "fp8": they hold (weight e4m3, weight_scale fp32 [N]) in
    # quantize/fp8.py's layout and run on the rowwise FP8 GEMMs.  WEIGHT_FORMATS: the formats the subclass accepts
    weight_format = "bf16"
    WEIGHT_FORMATS = ("bf16",)
    QUANT_LINEARS = ()

    def __init__(self, cfg, max_reqs: int, max_seq_len: int, device, page_size: int, seed: int, tp_rank: int,
                 tp_size: int, process_group, use_fused_allreduce: bool, attn_ws: tuple, lin_n: int, max_draft: int = 0):
        """attn_ws: (heads, head_dim_v, max_splits) the attention workspace is sized for; lin_n: the widest N the
        linear workspace is sized for; max_draft: the draft tokens per request a verify step checks (0: none), which
        sizes the row buffers for max_reqs * (max_draft + 1) rows."""
        self.cfg, self.B, self.device = cfg, max_reqs, torch.device(device)
        self.max_draft = max_draft
        rows = max_reqs * (max_draft + 1)         # rows of the widest step: the decode step's B, or a verify step's
        self.tp_rank, self.tp_size, self.pg = tp_rank, tp_size, process_group
        self.tp_on = process_group is not None and tp_size > 1
        self.lib = _lib.load()
        dev, B, dim = self.device, max_reqs, cfg.dim
        self.g = torch.Generator(device=dev).manual_seed(seed + 1000 * tp_rank)       # this rank's shards
        self.g_rep = torch.Generator(device=dev).manual_seed(seed + 7)                # replicated across TP ranks
        # paged KV cache (PagedKVCacheManager, cache_manager.py:71-87): persistent int32 block_table and seq_lens
        self.page, self.max_seq_len = page_size, max_seq_len
        self.max_blocks = max_seq_len // page_size + 1
        self.block_table = torch.zeros(max_reqs, self.max_blocks, dtype=torch.int32, device=dev)
        self.seq_lens = torch.zeros(max_reqs, dtype=torch.int32, device=dev)
        # persistent step I/O and residual stream (CUDA-graph safe)
        self.tokens = torch.zeros(B, dtype=torch.int64, device=dev)
        self.h, self.h2, self.xn = (torch.zeros(rows, dim, dtype=BF, device=dev) for _ in range(3))
        self.logits = torch.zeros(rows, cfg.vocab_size // tp_size, dtype=BF, device=dev)
        self.next_tokens = torch.zeros(B, dtype=torch.int64, device=dev)
        self.tp_gather = torch.empty(tp_size, B, 2, dtype=torch.float32, device=dev) if self.tp_on else None
        heads, head_dim_v, max_splits = attn_ws
        self.attn_ws = torch.zeros(self.lib.chitu_b200_attn_workspace_bytes(B, heads, head_dim_v, max_splits),
                                   dtype=torch.uint8, device=dev)
        self.lin_ws = torch.zeros(max(self.lib.chitu_b200_linear_workspace_bytes(rows, lin_n), 256), dtype=torch.uint8,
                                  device=dev)                    # split-K tickets start at 0
        # push mode: the row-parallel product's epilogue starts the all-reduce (every product the base and the
        # DeepSeek / Mixtral engines reduce has a push epilogue; the pull kernel reduces products without one)
        self.ar_push = True
        # fused one-shot all-reduce + residual + RMSNorm(+quant) over NVLink peer memory (csrc/comm.cu); NCCL otherwise
        self.comm = None
        if self.tp_on and use_fused_allreduce:
            from .comm import FusedAllReduce
            self.comm = FusedAllReduce(process_group, rows, dim, dev)
        self.graph = None
        self.launches_per_step = 0
        # set to [] to record the residual stream entering every layer, and the last layer's output (tests; eager steps
        # only, never under a graph)
        self.capture_h = None

    def _set_weight_format(self, weight_format: str, tp_size: int, process_group):
        if weight_format not in self.WEIGHT_FORMATS:
            raise ValueError(f"weight_format must be one of {self.WEIGHT_FORMATS}, not {weight_format!r}")
        if weight_format != "bf16" and process_group is not None and tp_size > 1:
            raise ValueError(f"weight_format={weight_format!r} runs on one GPU or one shard: its GEMM has no push "
                             "epilogue for the tensor-parallel all-reduce")
        self.weight_format = weight_format

    def _quantized(self, lw: dict) -> dict:
        """The layer's weights `lw`, with its QUANT_LINEARS quantised in place into the engine's weight format; a stack
        of expert weights [E, N, K] is quantised one expert at a time and restacked."""
        if self.weight_format != "bf16":
            quantize, _ = QUANT_FORMATS[self.weight_format]
            for name in self.QUANT_LINEARS:
                w = lw[name]
                lw[name] = quantize(w) if w.dim() == 2 else tuple(torch.stack(t) for t in zip(*map(quantize, w)))
        return lw

    def _dequantized(self, lw: dict) -> dict:
        """A copy of the layer's weights with the quantised ones as the values the kernels multiply (the oracle side of
        the tests)."""
        d = dict(lw)
        if self.weight_format != "bf16":
            _, dequantize = QUANT_FORMATS[self.weight_format]
            d.update({name: dequantize(*lw[name]) for name in self.QUANT_LINEARS})
        return d

    def _rnd(self, gen, *shape, scale=0.02, dtype=BF):
        """A synthetic weight: normal(0, scale) drawn in fp32 from `gen`, then cast to `dtype`."""
        return (torch.randn(*shape, generator=gen, dtype=torch.float32, device=self.device) * scale).to(dtype)

    def _rope_tables(self, ang: torch.Tensor, dtype=torch.float32):
        """cos / sin tables from the rotary angles [positions, rot_dim / 2], and the per-step buffers that
        `_step_body` gathers them into by position."""
        self.cos_table, self.sin_table = ang.cos().to(dtype).to(self.device), ang.sin().to(dtype).to(self.device)
        self.cos = torch.zeros(self.B, ang.shape[1], dtype=dtype, device=self.device)
        self.sin = torch.zeros_like(self.cos)

    # ---- cache bookkeeping (host side of PagedKVCacheManager, cache_manager.py:148-209) ----------
    def set_synthetic_context(self, seq_len: int, seed: int = 2):
        """Fill the KV cache with `seq_len` random cached tokens per request and a shuffled
        (non-identity) block table (SURVEY §8d synthetic inputs)."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        gd = torch.Generator(device=self.device).manual_seed(seed + 11)     # deterministic cache contents
        perm = torch.randperm(self.block_table.numel(), generator=g).to(torch.int32)
        self.block_table.copy_(perm.view(self.B, self.max_blocks))
        self.seq_lens.fill_(seq_len)
        for l in range(self.cfg.n_layers):
            for cache in self.caches:
                if cache.dtype == torch.float8_e4m3fn:        # normal_ is not defined for fp8: draw, clamp, cast
                    x = torch.empty(cache[l].shape, dtype=torch.float32, device=self.device).normal_(0, 1, generator=gd)
                    cache[l].copy_(x.clamp_(-448.0, 448.0))
                else:
                    cache[l].normal_(0, 1, generator=gd)

    # ---- one decode step ---------------------------------------------------------------------------
    def _linear(self, x, w, y, M, residual=None):
        N, K = w.shape
        check(self.lib.chitu_b200_linear_bf16(ptr(x), ptr(w), None, ptr(residual), ptr(y), M, N, K, _lib.CB_BF16,
                                              ptr(self.lin_ws), self.lin_ws.numel(), self.linear_impl,
                                              current_stream()), "linear_bf16")

    def _layer_linear(self, x, lw, name, y, M, residual=None, silu_pairs=False):
        """y = x . lw[name]^T (+ residual) in the engine's weight format; silu_pairs: y = SiluAndMul of that product,
        whose rows hold interleaved gate / up pairs (no residual).  fp8: x is the e4m3 self.xq with the per-token scales
        in self.xs."""
        fmt, lib, w = self.weight_format, self.lib, lw[name]
        if fmt == "bf16" and not silu_pairs:
            return self._linear(x, w, y, M, residual=residual)
        ws = (ptr(self.lin_ws), self.lin_ws.numel(), current_stream())
        if fmt == "bf16":
            N, K = w.shape
            rc = lib.chitu_b200_linear_bf16_silu_pairs(ptr(x), ptr(w), ptr(y), M, N, K, *ws)
        elif fmt == "fp8":
            q, s = w
            N, K = q.shape
            operands = (ptr(x), ptr(self.xs), ptr(q), ptr(s))
            rc = (lib.chitu_b200_fp8_rowwise_gemm_silu_pairs(*operands, ptr(y), M, N, K, *ws) if silu_pairs else
                  lib.chitu_b200_fp8_rowwise_gemm(*operands, None, ptr(residual), ptr(y), M, N, K, *ws))
        else:
            q, s, z = w
            N, K = q.shape[0], 2 * q.shape[1]
            operands = (ptr(x), ptr(q), ptr(s), ptr(z))
            rc = (lib.chitu_b200_w4a16_gemm_silu_pairs(*operands, ptr(y), M, N, K, _lib.CB_BF16, *ws) if silu_pairs else
                  lib.chitu_b200_w4a16_gemm(*operands, ptr(residual), ptr(y), M, N, K, _lib.CB_BF16, *ws))
        check(rc, f"{fmt} {name}" + (" + silu" if silu_pairs else ""))

    def _norm(self, x, w, y, q=None, qs=None, rows=None):
        """RMSNorm of `rows` rows (default B) into bf16 `y`; with `q`, into the e4m3 `q` and per-token scales `qs` as
        well (y may then be None)."""
        M = self.B if rows is None else rows
        if q is not None:
            check(self.lib.chitu_b200_rmsnorm_quant_fp8_rowwise(ptr(x), ptr(w), ptr(y), ptr(q), ptr(qs), M,
                                                                self.cfg.dim, self.cfg.norm_eps, current_stream()),
                  "rmsnorm_quant_fp8_rowwise")
            return
        check(self.lib.chitu_b200_rmsnorm(ptr(x), ptr(w), ptr(y), M, self.cfg.dim, self.cfg.norm_eps, _lib.CB_BF16,
                                          current_stream()), "rmsnorm")

    def _allreduce(self, t):
        if self.tp_on:
            torch.distributed.all_reduce(t, group=self.pg)

    def _row_parallel(self, gemm, push, residual, h_out, norm_w, y=None, q=None, qs=None, partial=None, rows=None):
        """h_out = residual + the sum over ranks of a row-parallel product, then RMSNorm(h_out) * norm_w into the
        wanted outputs (bf16 `y`, fp8 `q` + scales `qs`), over `rows` rows (default B).

        `gemm(out, residual)` writes this rank's product into `out`, adding `residual` when it is given; `push()` is the
        same product with the epilogue that starts the fused all-reduce.  Single GPU (and shard mode) fuses the residual
        into the GEMM; tensor parallel reduces by push + consume, by the fused pull kernel, or by NCCL + add + norm,
        with this rank's product in `partial` (default: `h_out`)."""
        B, dim, eps = self.B if rows is None else rows, self.cfg.dim, self.cfg.norm_eps
        if not self.tp_on:
            gemm(h_out, residual)
            self._norm(h_out, norm_w, y, q, qs, rows=B)
        elif self.comm is not None and self.ar_push:
            push()
            self.comm.consume(residual, h_out, norm_w, y, q, qs, B, dim, eps)
        else:
            partial = h_out if partial is None else partial
            gemm(partial, None)
            if self.comm is not None:
                self.comm(partial, residual, h_out, norm_w, y, q, qs, B, dim, eps)
            else:
                self._allreduce(partial)
                check(self.lib.chitu_b200_add(ptr(partial), ptr(residual), ptr(h_out), B * dim, _lib.CB_BF16,
                                              current_stream()), "add")
                self._norm(h_out, norm_w, y, q, qs, rows=B)

    # ---- GQA attention over the paged K / V caches (LLaMA, Mixtral) ----------------------------------
    def _gqa_buffers(self, kv_dtype, rows: int):
        """The paged K / V caches [L, blocks, page, Hkv, D] in kv_dtype, and the attention's buffers for `rows` rows: the
        merged qkv projection, the rotated q / k and the attention output."""
        dev, D, Hq, Hkv = self.device, self.D, self.Hq, self.Hkv
        self.k_cache = torch.zeros(self.cfg.n_layers, self.max_blocks * self.B, self.page, Hkv, D, dtype=kv_dtype,
                                   device=dev)
        self.v_cache = torch.zeros_like(self.k_cache)
        self.caches = (self.k_cache, self.v_cache)
        self.qkv = torch.zeros(rows, (Hq + 2 * Hkv) * D, dtype=BF, device=dev)
        self.q_rot = torch.zeros(rows, Hq, D, dtype=BF, device=dev)
        self.k_rot = torch.zeros(rows, Hkv, D, dtype=BF, device=dev)
        self.attn_out = torch.zeros(rows, Hq * D, dtype=BF, device=dev)

    def _gqa_attention(self, li, q, k, sq=1, rope=None):
        """Paged GQA attention of layer li into attn_out: sq query rows per request (row b * sq + i is token i of
        request b), q and the new k rows as given (any row stride), v in the qkv output.  The new k / v rows are
        appended at seq_lens[b] + i and query i attends causally.  rope: the (cos, sin) rows that rotate q and k inside
        the kernel (sq == 1); without it they are rotated already."""
        D = self.D
        v = self.qkv[:, (self.Hq + self.Hkv) * D:]
        kv_strides = (sq * k.stride(0), k.stride(0) if sq > 1 else 0, sq * v.stride(0), v.stride(0) if sq > 1 else 0)
        ws = self.attn_ws if sq == 1 else self.verify_attn_ws
        gqa_paged_attention(q, sq * q.stride(0), self.k_cache[li], self.v_cache[li], k, v, kv_strides, rope,
                            self.seq_lens, self.block_table, self.B, sq, self.Hq, self.max_seq_len, True,
                            1.0 / math.sqrt(D), self.attn_out, ws)

    # ---- the MoE block (Mixtral, DeepSeek) ------------------------------------------------------------
    def _init_moe(self, n_routed: int, topk: int, slots: int, n_stacked: int, n1: int, score_mode: int,
                  route_scale: float = 1.0, groups=(1, 1), bias: bool = False, first_layer: int = 0,
                  weights=("w1", "w2", None, None), wmode: int = 0):
        """The engine's routing, stated once.  The gate (chitu_b200_moe_gate, `score_mode`) scores `n_routed` experts,
        within the best `groups[1]` of `groups[0]` groups, with the layer's fp32 bias `gate_b` when `bias`, and picks
        `topk` of them into `slots` slots per token (the engine fills the slots past topk).  Layers from `first_layer` on
        are MoE layers; each holds its `n_stacked` experts stacked, as the layer entries `weights` (w1 [n_stacked, n1,
        dim], w2, and their scales for wmode 1) in chitu_b200_fused_experts' `wmode`, or as (qweight, scales, zeros)
        under weight_format "w4a16".  Allocates every layer's routing results (resident: bench.py counts the distinct
        experts per layer), the workspaces and `y`, this rank's expert sum under tensor parallelism."""
        B, dev, dim = self.B, self.device, self.cfg.dim
        self.gate_w_all = torch.zeros(self.cfg.n_layers, B, slots, dtype=BF, device=dev)
        self.gate_i_all = torch.zeros(self.cfg.n_layers, B, slots, dtype=torch.int64, device=dev)
        self.moe_ws = torch.zeros(self.lib.chitu_b200_moe_workspace_bytes(B, slots, n_stacked, n1, dim), dtype=torch.uint8,
                                  device=dev)
        self.gate_ws = torch.zeros(self.lib.chitu_b200_moe_gate_workspace_bytes(B, n_routed), dtype=torch.uint8,
                                   device=dev)
        self.y = torch.zeros(B, dim, dtype=BF, device=dev)
        self._gate = (n_routed, *groups, topk, score_mode, float(route_scale))       # chitu_b200_moe_gate's E .. scale
        self._moe = dict(topk=topk, bias=bias, first_layer=first_layer, weights=weights, wmode=wmode,
                         stack=(slots, n_stacked, n1))

    def _moe_gate(self, li):
        """Route every token of layer li on self.xn into gate_w_all[li] / gate_i_all[li]."""
        lw = self.layers[li]
        bias = lw["gate_b"] if self._moe["bias"] else None
        check(self.lib.chitu_b200_moe_gate(ptr(self.xn), ptr(lw["gate_w"]), ptr(bias), 0 if bias is None else _lib.CB_F32,
                                           self.B, self.cfg.dim, *self._gate, ptr(self.gate_w_all[li]),
                                           ptr(self.gate_i_all[li]), self.gate_w_all.shape[2], ptr(self.gate_ws),
                                           self.gate_ws.numel(), current_stream()), "moe_gate")

    def _moe_block(self, li, residual, h_out, norm_w, **norm_out):
        """Layer li's MoE block on self.xn: the gate, then h_out = residual + the experts' sum over ranks, and its
        RMSNorm by norm_w into `norm_out` (`_row_parallel`)."""
        self._moe_gate(li)
        lw, (slots, n_stacked, n1) = self.layers[li], self._moe["stack"]
        w1, w2, s1, s2 = (lw[n] if n else None for n in self._moe["weights"])
        # the arguments up to the output, as tensors: the local call passes their pointers, the push epilogue takes them
        route = (self.gate_w_all[li], _lib.CB_BF16, self.gate_i_all[li], _lib.CB_I64, self.B, slots, n_stacked, n1,
                 self.cfg.dim)
        if self.weight_format == "w4a16":
            fn, name, args = self.lib.chitu_b200_fused_experts_w4a16, "fused_experts_w4a16", (self.xn, *w1, *w2, *route)
        else:
            fn, name, args = (self.lib.chitu_b200_fused_experts, "fused_experts",
                              (self.xn, w1, w2, s1, s2, *route, self._moe["wmode"]))

        def local(out, res):
            check(fn(*(ptr(a) if isinstance(a, torch.Tensor) else a for a in args), ptr(out), ptr(res), ptr(self.moe_ws),
                     self.moe_ws.numel(), current_stream()), name)

        self._row_parallel(local, lambda: self.comm.experts_push(*args, self.moe_ws), residual, h_out, norm_w,
                           partial=self.y, **norm_out)

    def distinct_experts_per_layer(self) -> float:
        """Mean number of distinct routed experts per MoE layer in the last step."""
        ids = self.gate_i_all[self._moe["first_layer"]:, :, :self._moe["topk"]].cpu()
        if ids.numel() == 0:
            return 0.0
        return float(sum(len(torch.unique(ids[l])) for l in range(ids.shape[0])) / ids.shape[0])

    def _step_body(self):
        lib, B, cfg = self.lib, self.B, self.cfg
        st = current_stream()
        # prepare_freqs_cis_decode (models/model.py:429-448): gather cos/sin by position
        torch.index_select(self.cos_table, 0, self.seq_lens, out=self.cos)
        torch.index_select(self.sin_table, 0, self.seq_lens, out=self.sin)
        # (embedding table replicated per rank here; the reference shards it by vocab + all_reduce)
        check(lib.chitu_b200_embedding(ptr(self.tokens), ptr(self.embed), ptr(self.h), B, cfg.dim, 0, cfg.vocab_size,
                                       _lib.CB_BF16, st), "embedding")
        self._decode_layers()
        self._linear(self.xn, self.head, self.logits, B)          # self.xn = norm(h) already
        vocab_local = self.head.shape[0]
        check(lib.chitu_b200_argmax(ptr(self.logits), ptr(self.next_tokens), B, vocab_local, _lib.CB_BF16, st),
              "argmax")
        if self.tp_on:
            # vocab-parallel head: the reference all-gathers the logits shards before sampling
            # (tensor_parallel.py:94-102); the same token from a (max, index) all-gather of B*8 bytes per rank
            self.next_tokens.copy_(global_argmax(self.logits[:B], self.next_tokens, self.tp_rank, vocab_local, self.pg,
                                                 self.tp_gather))
        self.seq_lens.add_(1)     # finalize_cache_single_decode (cache_manager.py)

    def _capture(self, body, generators=()):
        """(a CUDA graph of `body`, the launches it holds); seq_lens is restored after the warm-up and the capture.
        `generators`: the torch generators `body` draws from, registered with the graph so each replay draws anew."""
        torch.cuda.synchronize(self.device)
        saved = self.seq_lens.clone()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(2):
                body()                    # warm-up outside capture
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        self.seq_lens.copy_(saved)
        before = _lib.launch_count()
        graph = torch.cuda.CUDAGraph()
        for gen in generators:
            graph.register_generator_state(gen)
        with torch.cuda.graph(graph):
            body()
        launches = _lib.launch_count() - before
        self.seq_lens.copy_(saved)
        torch.cuda.synchronize(self.device)
        return graph, launches

    def capture(self):
        """Capture the decode step in a CUDA graph (models/model.py:572-611)."""
        self.graph, self.launches_per_step = self._capture(self._step_body)

    @staticmethod
    def _run(graph, body, launches):
        """Replay `graph`, or run `body` eagerly when it has not been captured; returns the launches of one step
        (`launches`, what the capture counted, on a replay)."""
        if graph is not None:
            graph.replay()
            return launches
        before = _lib.launch_count()
        body()
        return _lib.launch_count() - before

    def step(self):
        """One decode step over the persistent buffers (tokens in self.tokens)."""
        self.launches_per_step = self._run(self.graph, self._step_body, self.launches_per_step)

    def decode(self, tokens_host: torch.Tensor) -> torch.Tensor:
        """Public API: host tokens [B] int64 (pinned) -> host next tokens [B] (greedy).
        Includes the H2D copy of the inputs and the D2H read of the result."""
        self.tokens.copy_(tokens_host, non_blocking=True)
        self.step()
        return self.next_tokens.cpu()


class LlamaDecodeEngine(DecodeEngine):
    """Single-GPU (tp=1) or tensor-parallel LLaMA decode.  Weights are random (`do_load=False`,
    serve_config.yaml:9).  KV cache layout = PagedKVCacheManager (cache_manager.py:71-87):
    paged_k_cache / paged_v_cache [L, num_blocks, page, n_local_kv_heads, head_dim], page 256
    (backend.py:237).  kv_dtype=torch.float8_e4m3fn keeps the caches in e4m3 (half the KV bytes; new rows rounded
    to nearest even after a clamp to +-448, no scale) and decodes through chitu_b200_gqa_paged_attn_fp8kv.

    weight_format="w4a16" holds qkv, o, w13 and w2 as 4-bit groups of 128 (quantize/w4a16.py's round-to-nearest rule
    applied to the same synthetic weights) and runs them through chitu_b200_w4a16_gemm[_silu_pairs]; embedding, head,
    norms, rotary and attention stay bf16.  The W4 GEMM has no push epilogue, so it runs on one GPU or in shard mode.

    weight_format="fp8" holds the same four linears as e4m3 with per-channel scales (quantize/fp8.py's rule applied to
    the same synthetic weights) and runs them through chitu_b200_fp8_rowwise_gemm[_silu_pairs] on per-token e4m3
    activations: the RMSNorms before qkv and w13 emit them (chitu_b200_rmsnorm_quant_fp8_rowwise), and the attention
    output and the SiLU product are quantised by chitu_b200_quant_fp8_rowwise before wo and w2.  Embedding, head,
    rotary, attention and the KV cache stay as in bf16; one GPU or shard mode, as for W4.

    max_draft=k > 0 adds a speculative verify step (`verify`, `capture_verify`): every request's token and up to k draft
    tokens run through the model as B * (k + 1) rows with causal attention over the cache, and the greedy acceptance
    kernel advances `seq_lens` on the device.  The row buffers are then sized for B * (k + 1) rows; the decode step is
    unchanged.

    sampled_verify=True verifies under each request's temperature / top_k / top_p instead (speculative sampling,
    chitu_b200_spec_accept_sampled): the emitted tokens have the distribution of sampling the model one token at a
    time, and T = 0 requests are accepted greedily as before.  Its uniforms are drawn on the device inside the verify
    step from an engine-owned generator (`sample_generator`, seeded from `seed`).  draft_probs=True also takes the
    drafter's distributions [B, k', V] (a draft model's); without it the drafts are token-only (q one-hot).  One GPU
    only: the vocab-parallel head leaves each rank a vocabulary shard."""

    WEIGHT_FORMATS = ("bf16", "w4a16", "fp8")
    QUANT_LINEARS = ("wqkv", "wo", "w13", "w2")

    def __init__(self, cfg: LlamaConfig, max_reqs: int, max_seq_len: int, device="cuda:0", page_size: int = 256,
                 seed: int = 0, tp_rank: int = 0, tp_size: int = 1, process_group=None, linear_impl: int = 0,
                 use_fused_allreduce: bool = True, kv_dtype: torch.dtype = BF, weight_format: str = "bf16",
                 max_draft: int = 0, sampled_verify: bool = False, draft_probs: bool = False):
        D = cfg.head_dim
        self._set_weight_format(weight_format, tp_size, process_group)
        if weight_format != "bf16" and linear_impl == 1:
            raise ValueError(f"weight_format={weight_format!r} runs on the wgmma GEMM only (linear_impl=1 selects the "
                             "SIMT GEMV)")
        assert cfg.n_heads % tp_size == 0 and cfg.n_kv_heads % tp_size == 0
        self.Hq, self.Hkv, self.D = cfg.n_heads // tp_size, cfg.n_kv_heads // tp_size, D
        self.F = cfg.ffn_dim // tp_size
        self.linear_impl = linear_impl
        if max_draft < 0:
            raise ValueError(f"max_draft must be >= 0, not {max_draft}")
        if max_draft > 0:
            # what the multi-token attention kernels are built for, and the rows one GEMM token tile set and the
            # all-reduce kernels take
            if linear_impl == 1:
                raise ValueError("the verify step runs on the wgmma GEMMs (linear_impl=1 selects the SIMT GEMV)")
            if D != 128 or page_size % 64 != 0 or self.Hq // self.Hkv not in (1, 2, 4, 8):
                raise ValueError("the verify step needs head dim 128, Hq / Hkv in {1, 2, 4, 8} and a page that is a "
                                 f"multiple of 64 (head dim {D}, page {page_size})")
            if max_reqs * (max_draft + 1) > 256:
                raise ValueError(f"the verify step runs at most 256 rows: max_reqs * (max_draft + 1) = "
                                 f"{max_reqs * (max_draft + 1)}")
        if sampled_verify and max_draft == 0:
            raise ValueError("sampled_verify needs a verify step: build the engine with max_draft > 0")
        if draft_probs and not sampled_verify:
            raise ValueError("draft_probs are read by the sampled verify step only: build with sampled_verify=True")
        if sampled_verify and tp_size > 1:
            raise ValueError("sampled_verify runs on one GPU: under tensor parallelism each rank's head holds a "
                             "vocabulary shard")
        self.sampled_verify = sampled_verify
        super().__init__(cfg, max_reqs, max_seq_len, device, page_size, seed, tp_rank, tp_size, process_group,
                         use_fused_allreduce, attn_ws=(self.Hq, D, 64),
                         lin_n=max(2 * self.F, cfg.vocab_size // tp_size), max_draft=max_draft)
        dev, g, dim, rnd = self.device, self.g, cfg.dim, self._rnd
        # SiluAndMul inside the w13 GEMM epilogue: the merged gate/up weight is stored with its rows interleaved
        # (row 2i = gate_i, row 2i+1 = up_i) — a load-time permutation of the reference's merged tensor.
        # It and push mode need the wgmma GEMM, which linear_impl=1 (the SIMT GEMV) turns off.
        self.fuse_silu = linear_impl != 1
        self.ar_push = linear_impl != 1
        self.embed = rnd(self.g_rep, cfg.vocab_size, dim)
        self.layers = []
        for _ in range(cfg.n_layers):
            lw = dict(
                attn_norm=torch.ones(dim, dtype=BF, device=dev),
                ffn_norm=torch.ones(dim, dtype=BF, device=dev),
                # column-parallel wq|wk|wv merged along N (shards of each concatenated); row-parallel wo
                wqkv=rnd(g, (self.Hq + 2 * self.Hkv) * D, dim),
                wo=rnd(g, dim, self.Hq * D),
                w13=rnd(g, 2 * self.F, dim),          # [w1 (gate) ; w3 (up)]
                w2=rnd(g, dim, self.F),
            )
            if self.fuse_silu:
                lw["w13"] = lw["w13"].view(2, self.F, dim).transpose(0, 1).reshape(2 * self.F, dim).contiguous()
            # quantised per row after the interleave: w13's interleaved rows carry their own scales (and zeros)
            self.layers.append(self._quantized(lw))
        self.norm = torch.ones(dim, dtype=BF, device=dev)
        self.head = rnd(g, cfg.vocab_size // tp_size, dim)
        if kv_dtype not in (BF, torch.float8_e4m3fn):
            raise ValueError(f"kv_dtype must be torch.bfloat16 or torch.float8_e4m3fn, not {kv_dtype}")
        self.kv_fp8 = kv_dtype == torch.float8_e4m3fn
        B = max_reqs * (max_draft + 1)                     # rows of the widest step
        self._gqa_buffers(kv_dtype, B)
        # precompute_freqs_cis (models/model.py:81-89) as cos/sin tables
        freqs = 1.0 / (cfg.rope_theta ** (torch.arange(0, D, 2)[: D // 2].float() / D))
        self._rope_tables(torch.outer(torch.arange(max_seq_len * 2, dtype=torch.float32), freqs))
        self.gate_up = torch.zeros(B, 2 * self.F, dtype=BF, device=dev)
        self.act = torch.zeros(B, self.F, dtype=BF, device=dev)
        self.verify_graph = None
        self.launches_per_verify = 0
        if max_draft > 0:
            # verify step I/O: [tokens | drafts] per request, the positions and rotary rows of its B * (k + 1) rows, the
            # argmax at each row, the acceptance outputs; its attention workspace splits B * (k + 1) query rows
            k, R = max_draft, B
            self.draft_tokens = torch.zeros(max_reqs, k, dtype=torch.int64, device=dev)
            self.n_draft = torch.zeros(max_reqs, dtype=torch.int32, device=dev)
            self.verify_tokens = torch.zeros(max_reqs, k + 1, dtype=torch.int64, device=dev)
            self.verify_offsets = torch.arange(k + 1, dtype=torch.int32, device=dev)
            self.verify_pos = torch.zeros(max_reqs, k + 1, dtype=torch.int32, device=dev)
            self.verify_cos = torch.zeros(R, D // 2, dtype=torch.float32, device=dev)
            self.verify_sin = torch.zeros_like(self.verify_cos)
            self.target = torch.zeros(max_reqs, k + 1, dtype=torch.int64, device=dev)
            self.out_tokens = torch.zeros(max_reqs, k + 1, dtype=torch.int64, device=dev)
            self.accepted = torch.zeros(max_reqs, dtype=torch.int32, device=dev)
            self.verify_gather = torch.empty(tp_size, R, 2, dtype=torch.float32, device=dev) if self.tp_on else None
            self.verify_attn_ws = torch.zeros(self.lib.chitu_b200_attn_workspace_bytes(R, self.Hq, D, 64),
                                              dtype=torch.uint8, device=dev)
        if sampled_verify:
            # each request's sampling parameters; the uniforms of one step: u_accept [B, k] then u_draw [B]
            self.temperatures = torch.zeros(max_reqs, dtype=torch.float32, device=dev)
            self.top_ks = torch.zeros(max_reqs, dtype=torch.int32, device=dev)
            self.top_ps = torch.ones(max_reqs, dtype=torch.float32, device=dev)
            self.uniforms = torch.zeros(max_reqs * (max_draft + 1), dtype=torch.float32, device=dev)
            self.u_accept = self.uniforms[:max_reqs * max_draft].view(max_reqs, max_draft)
            self.u_draw = self.uniforms[max_reqs * max_draft:]
            self.sample_generator = torch.Generator(device=dev).manual_seed(seed + 13)
            self.spec_ws = torch.zeros(self.lib.chitu_b200_spec_accept_sampled_workspace_bytes(max_reqs, max_draft),
                                       dtype=torch.uint8, device=dev)
            self.draft_probs = (torch.zeros(max_reqs, max_draft, cfg.vocab_size, dtype=torch.float32, device=dev)
                                if draft_probs else None)
        if weight_format == "fp8":
            # the e4m3 activations and their per-token scales of whichever linear runs next
            self.xq = torch.zeros(B, max(dim, self.Hq * D, self.F), dtype=torch.float8_e4m3fn, device=dev)
            self.xs = torch.zeros(B, dtype=torch.float32, device=dev)
        # rotary fused into the tensor-core decode kernel (head dim 128, power-of-two pages)
        self.fuse_rope = D == 128 and (page_size & (page_size - 1)) == 0 and self.Hq // self.Hkv in (1, 2, 4, 8)
        if self.kv_fp8 and not (self.fuse_rope and page_size % 64 == 0):
            raise ValueError("the fp8 KV cache needs head dim 128, Hq / Hkv in {1, 2, 4, 8} and a power-of-two page "
                             "that is a multiple of 64")

    def ref_layers(self):
        """The layer weights in the REFERENCE's layout (w13 = [w1 ; w3] halves) for the oracle side of the tests."""
        out = []
        for lw in self.layers:
            d = self._dequantized(lw)
            if self.fuse_silu:
                d["w13"] = d["w13"].view(self.F, 2, self.cfg.dim).transpose(0, 1).reshape(2 * self.F, self.cfg.dim).contiguous()
            out.append(d)
        return out

    def _quant(self, x, rows):
        """The input of the linear that reads the first `rows` rows of x: fp8 quantises them per token into self.xq /
        self.xs."""
        if self.weight_format != "fp8":
            return x
        check(self.lib.chitu_b200_quant_fp8_rowwise(ptr(x), ptr(self.xq), ptr(self.xs), rows, x.shape[1], None, None,
                                                    current_stream()), "quant_fp8_rowwise")
        return self.xq

    def _decode_layers(self, sq=1):
        """The layers over B * sq rows: the decode step (sq = 1) or the verify step (sq = max_draft + 1)."""
        lib, B, D = self.lib, self.B * sq, self.D
        st = current_stream()
        h, h2 = self.h, self.h2
        qkv_w = (self.Hq + 2 * self.Hkv) * D
        n_layers = len(self.layers)
        # what the norms before qkv and w13 write, and what those linears read
        fp8 = self.weight_format == "fp8"
        norm_out, x_in = (dict(y=None, q=self.xq, qs=self.xs), self.xq) if fp8 else (dict(y=self.xn), self.xn)
        self._norm(h, self.layers[0]["attn_norm"], **norm_out, rows=B)
        for li, lw in enumerate(self.layers):
            if self.capture_h is not None:
                self.capture_h.append(h.clone())
            last = li + 1 == n_layers
            next_norm = self.norm if last else self.layers[li + 1]["attn_norm"]
            self._layer_linear(x_in, lw, "wqkv", self.qkv, B)
            k_view = self.qkv[:, self.Hq * D:]
            if sq == 1 and self.fuse_rope:
                # rotary (q and the new k) inside the attention kernel: q / k / v are views of the qkv GEMM output; an
                # e4m3 cache (which implies fuse_rope) rounds the new k / v rows to e4m3 as they are stored
                self._gqa_attention(li, self.qkv, k_view, rope=(self.cos, self.sin))
            else:
                cos, sin = (self.cos, self.sin) if sq == 1 else (self.verify_cos, self.verify_sin)
                check(lib.chitu_b200_rotary_interleaved(ptr(self.qkv), ptr(k_view), ptr(self.q_rot), ptr(self.k_rot),
                                                        ptr(cos), ptr(sin), B, self.Hq, self.Hkv, D, qkv_w, D, qkv_w, D,
                                                        _lib.CB_BF16, st), "rotary")
                self._gqa_attention(li, self.q_rot, self.k_rot, sq)
            # h2 = wo(o) + h
            self._row_parallel(lambda out, res: self._layer_linear(self._quant(self.attn_out, B), lw, "wo", out, B,
                                                                   residual=res),
                               lambda: self.comm.linear_push(self.attn_out, lw["wo"], B, self.lin_ws),
                               h, h2, lw["ffn_norm"], **norm_out, rows=B)
            if self.fuse_silu:
                self._layer_linear(x_in, lw, "w13", self.act, B, silu_pairs=True)
            else:                          # linear_impl=1, bf16 only: the SIMT GEMV, then SiluAndMul
                self._linear(self.xn, lw["w13"], self.gate_up, B)
                check(lib.chitu_b200_silu_and_mul(ptr(self.gate_up), ptr(self.act), B, self.F, _lib.CB_BF16, st), "silu")
            # h = w2(act) + h2; the head reads the final norm in bf16
            self._row_parallel(lambda out, res: self._layer_linear(self._quant(self.act, B), lw, "w2", out, B,
                                                                   residual=res),
                               lambda: self.comm.linear_push(self.act, lw["w2"], B, self.lin_ws),
                               h2, h, next_norm, **(dict(y=self.xn) if last else norm_out), rows=B)
        if self.capture_h is not None:
            self.capture_h.append(h.clone())

    # ---- speculative verify step ------------------------------------------------------------------
    def _verify_body(self):
        lib, B, k, cfg = self.lib, self.B, self.max_draft, self.cfg
        M, st = B * (k + 1), current_stream()
        self.verify_tokens[:, 0].copy_(self.tokens)
        self.verify_tokens[:, 1:].copy_(self.draft_tokens)
        # row b * (k + 1) + i sits at position seq_lens[b] + i
        torch.add(self.seq_lens.view(B, 1), self.verify_offsets, out=self.verify_pos)
        torch.index_select(self.cos_table, 0, self.verify_pos.view(-1), out=self.verify_cos)
        torch.index_select(self.sin_table, 0, self.verify_pos.view(-1), out=self.verify_sin)
        check(lib.chitu_b200_embedding(ptr(self.verify_tokens), ptr(self.embed), ptr(self.h), M, cfg.dim, 0,
                                       cfg.vocab_size, _lib.CB_BF16, st), "embedding")
        self._decode_layers(sq=k + 1)
        self._linear(self.xn, self.head, self.logits, M)
        vocab_local = self.head.shape[0]
        if self.sampled_verify:
            torch.rand(self.uniforms.shape, generator=self.sample_generator, out=self.uniforms)
            dp = self.draft_probs
            check(lib.chitu_b200_spec_accept_sampled(ptr(self.logits), self.logits.stride(0), vocab_local, _lib.CB_BF16,
                                                     ptr(self.temperatures), ptr(self.top_ks), ptr(self.top_ps),
                                                     ptr(self.draft_tokens), ptr(self.n_draft), ptr(dp),
                                                     0 if dp is None else dp.stride(1), ptr(self.u_accept),
                                                     ptr(self.u_draw), ptr(self.seq_lens), ptr(self.out_tokens),
                                                     ptr(self.accepted), ptr(self.next_tokens), B, k, ptr(self.spec_ws),
                                                     self.spec_ws.numel(), st), "spec_accept_sampled")
            return
        check(lib.chitu_b200_argmax(ptr(self.logits), ptr(self.target), M, vocab_local, _lib.CB_BF16, st), "argmax")
        if self.tp_on:
            self.target.view(-1).copy_(global_argmax(self.logits, self.target.view(-1), self.tp_rank, vocab_local,
                                                     self.pg, self.verify_gather))
        check(lib.chitu_b200_spec_accept_greedy(ptr(self.target), ptr(self.draft_tokens), ptr(self.n_draft),
                                                ptr(self.seq_lens), ptr(self.out_tokens), ptr(self.accepted),
                                                ptr(self.next_tokens), B, k, st), "spec_accept_greedy")

    def _need_verify(self):
        if self.max_draft == 0:
            raise ValueError("this engine has no verify step: build it with max_draft > 0")

    def capture_verify(self):
        """Capture the verify step in a CUDA graph of its own (the decode step's graph is separate)."""
        self._need_verify()
        self.verify_graph, self.launches_per_verify = self._capture(
            self._verify_body, generators=(self.sample_generator,) if self.sampled_verify else ())

    def verify_step(self):
        """One verify step over the persistent buffers (tokens in self.tokens, drafts in self.draft_tokens / n_draft)."""
        self._need_verify()
        self.launches_per_verify = self._run(self.verify_graph, self._verify_body, self.launches_per_verify)

    def verify(self, tokens_host: torch.Tensor, drafts_host: torch.Tensor, n_draft_host: torch.Tensor,
               temperature=None, top_k=None, top_p=None, draft_probs=None):
        """Speculative verification, greedy (or sampled: below).  tokens_host int64 [B]: each request's last token (what `decode` takes);
        drafts_host int64 [B, k'] with k' <= max_draft: the proposed continuations; n_draft_host int32 [B] in 0..k':
        how many of a request's drafts to check.  One step runs every request's token and drafts through the model
        (positions seq_lens[b] .. seq_lens[b] + max_draft), accepts the leading drafts equal to the model's greedy
        choice and advances seq_lens by the accepted count + 1 on the device.

        Returns host (out_tokens int64 [B, max_draft + 1]: the accepted drafts then the model's next token, -1 after;
        accepted int32 [B]).  self.next_tokens holds each request's last emitted token, the input of the next step.
        K / V rows are written for all max_draft + 1 positions; those past the accepted ones stay beyond seq_lens and are
        overwritten by later steps.  The caller keeps seq_lens[b] + max_draft + 1 <= max_seq_len, and the cache pages
        for those positions in the block table.

        An engine built with sampled_verify=True takes each request's temperature fp32 [B] (finite; <= 0: greedy),
        top_k int32 [B] (<= 0: no top-k) and top_p fp32 [B] (in (0, 1]) on the host, and accepts by speculative
        sampling; with draft_probs=True also draft_probs fp32 [B, k', V], the drafter's distribution at each draft.
        A greedy engine takes none of them."""
        self._need_verify()
        B, k = self.B, self.max_draft
        drafts_host = torch.as_tensor(drafts_host)
        n_draft_host = torch.as_tensor(n_draft_host)
        if tuple(torch.as_tensor(tokens_host).shape) != (B,):
            raise ValueError(f"tokens must be [{B}], not {tuple(torch.as_tensor(tokens_host).shape)}")
        if drafts_host.dim() != 2 or drafts_host.shape[0] != B or drafts_host.shape[1] > k:
            raise ValueError(f"drafts must be [{B}, k'] with k' <= max_draft = {k}, not {tuple(drafts_host.shape)}")
        if tuple(n_draft_host.shape) != (B,):
            raise ValueError(f"n_draft must be [{B}], not {tuple(n_draft_host.shape)}")
        if bool(((n_draft_host < 0) | (n_draft_host > drafts_host.shape[1])).any()):
            raise ValueError(f"n_draft must lie in 0..{drafts_host.shape[1]}")
        sampling = self._sampling_args(temperature, top_k, top_p, draft_probs, drafts_host.shape[1])
        self.tokens.copy_(tokens_host, non_blocking=True)
        if sampling is not None:
            temperature, top_k, top_p, draft_probs = sampling
            self.temperatures.copy_(temperature, non_blocking=True)
            self.top_ks.copy_(top_k, non_blocking=True)
            self.top_ps.copy_(top_p, non_blocking=True)
            if draft_probs is not None:
                self.draft_probs[:, :draft_probs.shape[1]].copy_(draft_probs, non_blocking=True)
        if drafts_host.shape[1] < k:       # the step always runs max_draft rows per request; pad with token 0
            drafts_host = torch.cat([drafts_host, drafts_host.new_zeros(B, k - drafts_host.shape[1])], dim=1)
        self.draft_tokens.copy_(drafts_host, non_blocking=True)
        self.n_draft.copy_(n_draft_host, non_blocking=True)
        self.verify_step()
        return self.out_tokens.cpu(), self.accepted.cpu()

    def _sampling_args(self, temperature, top_k, top_p, draft_probs, k_in):
        """The host-side checks of verify's sampling arguments: None on a greedy engine, else them as host tensors of
        the buffers' dtypes."""
        given = [x is not None for x in (temperature, top_k, top_p)]
        if not self.sampled_verify:
            if any(given) or draft_probs is not None:
                raise ValueError("temperature / top_k / top_p / draft_probs need an engine built with "
                                 "sampled_verify=True")
            return None
        if not all(given):
            raise ValueError("a sampled verify step needs temperature, top_k and top_p for every request")
        B = self.B
        temperature = torch.as_tensor(temperature).to(torch.float32)
        top_k = torch.as_tensor(top_k).to(torch.int32)
        top_p = torch.as_tensor(top_p).to(torch.float32)
        for name, t in (("temperature", temperature), ("top_k", top_k), ("top_p", top_p)):
            if t.is_cuda or tuple(t.shape) != (B,):
                raise ValueError(f"{name} must be a host tensor [{B}], not {tuple(t.shape)} on {t.device}")
        if not bool(torch.isfinite(temperature).all()):
            raise ValueError("temperature must be finite")
        if not bool(((top_p > 0) & (top_p <= 1)).all()):
            raise ValueError("top_p must lie in (0, 1]")
        if self.draft_probs is None:
            if draft_probs is not None:
                raise ValueError("draft_probs need an engine built with draft_probs=True")
        else:
            if draft_probs is None:
                raise ValueError("this engine verifies draft-model drafts: pass draft_probs")
            draft_probs = torch.as_tensor(draft_probs)
            V = self.draft_probs.shape[2]
            if draft_probs.is_cuda or draft_probs.dtype != torch.float32 or tuple(draft_probs.shape) != (B, k_in, V):
                raise ValueError(f"draft_probs must be a host fp32 tensor [{B}, {k_in}, {V}], not {draft_probs.dtype} "
                                 f"{tuple(draft_probs.shape)} on {draft_probs.device}")
        return temperature, top_k, top_p, draft_probs
