"""Decode-step engine: the caller side of the hot path, wired exactly like the reference's
`Transformer.decode_single_device` (chitu/models/model.py:467-474) + `TransformerBlockLlama`
(models/model_llama.py:152-185) + `Attention.decode_forward_paged` (models/model.py:167-198),
but every operator is a libchitu_b200 kernel and the whole step is one CUDA graph
(reference: per-batch-size graph capture, models/model.py:537-622).

It exists so `bench.py` can measure BASELINE.json's metric (decode tokens/s) on synthetic
weights of the named architecture; it is not a re-implementation of the reference's model zoo
(checkpoint loading, prefill, PP stay in the reference).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib, workspace
from ._lib import check, current_stream, dtype_code, ptr
from .tensor_parallel import global_argmax


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


class LlamaDecodeEngine:
    """Single-GPU (tp=1) or tensor-parallel LLaMA decode.  Weights are random (`do_load=False`,
    serve_config.yaml:9).  KV cache layout = PagedKVCacheManager (cache_manager.py:71-87):
    paged_k_cache / paged_v_cache [L, num_blocks, page, n_local_kv_heads, head_dim], page 256
    (backend.py:237), persistent int32 block_table [max_reqs, max_blocks] and seq_lens buffers."""

    def __init__(self, cfg: LlamaConfig, max_reqs: int, max_seq_len: int, device="cuda:0", page_size: int = 256,
                 seed: int = 0, tp_rank: int = 0, tp_size: int = 1, process_group=None, linear_impl: int = 0,
                 use_fused_allreduce: bool = True):
        self.cfg, self.B, self.device = cfg, max_reqs, torch.device(device)
        self.tp_rank, self.tp_size, self.pg = tp_rank, tp_size, process_group
        self.tp_gather = None
        self.linear_impl = linear_impl
        self.lib = _lib.load()
        dt = torch.bfloat16
        D = cfg.head_dim
        assert cfg.n_heads % tp_size == 0 and cfg.n_kv_heads % tp_size == 0
        self.Hq, self.Hkv, self.D = cfg.n_heads // tp_size, cfg.n_kv_heads // tp_size, D
        self.F = cfg.ffn_dim // tp_size
        self.page = page_size
        self.max_blocks = max_seq_len // page_size + 1
        nblk = self.max_blocks * max_reqs
        g = torch.Generator(device=self.device).manual_seed(seed + 1000 * tp_rank)

        def rnd(*shape, scale=0.02):
            return (torch.randn(*shape, generator=g, dtype=torch.float32, device=self.device) * scale).to(dt)

        dim = cfg.dim
        g_rep = torch.Generator(device=self.device).manual_seed(seed + 7)     # replicated across TP ranks
        self.embed = (torch.randn(cfg.vocab_size, dim, generator=g_rep, dtype=torch.float32, device=self.device) * 0.02).to(dt)
        self.layers = []
        for _ in range(cfg.n_layers):
            self.layers.append(dict(
                attn_norm=torch.ones(dim, dtype=dt, device=self.device),
                ffn_norm=torch.ones(dim, dtype=dt, device=self.device),
                # column-parallel wq|wk|wv merged along N (shards of each concatenated); row-parallel wo
                wqkv=rnd((self.Hq + 2 * self.Hkv) * D, dim),
                wo=rnd(dim, self.Hq * D),
                w13=rnd(2 * self.F, dim),          # [w1 (gate) ; w3 (up)]  (interleaved below when the epilogue fuses SiLU)
                w2=rnd(dim, self.F),
            ))
        self.norm = torch.ones(dim, dtype=dt, device=self.device)
        self.head = rnd(cfg.vocab_size // tp_size, dim)
        self.k_cache = torch.zeros(cfg.n_layers, nblk, page_size, self.Hkv, D, dtype=dt, device=self.device)
        self.v_cache = torch.zeros_like(self.k_cache)
        self.block_table = torch.zeros(max_reqs, self.max_blocks, dtype=torch.int32, device=self.device)
        self.seq_lens = torch.zeros(max_reqs, dtype=torch.int32, device=self.device)
        # precompute_freqs_cis (models/model.py:81-89) as cos/sin tables
        freqs = 1.0 / (cfg.rope_theta ** (torch.arange(0, D, 2)[: D // 2].float() / D))
        t = torch.arange(max_seq_len * 2, dtype=torch.float32)
        ang = torch.outer(t, freqs)
        self.cos_table, self.sin_table = ang.cos().to(self.device), ang.sin().to(self.device)
        # persistent activations (CUDA-graph safe)
        B = max_reqs
        self.tokens = torch.zeros(B, dtype=torch.int64, device=self.device)
        self.cos = torch.zeros(B, D // 2, dtype=torch.float32, device=self.device)
        self.sin = torch.zeros_like(self.cos)
        self.h = torch.zeros(B, dim, dtype=dt, device=self.device)
        self.h2 = torch.zeros_like(self.h)
        self.xn = torch.zeros_like(self.h)
        self.qkv = torch.zeros(B, (self.Hq + 2 * self.Hkv) * D, dtype=dt, device=self.device)
        self.q_rot = torch.zeros(B, self.Hq, D, dtype=dt, device=self.device)
        self.k_rot = torch.zeros(B, self.Hkv, D, dtype=dt, device=self.device)
        self.attn_out = torch.zeros(B, self.Hq * D, dtype=dt, device=self.device)
        self.gate_up = torch.zeros(B, 2 * self.F, dtype=dt, device=self.device)
        self.act = torch.zeros(B, self.F, dtype=dt, device=self.device)
        self.logits = torch.zeros(B, cfg.vocab_size // tp_size, dtype=dt, device=self.device)
        self.next_tokens = torch.zeros(B, dtype=torch.int64, device=self.device)
        if self.tp_size > 1:
            self.tp_gather = torch.empty(self.tp_size, B, 2, dtype=torch.float32, device=self.device)
        n_attn = self.lib.chitu_b200_attn_workspace_bytes(B, self.Hq, D, 64)
        self.attn_ws = torch.empty(n_attn, dtype=torch.uint8, device=self.device)
        n_lin = max(self.lib.chitu_b200_linear_workspace_bytes(B, max(2 * self.F, cfg.vocab_size // tp_size)), 256)
        self.lin_ws = torch.zeros(n_lin, dtype=torch.uint8, device=self.device)   # tickets start at 0
        self.max_seq_len = max_seq_len
        import os
        # SiluAndMul inside the w13 GEMM epilogue: the merged gate/up weight is stored with its rows interleaved
        # (row 2i = gate_i, row 2i+1 = up_i) — a load-time permutation of the reference's merged tensor
        self.fuse_silu = linear_impl != 1
        if self.fuse_silu:
            for lw in self.layers:
                lw["w13"] = lw["w13"].view(2, self.F, dim).transpose(0, 1).reshape(2 * self.F, dim).contiguous()
        # rotary fused into the tensor-core decode kernel (head dim 128, power-of-two pages)
        self.fuse_rope = D == 128 and (page_size & (page_size - 1)) == 0 and self.Hq // self.Hkv in (1, 2, 4, 8)
        self.graph = None
        self.launches_per_step = 0
        # push mode: the row-parallel GEMM's epilogue starts the all-reduce (A/B: CHITU_B200_AR_PUSH=0 -> pull kernel)
        self.ar_push = os.environ.get("CHITU_B200_AR_PUSH", "1") != "0" and linear_impl != 1
        # fused one-shot all-reduce + residual + RMSNorm over NVLink peer memory (csrc/comm.cu); NCCL otherwise
        self.comm = None
        if tp_size > 1 and process_group is not None and use_fused_allreduce:
            from .comm import FusedAllReduce
            self.comm = FusedAllReduce(process_group, max_reqs, dim, self.device)

    # ---- cache bookkeeping (host side of PagedKVCacheManager, cache_manager.py:148-209) ----------
    def set_synthetic_context(self, seq_len: int, seed: int = 2):
        """Fill the KV cache with `seq_len` random cached tokens per request and a shuffled
        (non-identity) block table (SURVEY §8d synthetic inputs)."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        gd = torch.Generator(device=self.device).manual_seed(seed + 11)     # deterministic cache contents
        nblk = self.k_cache.shape[1]
        perm = torch.randperm(nblk, generator=g).to(torch.int32)
        self.block_table.copy_(perm.view(self.B, self.max_blocks))
        self.seq_lens.fill_(seq_len)
        for l in range(self.cfg.n_layers):
            self.k_cache[l].normal_(0, 1, generator=gd)
            self.v_cache[l].normal_(0, 1, generator=gd)

    def ref_layers(self):
        """The layer weights in the REFERENCE's layout (w13 = [w1 ; w3] halves) for the oracle side of the tests."""
        out = []
        for lw in self.layers:
            d = dict(lw)
            if self.fuse_silu:
                d["w13"] = lw["w13"].view(self.F, 2, self.cfg.dim).transpose(0, 1).reshape(2 * self.F, self.cfg.dim).contiguous()
            out.append(d)
        return out

    # ---- one decode step ---------------------------------------------------------------------------
    def _linear(self, x, w, y, M, residual=None):
        N, K = w.shape
        check(self.lib.chitu_b200_linear_bf16(ptr(x), ptr(w), None, ptr(residual), ptr(y), M, N, K, _lib.CB_BF16,
                                              ptr(self.lin_ws), self.lin_ws.numel(), self.linear_impl,
                                              current_stream()), "linear_bf16")

    def _rmsnorm(self, x, w, y, M):
        check(self.lib.chitu_b200_rmsnorm(ptr(x), ptr(w), ptr(y), M, self.cfg.dim, self.cfg.norm_eps, _lib.CB_BF16,
                                          current_stream()), "rmsnorm")

    def _allreduce(self, t):
        if self.tp_size > 1:
            torch.distributed.all_reduce(t, group=self.pg)

    def _step_body(self):
        lib, B, D = self.lib, self.B, self.D
        st = current_stream()
        cfg = self.cfg
        # prepare_freqs_cis_decode (models/model.py:429-448): gather cos/sin by position
        torch.index_select(self.cos_table, 0, self.seq_lens, out=self.cos)
        torch.index_select(self.sin_table, 0, self.seq_lens, out=self.sin)
        vocab_local = cfg.vocab_size // self.tp_size
        check(lib.chitu_b200_embedding(ptr(self.tokens), ptr(self.embed), ptr(self.h), B, cfg.dim,
                                       0, cfg.vocab_size, _lib.CB_BF16, st), "embedding")
        h, h2 = self.h, self.h2
        qkv_w = (self.Hq + 2 * self.Hkv) * D
        n_layers = len(self.layers)

        def reduce_add_norm(partial, residual, h_out, norm_w):
            """h_out = all_reduce(partial) + residual ; self.xn = RMSNorm(h_out) * norm_w"""
            if self.comm is not None:
                self.comm(partial, residual, h_out, norm_w, self.xn, None, None, B, cfg.dim, cfg.norm_eps)
            else:
                self._allreduce(partial)
                check(lib.chitu_b200_add(ptr(partial), ptr(residual), ptr(h_out), B * cfg.dim, _lib.CB_BF16, st), "add")
                self._rmsnorm(h_out, norm_w, self.xn, B)

        self._rmsnorm(h, self.layers[0]["attn_norm"], self.xn, B)
        for li, lw in enumerate(self.layers):
            next_norm = self.layers[li + 1]["attn_norm"] if li + 1 < n_layers else self.norm
            self._linear(self.xn, lw["wqkv"], self.qkv, B)
            q_view, k_view = self.qkv, self.qkv[:, self.Hq * D:]
            v_view = self.qkv[:, (self.Hq + self.Hkv) * D:]
            if self.fuse_rope:
                # rotary (q and the new k) inside the attention kernel: q / k / v are views of the qkv GEMM output
                check(lib.chitu_b200_gqa_paged_decode_rope(
                    ptr(q_view), qkv_w, ptr(self.k_cache[li]), ptr(self.v_cache[li]), ptr(k_view), ptr(v_view), qkv_w, qkv_w,
                    ptr(self.cos), ptr(self.sin), ptr(self.seq_lens), ptr(self.block_table), self.max_blocks, B, self.Hq,
                    self.Hkv, D, self.page, self.max_seq_len, 1.0 / math.sqrt(D), ptr(self.attn_out), ptr(self.attn_ws),
                    self.attn_ws.numel(), _lib.CB_BF16, st), "gqa_paged_decode_rope")
            else:
                check(lib.chitu_b200_rotary_interleaved(ptr(q_view), ptr(k_view), ptr(self.q_rot), ptr(self.k_rot),
                                                        ptr(self.cos), ptr(self.sin), B, self.Hq, self.Hkv, D, qkv_w, D,
                                                        qkv_w, D, _lib.CB_BF16, st), "rotary")
                check(lib.chitu_b200_gqa_paged_decode(
                    ptr(self.q_rot), ptr(self.k_cache[li]), ptr(self.v_cache[li]), ptr(self.k_rot), ptr(v_view),
                    self.Hkv * D, qkv_w, ptr(self.seq_lens), ptr(self.block_table), self.max_blocks, B, self.Hq,
                    self.Hkv, D, self.page, self.max_seq_len, 1.0 / math.sqrt(D), ptr(self.attn_out), ptr(self.attn_ws),
                    self.attn_ws.numel(), _lib.CB_BF16, st), "gqa_paged_decode")
            if self.tp_size == 1:
                self._linear(self.attn_out, lw["wo"], h2, B, residual=h)      # h2 = wo(o) + h
                self._rmsnorm(h2, lw["ffn_norm"], self.xn, B)
            elif self.comm is not None and self.ar_push:
                self.comm.linear_push(self.attn_out, lw["wo"], B, self.lin_ws)
                self.comm.consume(h, h2, lw["ffn_norm"], self.xn, None, None, B, cfg.dim, cfg.norm_eps)
            else:
                self._linear(self.attn_out, lw["wo"], h2, B)
                reduce_add_norm(h2, h, h2, lw["ffn_norm"])
            if self.fuse_silu:
                check(lib.chitu_b200_linear_bf16_silu_pairs(ptr(self.xn), ptr(lw["w13"]), ptr(self.act), B, 2 * self.F, cfg.dim,
                                                            ptr(self.lin_ws), self.lin_ws.numel(), st), "w13 + silu")
            else:
                self._linear(self.xn, lw["w13"], self.gate_up, B)
                check(lib.chitu_b200_silu_and_mul(ptr(self.gate_up), ptr(self.act), B, self.F, _lib.CB_BF16, st), "silu")
            if self.tp_size == 1:
                self._linear(self.act, lw["w2"], h, B, residual=h2)           # h = w2(act) + h2
                self._rmsnorm(h, next_norm, self.xn, B)
            elif self.comm is not None and self.ar_push:
                self.comm.linear_push(self.act, lw["w2"], B, self.lin_ws)
                self.comm.consume(h2, h, next_norm, self.xn, None, None, B, cfg.dim, cfg.norm_eps)
            else:
                self._linear(self.act, lw["w2"], h, B)
                reduce_add_norm(h, h2, h, next_norm)
        self._linear(self.xn, self.head, self.logits, B)          # self.xn = norm(h) already
        check(lib.chitu_b200_argmax(ptr(self.logits), ptr(self.next_tokens), B, vocab_local, _lib.CB_BF16, st),
              "argmax")
        if self.tp_size > 1:
            # vocab-parallel head: the reference all-gathers the logits shards before sampling
            # (tensor_parallel.py:94-102); the same token from a (max, index) all-gather of B*8 bytes per rank
            self.next_tokens.copy_(global_argmax(self.logits, self.next_tokens, self.tp_rank, vocab_local, self.pg,
                                                 self.tp_gather))
        self.seq_lens.add_(1)     # finalize_cache_single_decode (cache_manager.py)

    def capture(self):
        """Capture the decode step in a CUDA graph (models/model.py:572-611)."""
        torch.cuda.synchronize(self.device)
        saved = self.seq_lens.clone()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(2):
                self._step_body()         # warm-up outside capture
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
        """One decode step over the persistent buffers (tokens in self.tokens)."""
        if self.graph is not None:
            self.graph.replay()
        else:
            before = _lib.launch_count()
            self._step_body()
            self.launches_per_step = _lib.launch_count() - before

    def decode(self, tokens_host: torch.Tensor) -> torch.Tensor:
        """Public API: host tokens [B] int64 (pinned) -> host next tokens [B] (greedy).
        Includes the H2D copy of the inputs and the D2H read of the result."""
        self.tokens.copy_(tokens_host, non_blocking=True)
        self.step()
        return self.next_tokens.cpu()
