"""DeepSeek-V3/R1 decode step (MLA-absorb paged decode + FP8 block-scaled linears + fused MoE),
wired like the reference's `TransformerBlockDeepSeekV3.forward` (models/model_deepseek_v3.py:1100-1114),
`AttentionDeepSeekV3.decode_forward_paged` (:672-699), `MLPDeepSeekV3.forward` (:755-771) and
`MoEDeepSeekV3.forward` (:921-1011), with every operator a libchitu_b200 kernel.

Tensor parallel exactly where the reference shards (SURVEY §8e): heads (wq_b / wkv_b / wo), FFN and
expert intermediate dims; wqkv_a, norms, gate replicated; the MLA KV cache replicated on every rank
(backend.py:196-197); all-reduce after wo and after each FFN/MoE (tensor_parallel.py:166,
model_deepseek_v3.py:1011).  `tp_size` shapes the per-rank shard; with `process_group=None` and
tp_size>1 the engine runs ONE rank's shard without collectives ("shard mode": the per-rank kernel
time of the tp=8 configuration measured on a single GPU).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib
from ._lib import check, current_stream, ptr
from .tensor_parallel import global_argmax

BF = torch.bfloat16
F8 = torch.float8_e4m3fn


@dataclass
class DeepSeekConfig:
    """chitu/config/models/DeepSeek-R1.yaml:6-29."""
    vocab_size: int = 129280
    dim: int = 7168
    inter_dim: int = 18432
    moe_inter_dim: int = 2048
    n_layers: int = 61
    n_dense_layers: int = 3
    n_heads: int = 128
    n_routed_experts: int = 256
    n_shared_experts: int = 1
    n_activated_experts: int = 8
    n_expert_groups: int = 8
    n_limited_groups: int = 4
    route_scale: float = 2.5
    score_func: str = "sigmoid"
    q_lora_rank: int = 1536
    kv_lora_rank: int = 512
    qk_nope_head_dim: int = 128
    qk_rope_head_dim: int = 64
    v_head_dim: int = 128
    rope_theta: float = 10000.0
    rope_factor: float = 40.0
    norm_eps: float = 1e-6

    @property
    def softmax_scale(self):
        # compute_softmax_scale_deepseek_v3 (model_deepseek_v3.py:1441-1445)
        mscale = 0.1 * math.log(self.rope_factor) + 1.0
        return ((self.qk_nope_head_dim + self.qk_rope_head_dim) ** -0.5) * mscale * mscale


DEEPSEEK_R1 = DeepSeekConfig()


def quantize_fp8_block(w: torch.Tensor, block: int = 128):
    """bf16/fp32 [..., N, K] -> (fp8 e4m3 weights, fp32 scales [..., ceil(N/128), ceil(K/128)]) in the
    DeepSeek `weight_scale_inv` convention (backend.py:453; SURVEY §8d synthetic inputs)."""
    *lead, N, K = w.shape
    nb, kb = (N + block - 1) // block, (K + block - 1) // block
    wp = torch.zeros(*lead, nb * block, kb * block, dtype=torch.float32, device=w.device)
    wp[..., :N, :K] = w
    blocks = wp.view(*lead, nb, block, kb, block)
    s = (blocks.abs().amax(dim=(-3, -1)) / 448.0).clamp(min=1e-12)
    q = (blocks / s[..., :, None, :, None]).reshape(*lead, nb * block, kb * block)[..., :N, :K]
    return q.to(F8).contiguous(), s.float().contiguous()


def yarn_freqs(cfg: DeepSeekConfig, max_pos: int) -> torch.Tensor:
    """precompute_freqs_cis_deepseek_v3 (model_deepseek_v3.py:1353-1438) -> angles [max_pos, rope/2]."""
    dim, base, factor = cfg.qk_rope_head_dim, cfg.rope_theta, cfg.rope_factor
    beta_fast, beta_slow, original = 32, 1, 4096

    def corr_dim(num_rot):
        return dim * math.log(original / (num_rot * 2 * math.pi)) / (2 * math.log(base))

    freqs = 1.0 / (base ** (torch.arange(0, dim, 2, dtype=torch.float32) / dim))
    if max_pos > original:
        low = max(math.floor(corr_dim(beta_fast)), 0)
        high = min(math.ceil(corr_dim(beta_slow)), dim - 1)
        if low == high:
            high += 0.001
        ramp = torch.clamp((torch.arange(dim // 2, dtype=torch.float32) - low) / (high - low), 0, 1)
        smooth = 1 - ramp
        freqs = freqs / factor * (1 - smooth) + freqs * smooth
    return torch.outer(torch.arange(max_pos, dtype=torch.float32), freqs)


class DeepSeekDecodeEngine:
    def __init__(self, cfg: DeepSeekConfig, max_reqs: int, max_seq_len: int, device="cuda:0", seed: int = 0,
                 tp_rank: int = 0, tp_size: int = 8, process_group=None, page_size: int = 64,
                 cache_dequant_wkv_b: bool = True, use_fused_allreduce: bool = True):
        self.cfg, self.B, self.device = cfg, max_reqs, torch.device(device)
        self.tp_rank, self.tp_size, self.pg = tp_rank, tp_size, process_group
        self.lib = _lib.load()
        self.page = page_size                          # backend.py:234-237: paged + absorb => 64
        c = cfg
        T = tp_size
        assert c.n_heads % T == 0
        self.H = c.n_heads // T
        self.qk_head = c.qk_nope_head_dim + c.qk_rope_head_dim
        self.C, self.R = c.kv_lora_rank, c.qk_rope_head_dim
        self.F_dense = c.inter_dim // T
        self.F_moe = c.moe_inter_dim // T
        self.cache_dequant = cache_dequant_wkv_b
        dev = self.device
        g = torch.Generator(device=dev).manual_seed(seed + 1000 * tp_rank)
        g_rep = torch.Generator(device=dev).manual_seed(seed + 7)        # replicated weights: same on all ranks

        def rnd(gen, *shape, scale=0.02):
            return torch.randn(*shape, generator=gen, dtype=torch.float32, device=dev) * scale

        def fp8(gen, *shape):
            # quantise in slabs to bound the fp32 temporaries for the [E, N, K] expert tensors
            if len(shape) == 3:
                qs, ss = [], []
                for e0 in range(0, shape[0], 32):
                    q, s = quantize_fp8_block(rnd(gen, min(32, shape[0] - e0), *shape[1:]))
                    qs.append(q), ss.append(s)
                return torch.cat(qs), torch.cat(ss)
            return quantize_fp8_block(rnd(gen, *shape))

        dim = c.dim
        self.embed = rnd(g_rep, c.vocab_size, dim).to(BF)
        self.layers = []
        for li in range(c.n_layers):
            L = dict(attn_norm=torch.ones(dim, dtype=BF, device=dev), ffn_norm=torch.ones(dim, dtype=BF, device=dev),
                     q_norm=torch.ones(c.q_lora_rank, dtype=BF, device=dev),
                     kv_norm=torch.ones(c.kv_lora_rank, dtype=BF, device=dev))
            L["wqkv_a"], L["wqkv_a_s"] = fp8(g_rep, c.q_lora_rank + self.C + self.R, dim)      # replicated
            L["wq_b"], L["wq_b_s"] = fp8(g, self.H * self.qk_head, c.q_lora_rank)
            L["wkv_b"], L["wkv_b_s"] = fp8(g, self.H * (c.qk_nope_head_dim + c.v_head_dim), self.C)
            L["wo"], L["wo_s"] = fp8(g, dim, self.H * c.v_head_dim)
            if li < c.n_dense_layers:
                L["w13"], L["w13_s"] = fp8(g, 2 * self.F_dense, dim)
                L["w2"], L["w2_s"] = fp8(g, dim, self.F_dense)
            else:
                L["gate_w"] = rnd(g_rep, c.n_routed_experts, dim).to(BF)
                L["gate_b"] = rnd(g_rep, c.n_routed_experts, scale=0.01)                       # fp32 bias
                # routed experts + the shared expert stored as expert index n_routed_experts, exactly like the
                # reference's stacked w1w3 / w2 tensors (model_deepseek_v3.py:1167-1191: `weight[-1]` is shared)
                assert c.n_shared_experts == 1
                L["we1"], L["we1_s"] = fp8(g, c.n_routed_experts + 1, 2 * self.F_moe, dim)
                L["we2"], L["we2_s"] = fp8(g, c.n_routed_experts + 1, dim, self.F_moe)
                L["ws13"], L["ws13_s"] = L["we1"][-1], L["we1_s"][-1]      # views (used by the tests)
                L["ws2"], L["ws2_s"] = L["we2"][-1], L["we2_s"][-1]
            if self.cache_dequant:
                # SURVEY §8f n1: dequantise wkv_b once instead of every step (model_deepseek_v3.py:516-528)
                L["wkv_b_bf16"] = self._dequant(L["wkv_b"], L["wkv_b_s"])
            self.layers.append(L)
        self.norm = torch.ones(dim, dtype=BF, device=dev)
        self.head = rnd(g, c.vocab_size // T, dim).to(BF)
        # paged MLA cache: [L, num_blocks, 64, 576], replicated on every rank (cache_manager.py:71-76)
        self.max_blocks = max_seq_len // page_size + 1
        nblk = self.max_blocks * max_reqs
        self.kv_cache = torch.zeros(c.n_layers, nblk, page_size, self.C + self.R, dtype=BF, device=dev)
        self.block_table = torch.zeros(max_reqs, self.max_blocks, dtype=torch.int32, device=dev)
        self.seq_lens = torch.zeros(max_reqs, dtype=torch.int32, device=dev)
        ang = yarn_freqs(c, max_seq_len * 2)
        self.cos_table, self.sin_table = ang.cos().to(dev), ang.sin().to(dev)
        B = max_reqs
        z = lambda *s, dt=BF: torch.zeros(*s, dtype=dt, device=dev)
        self.tokens = torch.zeros(B, dtype=torch.int64, device=dev)
        self.cos, self.sin = z(B, self.R // 2, dt=torch.float32), z(B, self.R // 2, dt=torch.float32)
        self.h, self.h2, self.xn = z(B, dim), z(B, dim), z(B, dim)
        kmax = max(dim, self.F_dense, self.H * c.v_head_dim, c.q_lora_rank)
        self.xq = torch.zeros(B, kmax, dtype=F8, device=dev)
        self.xs = z(B, kmax // 128 + 1, dt=torch.float32)
        self.qkv_a = z(B, c.q_lora_rank + self.C + self.R)
        self.qa_n = z(B, c.q_lora_rank)
        self.q = z(B, self.H, self.qk_head)
        self.q_pe = z(B, self.H, self.R)
        self.q_abs = z(B, self.H, self.C)
        self.new_kv = z(B, self.C + self.R)
        self.o_lat = z(B, self.H, self.C)
        self.o = z(B, self.H * c.v_head_dim)
        self.wkv_tmp = z(self.H * (c.qk_nope_head_dim + c.v_head_dim), self.C)
        self.ff = z(B, 2 * max(self.F_dense, self.F_moe))
        self.act = z(B, max(self.F_dense, self.F_moe))
        self.y, self.y1 = z(B, dim), z(B, dim)
        # routing results of every layer stay resident (bench.py counts the distinct experts per layer)
        # one extra slot per token = the shared expert (id n_routed_experts, weight 1): it rides through the
        # grouped expert GEMM instead of five separate launches
        self.topk1 = c.n_activated_experts + 1
        self.gate_w_all = z(c.n_layers, B, self.topk1)
        self.gate_i_all = torch.zeros(c.n_layers, B, self.topk1, dtype=torch.int64, device=dev)
        self.gate_w_all[..., -1] = 1.0
        self.gate_i_all[..., -1] = c.n_routed_experts
        self.logits = z(B, c.vocab_size // T)
        self.next_tokens = torch.zeros(B, dtype=torch.int64, device=dev)
        self.tp_gather = (torch.empty(self.tp_size, B, 2, dtype=torch.float32, device=dev)
                          if (self.pg is not None and self.tp_size > 1) else None)
        lib = self.lib
        self.attn_ws = torch.zeros(lib.chitu_b200_attn_workspace_bytes(B, self.H, self.C, 128), dtype=torch.uint8, device=dev)
        self.lin_ws = torch.zeros(max(lib.chitu_b200_linear_workspace_bytes(B, max(c.vocab_size // T, dim)), 256),
                                  dtype=torch.uint8, device=dev)
        self.moe_ws = torch.zeros(lib.chitu_b200_moe_workspace_bytes(B, self.topk1, c.n_routed_experts + 1,
                                                                     2 * self.F_moe, dim), dtype=torch.uint8, device=dev)
        self.gate_ws = torch.zeros(lib.chitu_b200_moe_gate_workspace_bytes(B, c.n_routed_experts), dtype=torch.uint8, device=dev)
        self.max_seq_len = max_seq_len
        # the wgmma MLA kernel can leave its split-KV partials for the absorb-o kernel to merge (one launch fewer)
        import os
        self.defer_merge = (page_size == 64 and os.environ.get("CHITU_B200_MLA_IMPL", "0") == "0"
                            and os.environ.get("CHITU_B200_MLA_DEFER_MERGE", "1") != "0"
                            and c.v_head_dim == 128 and self.C == 512)
        self.ar_push = os.environ.get("CHITU_B200_AR_PUSH", "1") != "0"
        # optional: the gate kernel's last CTA writes the expert plan (chitu_b200_moe_gate_plan, one launch fewer); off by
        # default: the in-kernel hand-off (fence + ticket + a 256-thread plan) is serial work on the critical path where the
        # separate plan kernel only costs a PDL launch.
        self.gate_plan = os.environ.get("CHITU_B200_GATE_PLAN", "0") == "1" and B * self.topk1 <= 8192
        self.graph = None
        self.launches_per_step = 0
        self.trace = None          # set to [] to record per-layer intermediates (tests; not under CUDA graphs)
        self.capture_h = None      # set to [] to record the residual stream at every layer boundary of the FAST path
        # fused one-shot all-reduce + residual + RMSNorm(+quant) over NVLink peer memory; NCCL otherwise
        self.comm = None
        if tp_size > 1 and process_group is not None and use_fused_allreduce:
            from .comm import FusedAllReduce
            self.comm = FusedAllReduce(process_group, max_reqs, dim, self.device)

    # ---- helpers -----------------------------------------------------------------------------------
    def _dequant(self, w, s):
        y = torch.empty(w.shape, dtype=BF, device=self.device)
        check(self.lib.chitu_b200_weight_dequant_fp8(ptr(w), ptr(s), ptr(y), 1, w.shape[0], w.shape[1], 128, 0,
                                                     current_stream()), "weight_dequant")
        return y

    def _rms(self, x, w, y, rows, dim, xs=None, ys=None):
        check(self.lib.chitu_b200_rmsnorm_strided(ptr(x), ptr(w), ptr(y), rows, dim, xs or dim, ys or dim,
                                                  self.cfg.norm_eps, _lib.CB_BF16, current_stream()), "rmsnorm")

    def _rms_quant(self, x, w, dim, rows, xs=None, y=None):
        """RMSNorm fused with act_quant_deepseek_v3: fp8 payload -> self.xq / self.xs (and bf16 -> y)."""
        check(self.lib.chitu_b200_rmsnorm_quant_fp8(ptr(x), ptr(w), ptr(y), ptr(self.xq), ptr(self.xs), rows, dim,
                                                    xs or dim, dim, self.cfg.norm_eps, current_stream()), "rmsnorm_quant")

    def _fp8_gemm(self, w, w_s, y, M, residual=None):
        """fp8_gemm_deepseek_v3 on the already quantised activations in self.xq / self.xs."""
        N, K = w.shape
        check(self.lib.chitu_b200_fp8_gemm(ptr(self.xq), ptr(self.xs), ptr(w), ptr(w_s), ptr(y), M, N, K, ptr(residual),
                                           ptr(self.lin_ws), self.lin_ws.numel(), 0, current_stream()), "fp8_gemm")

    def _allreduce(self, t):
        if self.pg is not None and self.tp_size > 1:
            torch.distributed.all_reduce(t, group=self.pg)

    def _add(self, a, b, y):
        check(self.lib.chitu_b200_add(ptr(a), ptr(b), ptr(y), a.numel(), _lib.CB_BF16, current_stream()), "add")

    def set_synthetic_context(self, seq_len: int, seed: int = 2):
        g = torch.Generator(device="cpu").manual_seed(seed)
        gd = torch.Generator(device=self.device).manual_seed(seed + 11)     # deterministic cache contents
        nblk = self.kv_cache.shape[1]
        self.block_table.copy_(torch.randperm(nblk, generator=g).to(torch.int32).view(self.B, self.max_blocks))
        self.seq_lens.fill_(seq_len)
        for l in range(self.cfg.n_layers):
            self.kv_cache[l].normal_(0, 1, generator=gd)

    # ---- one decode step ---------------------------------------------------------------------------
    def _step_body(self):
        if self.trace is None:
            return self._step_body_fast()
        return self._step_body_traced()

    def _step_body_fast(self):
        """Production flow: every RMSNorm is fused either into the collective that precedes it (tensor parallel:
        all-reduce + residual + norm + quant in one kernel) or into a norm+quant kernel; residual adds ride in
        the GEMM / expert-combine epilogues.  Arithmetic is identical to `_step_body_traced`."""
        lib, B, c = self.lib, self.B, self.cfg
        st = current_stream()
        H, C, R, dn, dv = self.H, self.C, self.R, c.qk_nope_head_dim, c.v_head_dim
        tp_on = self.pg is not None and self.tp_size > 1
        torch.index_select(self.cos_table, 0, self.seq_lens, out=self.cos)
        torch.index_select(self.sin_table, 0, self.seq_lens, out=self.sin)
        check(lib.chitu_b200_embedding(ptr(self.tokens), ptr(self.embed), ptr(self.h), B, c.dim, 0, c.vocab_size,
                                       _lib.CB_BF16, st), "embedding")
        h, h2 = self.h, self.h2
        qa_w = c.q_lora_rank + C + R
        n_layers = len(self.layers)

        def reduce_add_norm(partial, residual, h_out, norm_w, want_y, want_q):
            """h_out = all_reduce(partial) + residual; then RMSNorm(h_out)*norm_w -> self.xn (bf16) and/or xq/xs (fp8)"""
            y = self.xn if want_y else None
            if self.comm is not None:
                self.comm(partial, residual, h_out, norm_w, y, self.xq if want_q else None, self.xs if want_q else None,
                          B, c.dim, c.norm_eps)
            else:
                self._allreduce(partial)
                self._add(partial, residual, h_out)
                check(lib.chitu_b200_rmsnorm_quant_fp8(ptr(h_out), ptr(norm_w), ptr(y), ptr(self.xq) if want_q else None,
                                                       ptr(self.xs) if want_q else None, B, c.dim, c.dim, c.dim,
                                                       c.norm_eps, st), "rmsnorm_quant")

        def consume(residual, h_out, norm_w, want_y, want_q):
            """push-mode reduce: h_out = sum over ranks of the pushed partials + residual, then the fused norm (+ quant)"""
            self.comm.consume(residual, h_out, norm_w, self.xn if want_y else None, self.xq if want_q else None,
                              self.xs if want_q else None, B, c.dim, c.norm_eps)
        push = tp_on and self.comm is not None and self.ar_push

        def norm_only(x, norm_w, want_y, want_q):
            check(lib.chitu_b200_rmsnorm_quant_fp8(ptr(x), ptr(norm_w), ptr(self.xn) if want_y else None,
                                                   ptr(self.xq) if want_q else None, ptr(self.xs) if want_q else None,
                                                   B, c.dim, c.dim, c.dim, c.norm_eps, st), "rmsnorm_quant")

        norm_only(h, self.layers[0]["attn_norm"], False, True)
        for li, L in enumerate(self.layers):
            if self.capture_h is not None:       # tests: the residual stream entering every layer (never under a graph)
                self.capture_h.append(h.clone())
            last = li + 1 == n_layers
            next_norm = self.norm if last else self.layers[li + 1]["attn_norm"]
            is_moe = li >= c.n_dense_layers
            # ---------------- attention ----------------
            self._fp8_gemm(L["wqkv_a"], L["wqkv_a_s"], self.qkv_a, B)
            self._rms_quant(self.qkv_a, L["q_norm"], c.q_lora_rank, B, xs=qa_w)
            self._fp8_gemm(L["wq_b"], L["wq_b_s"], self.q, B)
            if self.cache_dequant:
                wkv = L["wkv_b_bf16"]
            else:
                check(lib.chitu_b200_weight_dequant_fp8(ptr(L["wkv_b"]), ptr(L["wkv_b_s"]), ptr(self.wkv_tmp), 1,
                                                        self.wkv_tmp.shape[0], C, 128, 0, st), "wkv_b dequant")
                wkv = self.wkv_tmp
            check(lib.chitu_b200_mla_prep(ptr(self.q), ptr(self.qkv_a[:, c.q_lora_rank:]), qa_w, ptr(L["kv_norm"]),
                                          ptr(self.cos), ptr(self.sin), ptr(wkv), ptr(self.q_abs), ptr(self.q_pe),
                                          ptr(self.new_kv), B, H, dn, dv, C, R, c.norm_eps, st), "mla_prep")
            if self.defer_merge:
                # split-KV partials stay in the workspace; the LSE merge happens inside the absorb-o kernel
                check(lib.chitu_b200_mla_decode(ptr(self.q_abs), ptr(self.q_pe), ptr(self.kv_cache[li]), ptr(self.new_kv),
                                                ptr(self.seq_lens), ptr(self.block_table), self.max_blocks, B, H, C, R,
                                                self.page, self.kv_cache.shape[1], self.max_seq_len, float(c.softmax_scale),
                                                None, ptr(self.attn_ws), self.attn_ws.numel(), st), "mla_decode")
                check(lib.chitu_b200_mla_absorb_o_merge_quant(ptr(self.attn_ws), self.attn_ws.numel(), self.max_seq_len,
                                                              ptr(wkv), None, None, ptr(self.xq), ptr(self.xs), B, H, dn, dv,
                                                              C, st), "absorb_o_merge")
            else:
                check(lib.chitu_b200_mla_decode(ptr(self.q_abs), ptr(self.q_pe), ptr(self.kv_cache[li]), ptr(self.new_kv),
                                                ptr(self.seq_lens), ptr(self.block_table), self.max_blocks, B, H, C, R,
                                                self.page, self.kv_cache.shape[1], self.max_seq_len, float(c.softmax_scale),
                                                ptr(self.o_lat), ptr(self.attn_ws), self.attn_ws.numel(), st), "mla_decode")
                check(lib.chitu_b200_mla_absorb_o_quant(ptr(self.o_lat), ptr(wkv), None, ptr(self.xq), ptr(self.xs), B, H, dn,
                                                        dv, C, st), "absorb_o")
            # the ffn_norm output is needed in bf16 by the gate / expert gather (MoE) and in fp8 by the dense FFN
            if push:
                self.comm.fp8_gemm_push(self.xq, self.xs, L["wo"], L["wo_s"], B, self.lin_ws)
                consume(h, h2, L["ffn_norm"], is_moe, not is_moe)
            elif tp_on:
                self._fp8_gemm(L["wo"], L["wo_s"], h2, B)
                reduce_add_norm(h2, h, h2, L["ffn_norm"], want_y=is_moe, want_q=not is_moe)
            else:
                self._fp8_gemm(L["wo"], L["wo_s"], h2, B, residual=h)
                norm_only(h2, L["ffn_norm"], is_moe, not is_moe)
            # ---------------- FFN ----------------
            if not is_moe:
                self._fp8_gemm(L["w13"], L["w13_s"], self.ff, B)
                check(lib.chitu_b200_silu_mul_quant_fp8(ptr(self.ff), ptr(self.xq), ptr(self.xs), B, self.F_dense, st),
                      "silu_quant")
                if push:
                    self.comm.fp8_gemm_push(self.xq, self.xs, L["w2"], L["w2_s"], B, self.lin_ws)
                    consume(h2, h, next_norm, last, not last)
                elif tp_on:
                    self._fp8_gemm(L["w2"], L["w2_s"], self.y, B)
                    reduce_add_norm(self.y, h2, h, next_norm, want_y=last, want_q=not last)
                else:
                    self._fp8_gemm(L["w2"], L["w2_s"], h, B, residual=h2)
                    norm_only(h, next_norm, last, not last)
            else:
                E1 = c.n_routed_experts + 1
                planned = 1 if self.gate_plan else 0
                if planned:
                    # the gate's last CTA also writes the expert plan of the fused_experts call below (one launch fewer)
                    check(lib.chitu_b200_moe_gate_plan(ptr(self.xn), ptr(L["gate_w"]), ptr(L["gate_b"]), _lib.CB_F32, B, c.dim,
                                                       c.n_routed_experts, c.n_expert_groups, c.n_limited_groups,
                                                       c.n_activated_experts, 1 if c.score_func == "sigmoid" else 0,
                                                       float(c.route_scale), ptr(self.gate_w_all[li]), ptr(self.gate_i_all[li]),
                                                       self.topk1, ptr(self.gate_ws), self.gate_ws.numel(), E1, 2 * self.F_moe,
                                                       c.dim, ptr(self.moe_ws), self.moe_ws.numel(), st), "moe_gate_plan")
                else:
                    check(lib.chitu_b200_moe_gate(ptr(self.xn), ptr(L["gate_w"]), ptr(L["gate_b"]), _lib.CB_F32, B, c.dim,
                                                  c.n_routed_experts, c.n_expert_groups, c.n_limited_groups,
                                                  c.n_activated_experts, 1 if c.score_func == "sigmoid" else 0,
                                                  float(c.route_scale), ptr(self.gate_w_all[li]), ptr(self.gate_i_all[li]),
                                                  self.topk1, ptr(self.gate_ws), self.gate_ws.numel(), st), "moe_gate")
                if push:
                    self.comm.experts_push(self.xn, L["we1"], L["we2"], L["we1_s"], L["we2_s"], self.gate_w_all[li], _lib.CB_BF16,
                                               self.gate_i_all[li], _lib.CB_I64, B, self.topk1, E1,
                                               2 * self.F_moe, c.dim, 1, self.moe_ws, planned=planned)
                    consume(h2, h, next_norm, last, not last)
                else:
                    fe = lib.chitu_b200_fused_experts_planned if planned else lib.chitu_b200_fused_experts
                    check(fe(
                        ptr(self.xn), ptr(L["we1"]), ptr(L["we2"]), ptr(L["we1_s"]), ptr(L["we2_s"]), ptr(self.gate_w_all[li]),
                        _lib.CB_BF16, ptr(self.gate_i_all[li]), _lib.CB_I64, B, self.topk1, E1,
                        2 * self.F_moe, c.dim, 1, ptr(self.y if tp_on else h), None if tp_on else ptr(h2), ptr(self.moe_ws),
                        self.moe_ws.numel(), st), "fused_experts")
                    if tp_on:
                        reduce_add_norm(self.y, h2, h, next_norm, want_y=last, want_q=not last)
                    else:
                        norm_only(h, next_norm, last, not last)
        if self.capture_h is not None:
            self.capture_h.append(h.clone())
        N, K = self.head.shape
        check(lib.chitu_b200_linear_bf16(ptr(self.xn), ptr(self.head), None, None, ptr(self.logits), B, N, K,
                                         _lib.CB_BF16, ptr(self.lin_ws), self.lin_ws.numel(), 0, st), "head")
        check(lib.chitu_b200_argmax(ptr(self.logits), ptr(self.next_tokens), B, N, _lib.CB_BF16, st), "argmax")
        if self.pg is not None and self.tp_size > 1:
            # vocab-parallel head: the reference all-gathers the logits shards before sampling
            # (tensor_parallel.py:94-102); the same token from a (max, index) all-gather of B*8 bytes per rank
            self.next_tokens.copy_(global_argmax(self.logits, self.next_tokens, self.tp_rank, N, self.pg, self.tp_gather))
        self.seq_lens.add_(1)

    def _step_body_traced(self):
        lib, B, c = self.lib, self.B, self.cfg
        st = current_stream()
        H, C, R, dn, dv = self.H, self.C, self.R, c.qk_nope_head_dim, c.v_head_dim
        torch.index_select(self.cos_table, 0, self.seq_lens, out=self.cos)
        torch.index_select(self.sin_table, 0, self.seq_lens, out=self.sin)
        check(lib.chitu_b200_embedding(ptr(self.tokens), ptr(self.embed), ptr(self.h), B, c.dim, 0, c.vocab_size,
                                       _lib.CB_BF16, st), "embedding")
        # (embedding table replicated per rank here; the reference shards it by vocab + all_reduce)
        h, h2 = self.h, self.h2
        qa_w = c.q_lora_rank + C + R
        for li, L in enumerate(self.layers):
            tr = None
            if self.trace is not None:
                tr = {}
                self.trace.append(tr)
                tr["h_in"] = h.clone()
            # ---------------- attention (decode_forward_paged, :672-699) ----------------
            tp_on = self.pg is not None and self.tp_size > 1
            self._rms_quant(h, L["attn_norm"], c.dim, B, y=self.xn if tr is not None else None)
            if tr is not None: tr["xn_attn"] = self.xn.clone()
            self._fp8_gemm(L["wqkv_a"], L["wqkv_a_s"], self.qkv_a, B)
            if tr is not None: tr["qkv_a"] = self.qkv_a.clone()
            self._rms_quant(self.qkv_a, L["q_norm"], c.q_lora_rank, B, xs=qa_w, y=self.qa_n if tr is not None else None)
            if tr is not None: tr["qa_n"] = self.qa_n.clone()
            self._fp8_gemm(L["wq_b"], L["wq_b_s"], self.q, B)
            if tr is not None: tr["q"] = self.q.clone()
            if self.cache_dequant:
                wkv = L["wkv_b_bf16"]
            else:
                check(lib.chitu_b200_weight_dequant_fp8(ptr(L["wkv_b"]), ptr(L["wkv_b_s"]), ptr(self.wkv_tmp), 1,
                                                        self.wkv_tmp.shape[0], C, 128, 0, st), "wkv_b dequant")
                wkv = self.wkv_tmp
            # rotary(q_pe, k_pe) + kv_norm + cat + W_UK absorption in one launch
            check(lib.chitu_b200_mla_prep(ptr(self.q), ptr(self.qkv_a[:, c.q_lora_rank:]), qa_w, ptr(L["kv_norm"]),
                                          ptr(self.cos), ptr(self.sin), ptr(wkv), ptr(self.q_abs), ptr(self.q_pe),
                                          ptr(self.new_kv), B, H, dn, dv, C, R, c.norm_eps, st), "mla_prep")
            if tr is not None: tr["q_pe"] = self.q_pe.clone()
            if tr is not None: tr["q_abs"] = self.q_abs.clone()
            if tr is not None: tr["new_kv"] = self.new_kv.clone()
            if tr is not None: tr["cache_before"] = self.kv_cache[li].clone(); tr["lens"] = self.seq_lens.clone()
            check(lib.chitu_b200_mla_decode(ptr(self.q_abs), ptr(self.q_pe), ptr(self.kv_cache[li]), ptr(self.new_kv),
                                            ptr(self.seq_lens), ptr(self.block_table), self.max_blocks, B, H, C, R,
                                            self.page, self.kv_cache.shape[1], self.max_seq_len, float(c.softmax_scale), ptr(self.o_lat),
                                            ptr(self.attn_ws), self.attn_ws.numel(), st), "mla_decode")
            # absorb_o fused with the act_quant of the `wo` linear (one head = one 128-wide group)
            check(lib.chitu_b200_mla_absorb_o_quant(ptr(self.o_lat), ptr(wkv), ptr(self.o) if tr is not None else None,
                                                    ptr(self.xq), ptr(self.xs), B, H, dn, dv, C, st), "absorb_o")
            if tr is not None: tr["o_lat"] = self.o_lat.clone()
            if tr is not None: tr["o"] = self.o.clone()
            if tp_on or tr is not None:
                self._fp8_gemm(L["wo"], L["wo_s"], h2, B)
                if tr is not None: tr["attn_out"] = h2.clone()
                self._allreduce(h2)
                self._add(h2, h, h2)                                # x = x + attn(...)
            else:
                self._fp8_gemm(L["wo"], L["wo_s"], h2, B, residual=h)      # residual fused in the epilogue
            if tr is not None: tr["h_mid"] = h2.clone()
            # ---------------- FFN ----------------
            self._rms_quant(h2, L["ffn_norm"], c.dim, B, y=self.xn)         # bf16 copy feeds the gate / experts
            if tr is not None: tr["xn_ffn"] = self.xn.clone()
            if li < c.n_dense_layers:
                F = self.F_dense
                self._fp8_gemm(L["w13"], L["w13_s"], self.ff, B)
                if tr is not None:
                    check(lib.chitu_b200_silu_and_mul(ptr(self.ff), ptr(self.act), B, F, _lib.CB_BF16, st), "silu")
                    tr["ff"] = self.ff.clone(); tr["act"] = self.act.clone()
                check(lib.chitu_b200_silu_mul_quant_fp8(ptr(self.ff), ptr(self.xq), ptr(self.xs), B, F, st), "silu_quant")
                if tp_on or tr is not None:
                    self._fp8_gemm(L["w2"], L["w2_s"], self.y, B)
                    if tr is not None: tr["y"] = self.y.clone()
                    self._allreduce(self.y)
                    self._add(self.y, h2, h)                        # x = x + ffn(...)
                else:
                    self._fp8_gemm(L["w2"], L["w2_s"], h, B, residual=h2)
            else:
                F = self.F_moe
                check(lib.chitu_b200_moe_gate(ptr(self.xn), ptr(L["gate_w"]), ptr(L["gate_b"]), _lib.CB_F32, B, c.dim,
                                              c.n_routed_experts, c.n_expert_groups, c.n_limited_groups,
                                              c.n_activated_experts, 1 if c.score_func == "sigmoid" else 0,
                                              float(c.route_scale), ptr(self.gate_w_all[li]), ptr(self.gate_i_all[li]),
                                              self.topk1, ptr(self.gate_ws), self.gate_ws.numel(), st),
                      "moe_gate")
                # shared expert (model_deepseek_v3.py:936-949) + routed experts (fused_experts, :995-1009) in ONE
                # grouped fp8 GEMM pass: the shared expert is slot `topk` of every token with weight 1
                fuse_res = not (tp_on or tr is not None)
                check(lib.chitu_b200_fused_experts(
                    ptr(self.xn), ptr(L["we1"]), ptr(L["we2"]), ptr(L["we1_s"]), ptr(L["we2_s"]), ptr(self.gate_w_all[li]),
                    _lib.CB_BF16, ptr(self.gate_i_all[li]), _lib.CB_I64, B, self.topk1, c.n_routed_experts + 1,
                    2 * F, c.dim, 1, ptr(h if fuse_res else self.y), ptr(h2) if fuse_res else None, ptr(self.moe_ws),
                    self.moe_ws.numel(), st), "fused_experts")
                if not fuse_res:
                    if tr is not None: tr["y"] = self.y.clone()
                    self._allreduce(self.y)
                    self._add(self.y, h2, h)                        # x = x + ffn(...)
            if tr is not None: tr["h_out"] = h.clone()
        self._rms(h, self.norm, self.xn, B, c.dim)
        N, K = self.head.shape
        check(lib.chitu_b200_linear_bf16(ptr(self.xn), ptr(self.head), None, None, ptr(self.logits), B, N, K,
                                         _lib.CB_BF16, ptr(self.lin_ws), self.lin_ws.numel(), 0, st), "head")
        check(lib.chitu_b200_argmax(ptr(self.logits), ptr(self.next_tokens), B, N, _lib.CB_BF16, st), "argmax")
        if self.pg is not None and self.tp_size > 1:
            # vocab-parallel head: the reference all-gathers the logits shards before sampling
            # (tensor_parallel.py:94-102); the same token from a (max, index) all-gather of B*8 bytes per rank
            self.next_tokens.copy_(global_argmax(self.logits, self.next_tokens, self.tp_rank, N, self.pg, self.tp_gather))
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
        """Mean number of distinct routed experts per MoE layer in the last step."""
        c = self.cfg
        ids = self.gate_i_all[c.n_dense_layers:, :, : c.n_activated_experts].cpu()
        if ids.numel() == 0:
            return 0.0
        return float(sum(len(torch.unique(ids[l])) for l in range(ids.shape[0])) / ids.shape[0])

    # ---- algorithmic bytes of one step on this rank (SURVEY §8d formula) ---------------------------
    def algorithmic_bytes(self, seq_len: int, distinct_experts_per_layer: Optional[float] = None) -> int:
        c = self.cfg

        def fp8_bytes(n, k):
            return n * k + ((n + 127) // 128) * ((k + 127) // 128) * 4

        attn = (fp8_bytes(c.q_lora_rank + self.C + self.R, c.dim) + fp8_bytes(self.H * self.qk_head, c.q_lora_rank)
                + fp8_bytes(self.H * (c.qk_nope_head_dim + c.v_head_dim), self.C) + fp8_bytes(c.dim, self.H * c.v_head_dim))
        dense = fp8_bytes(2 * self.F_dense, c.dim) + fp8_bytes(c.dim, self.F_dense)
        expert = fp8_bytes(2 * self.F_moe, c.dim) + fp8_bytes(c.dim, self.F_moe)
        if distinct_experts_per_layer is None:
            distinct_experts_per_layer = c.n_routed_experts * (1 - (1 - c.n_activated_experts / c.n_routed_experts) ** self.B)
        moe = c.n_routed_experts * c.dim * 2 + (c.n_shared_experts + distinct_experts_per_layer) * expert
        kv = self.B * (seq_len + 1) * (self.C + self.R) * 2
        n_moe = max(c.n_layers - c.n_dense_layers, 0)
        n_dense = min(c.n_layers, c.n_dense_layers)
        head = self.head.numel() * 2
        return int(c.n_layers * (attn + kv) + n_dense * dense + n_moe * moe + head)
