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

from ._lib import check, current_stream, ptr
from .attn_backend import mla_paged_attention
from .engine import DecodeEngine

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


class DeepSeekDecodeEngine(DecodeEngine):
    def __init__(self, cfg: DeepSeekConfig, max_reqs: int, max_seq_len: int, device="cuda:0", seed: int = 0,
                 tp_rank: int = 0, tp_size: int = 8, process_group=None, page_size: int = 64,
                 use_fused_allreduce: bool = True, kv_dtype: torch.dtype = BF):
        """kv_dtype=torch.float8_e4m3fn keeps the latent cache in e4m3 (half the cache bytes, twice the tokens per
        pool; new rows rounded to nearest even after a clamp to +-448, no scale) and attends through
        chitu_b200_mla_attn_fp8kv."""
        c = cfg
        if kv_dtype not in (BF, F8):
            raise ValueError(f"kv_dtype must be torch.bfloat16 or torch.float8_e4m3fn, not {kv_dtype}")
        T = tp_size
        assert c.n_heads % T == 0
        # the MLA kernels stage 64-token pages of a 512 + 64 wide latent; absorb-o quantises one 128-wide head per
        # act_quant group
        assert page_size == 64 and c.kv_lora_rank == 512 and c.qk_rope_head_dim == 64 and c.v_head_dim == 128, \
            "the MLA decode kernels are built for page 64, kv_lora_rank 512, qk_rope_head_dim 64, v_head_dim 128"
        self.H = c.n_heads // T
        self.qk_head = c.qk_nope_head_dim + c.qk_rope_head_dim
        self.C, self.R = c.kv_lora_rank, c.qk_rope_head_dim
        self.F_dense = c.inter_dim // T
        self.F_moe = c.moe_inter_dim // T
        super().__init__(cfg, max_reqs, max_seq_len, device, page_size, seed, tp_rank, tp_size, process_group,
                         use_fused_allreduce, attn_ws=(self.H, self.C, 128), lin_n=max(c.vocab_size // T, c.dim))
        dev, g, g_rep, rnd = self.device, self.g, self.g_rep, self._rnd

        def fp8(gen, *shape):
            # quantise in slabs to bound the fp32 temporaries for the [E, N, K] expert tensors
            if len(shape) == 3:
                qs, ss = [], []
                for e0 in range(0, shape[0], 32):
                    q, s = quantize_fp8_block(rnd(gen, min(32, shape[0] - e0), *shape[1:], dtype=torch.float32))
                    qs.append(q), ss.append(s)
                return torch.cat(qs), torch.cat(ss)
            return quantize_fp8_block(rnd(gen, *shape, dtype=torch.float32))

        dim = c.dim
        self.embed = rnd(g_rep, c.vocab_size, dim)
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
                L["gate_w"] = rnd(g_rep, c.n_routed_experts, dim)
                L["gate_b"] = rnd(g_rep, c.n_routed_experts, scale=0.01, dtype=torch.float32)      # fp32 bias
                # routed experts + the shared expert stored as expert index n_routed_experts, exactly like the
                # reference's stacked w1w3 / w2 tensors (model_deepseek_v3.py:1167-1191: `weight[-1]` is shared)
                assert c.n_shared_experts == 1
                L["we1"], L["we1_s"] = fp8(g, c.n_routed_experts + 1, 2 * self.F_moe, dim)
                L["we2"], L["we2_s"] = fp8(g, c.n_routed_experts + 1, dim, self.F_moe)
                L["ws13"], L["ws13_s"] = L["we1"][-1], L["we1_s"][-1]      # views (used by the tests)
                L["ws2"], L["ws2_s"] = L["we2"][-1], L["we2_s"][-1]
            # SURVEY §8f n1: dequantise wkv_b once instead of every step (model_deepseek_v3.py:516-528)
            L["wkv_b_bf16"] = self._dequant(L["wkv_b"], L["wkv_b_s"])
            self.layers.append(L)
        self.norm = torch.ones(dim, dtype=BF, device=dev)
        self.head = rnd(g, c.vocab_size // T, dim)
        # paged MLA cache: [L, num_blocks, 64, 576], replicated on every rank (cache_manager.py:71-76)
        nblk = self.max_blocks * max_reqs
        self.kv_cache = torch.zeros(c.n_layers, nblk, page_size, self.C + self.R, dtype=kv_dtype, device=dev)
        self.caches = (self.kv_cache,)
        self._rope_tables(yarn_freqs(c, max_seq_len * 2))
        B = max_reqs
        z = lambda *s, dt=BF: torch.zeros(*s, dtype=dt, device=dev)
        kmax = max(dim, self.F_dense, self.H * c.v_head_dim, c.q_lora_rank)
        self.xq = torch.zeros(B, kmax, dtype=F8, device=dev)
        self.xs = z(B, kmax // 128 + 1, dt=torch.float32)
        self.qkv_a = z(B, c.q_lora_rank + self.C + self.R)
        self.q = z(B, self.H, self.qk_head)
        self.q_pe = z(B, self.H, self.R)
        self.q_abs = z(B, self.H, self.C)
        self.new_kv = z(B, self.C + self.R)
        self.ff = z(B, 2 * max(self.F_dense, self.F_moe))
        # the routed experts of the MoE layers (fp8 block-scaled w8a8, wmode 1), plus one slot per token for the shared
        # expert (id n_routed_experts, weight 1): it rides through the grouped expert GEMM instead of five separate
        # launches
        E = c.n_routed_experts
        self._init_moe(n_routed=E, topk=c.n_activated_experts, slots=c.n_activated_experts + 1, n_stacked=E + 1,
                       n1=2 * self.F_moe, score_mode=1 if c.score_func == "sigmoid" else 0, route_scale=c.route_scale,
                       groups=(c.n_expert_groups, c.n_limited_groups), bias=True, first_layer=c.n_dense_layers,
                       weights=("we1", "we2", "we1_s", "we2_s"), wmode=1)
        self.gate_w_all[..., -1] = 1.0
        self.gate_i_all[..., -1] = E

    # ---- helpers -----------------------------------------------------------------------------------
    def _dequant(self, w, s):
        y = torch.empty(w.shape, dtype=BF, device=self.device)
        check(self.lib.chitu_b200_weight_dequant_fp8(ptr(w), ptr(s), ptr(y), 1, w.shape[0], w.shape[1], 128, 0,
                                                     current_stream()), "weight_dequant")
        return y

    def _norm(self, x, w, y=None, q=None, qs=None, rows=None):
        """RMSNorm of the residual stream into bf16 `y` and / or the fp8 activations `q` + scales `qs` (`rows`
        rows, default B)."""
        c = self.cfg
        M = self.B if rows is None else rows
        check(self.lib.chitu_b200_rmsnorm_quant_fp8(ptr(x), ptr(w), ptr(y), ptr(q), ptr(qs), M, c.dim, c.dim, c.dim,
                                                    c.norm_eps, current_stream()), "rmsnorm_quant")

    def _norm_out(self, bf16: bool):
        """The norm outputs the next consumer reads: bf16 for the MoE gate / experts and the head, fp8 for a GEMM."""
        return dict(y=self.xn) if bf16 else dict(q=self.xq, qs=self.xs)

    def _fp8_gemm(self, w, w_s, y, M, residual=None):
        """fp8_gemm_deepseek_v3 on the already quantised activations in self.xq / self.xs."""
        N, K = w.shape
        check(self.lib.chitu_b200_fp8_gemm(ptr(self.xq), ptr(self.xs), ptr(w), ptr(w_s), ptr(y), M, N, K, ptr(residual),
                                           ptr(self.lin_ws), self.lin_ws.numel(), 0, current_stream()), "fp8_gemm")

    def _mla_prep(self, li):
        """rotary(q_pe, k_pe) + kv_norm + cat + W_UK absorption in one launch"""
        c, L = self.cfg, self.layers[li]
        check(self.lib.chitu_b200_mla_prep(ptr(self.q), ptr(self.qkv_a[:, c.q_lora_rank:]), c.q_lora_rank + self.C + self.R,
                                           ptr(L["kv_norm"]), ptr(self.cos), ptr(self.sin), ptr(L["wkv_b_bf16"]),
                                           ptr(self.q_abs), ptr(self.q_pe), ptr(self.new_kv), self.B, self.H,
                                           c.qk_nope_head_dim, c.v_head_dim, self.C, self.R, c.norm_eps, current_stream()),
              "mla_prep")

    def _mla_decode(self, li):
        """paged absorbed-MLA decode, appending new_kv; the split-KV partials stay in the workspace"""
        mla_paged_attention(self.q_abs, self.q_pe, self.kv_cache[li], self.new_kv, self.seq_lens, self.block_table,
                            self.max_seq_len, True, self.cfg.softmax_scale, None, self.attn_ws)

    # ---- one decode step ---------------------------------------------------------------------------
    def _decode_layers(self):
        """Every RMSNorm is fused either into the collective that precedes it (tensor parallel: all-reduce + residual +
        norm + quant in one kernel) or into a norm+quant kernel; residual adds ride in the GEMM / expert-combine
        epilogues."""
        lib, B, c = self.lib, self.B, self.cfg
        st = current_stream()
        h, h2 = self.h, self.h2
        n_layers = len(self.layers)
        self._norm(h, self.layers[0]["attn_norm"], **self._norm_out(False))
        for li, L in enumerate(self.layers):
            if self.capture_h is not None:
                self.capture_h.append(h.clone())
            last = li + 1 == n_layers
            next_norm = self.norm if last else self.layers[li + 1]["attn_norm"]
            is_moe = li >= c.n_dense_layers
            # ---------------- attention ----------------
            self._fp8_gemm(L["wqkv_a"], L["wqkv_a_s"], self.qkv_a, B)
            # q_norm fused with the act_quant of wq_b's input
            check(lib.chitu_b200_rmsnorm_quant_fp8(ptr(self.qkv_a), ptr(L["q_norm"]), None, ptr(self.xq), ptr(self.xs), B,
                                                   c.q_lora_rank, c.q_lora_rank + self.C + self.R, c.q_lora_rank,
                                                   c.norm_eps, st), "rmsnorm_quant")
            self._fp8_gemm(L["wq_b"], L["wq_b_s"], self.q, B)
            self._mla_prep(li)
            # split-KV partials stay in the workspace; the LSE merge happens inside the absorb-o kernel
            self._mla_decode(li)
            check(lib.chitu_b200_mla_absorb_o_merge_quant(ptr(self.attn_ws), self.attn_ws.numel(), self.max_seq_len,
                                                          ptr(L["wkv_b_bf16"]), None, None, ptr(self.xq), ptr(self.xs),
                                                          B, self.H, c.qk_nope_head_dim, c.v_head_dim, self.C, st),
                  "absorb_o_merge")
            # the ffn_norm output is needed in bf16 by the gate / expert gather (MoE) and in fp8 by the dense FFN
            self._row_parallel(lambda out, res: self._fp8_gemm(L["wo"], L["wo_s"], out, B, residual=res),
                               lambda: self.comm.fp8_gemm_push(self.xq, self.xs, L["wo"], L["wo_s"], B, self.lin_ws),
                               h, h2, L["ffn_norm"], **self._norm_out(is_moe))
            # ---------------- FFN ----------------
            if not is_moe:
                self._fp8_gemm(L["w13"], L["w13_s"], self.ff, B)
                check(lib.chitu_b200_silu_mul_quant_fp8(ptr(self.ff), ptr(self.xq), ptr(self.xs), B, self.F_dense, st),
                      "silu_quant")
                self._row_parallel(lambda out, res: self._fp8_gemm(L["w2"], L["w2_s"], out, B, residual=res),
                                   lambda: self.comm.fp8_gemm_push(self.xq, self.xs, L["w2"], L["w2_s"], B, self.lin_ws),
                                   h2, h, next_norm, partial=self.y, **self._norm_out(last))
            else:
                # shared expert (model_deepseek_v3.py:936-949) + routed experts (fused_experts, :995-1009) in ONE
                # grouped fp8 GEMM pass: the shared expert is slot `topk` of every token with weight 1
                self._moe_block(li, h2, h, next_norm, **self._norm_out(last))
        if self.capture_h is not None:
            self.capture_h.append(h.clone())

    # ---- algorithmic bytes of one step on this rank (SURVEY §8d formula) ---------------------------
    def algorithmic_bytes(self, seq_len: int, distinct_experts_per_layer: Optional[float] = None) -> int:
        """Every attention and dense-FFN weight byte once, the router, the shared expert and each DISTINCT routed
        expert once, KV rows once, the bf16 head.  The weights count the bytes of the tensors the engine holds: fp8
        weights with their block scales (wkv_b, not its dequantised copy), the bf16 router without its bias."""
        c = self.cfg
        n_dense = min(c.n_layers, c.n_dense_layers)
        n_moe = c.n_layers - n_dense

        def nbytes(li, *names):
            return sum(self.layers[li][n].nbytes for n in names)

        attn = nbytes(0, "wqkv_a", "wqkv_a_s", "wq_b", "wq_b_s", "wkv_b", "wkv_b_s", "wo", "wo_s")
        dense = nbytes(0, "w13", "w13_s", "w2", "w2_s") if n_dense else 0
        moe = 0
        if n_moe:
            if distinct_experts_per_layer is None:
                distinct_experts_per_layer = c.n_routed_experts * (1 - (1 - c.n_activated_experts / c.n_routed_experts)
                                                                   ** self.B)
            expert = nbytes(-1, "we1", "we1_s", "we2", "we2_s") // (c.n_routed_experts + 1)
            moe = nbytes(-1, "gate_w") + (c.n_shared_experts + distinct_experts_per_layer) * expert
        kv = self.B * (seq_len + 1) * (self.C + self.R) * self.kv_cache.element_size()
        return int(c.n_layers * (attn + kv) + n_dense * dense + n_moe * moe + self.head.nbytes)
