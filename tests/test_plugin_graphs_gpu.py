"""The plugin surface driven the way the reference drives it after `plugin.install()`: one CUDA graph per decode batch
size, captured in the order the batch sizes arrive (models/model.py:537-622) and then replayed interleaved, with
`prepare_metadata_for_decode` outside the graph (models/model.py:540), over the persistent workspaces of
chitu_b200/workspace.py.  Nothing here goes through the decode engines, which own their workspaces.

Three stand-in decode steps use only `ops`, `fused_moe`, `B200AttnBackend` and the quantised linear modules:
  * LLaMA-shaped: two layers of rms_norm, linear, the interleaved rotary, attn_with_kvcache over paged bf16 caches
    (layer 0) and e4m3 caches (layer 1) (page 256, D 128, Hq 4, Hkv 1) and silu_and_mul, then one MLP block each
    through W4A16Linear, Fp8Linear and W8A8Linear;
  * Mixtral-shaped: moe_gate("softmax_renorm") and bf16 fused_experts (8 experts, top 2);
  * DeepSeek-shaped: linear_deepseek_v3 (fp8 and soft fp8), mla_attn_with_kvcache (page 64, C 512, R 64, 16 local
    heads), the sigmoid grouped gate (256 experts, 8 groups, top 4 groups, top 8) and fp8 fused_experts at the tp8
    shard shape (E 257 with the shared expert, N1 512, K 7168).

The guarantees pinned:
  1. after the workspaces are reserved, capturing at B = 3, 1, 16, 8, 32 (one eager step at 3 only) moves no buffer and
     retires none;
  2. over 12 interleaved replays, whose lengths advance across page boundaries, every replay equals an eager run of the
     same body on a cloned state bit for bit (outputs and every cache byte) and every block stays within the fp64 bound
     of tests/test_engine_steps_gpu.py (teacher-forced from the replay's own block inputs);
  3. an eager call that outgrows a tag the graphs hold moves it and retires the old buffer; with tensors of the retired
     sizes allocated and filled with 0xFF, every graph replays exactly as before;
  4. a capture that would grow a tag raises, naming the tag, and leaves the buffer where it was;
  5. the split plan in the tail of "attn" survives a GQA call at the largest split count, equals the host model of
     attn_plan_kernel, and an MLA replay at another batch size refuses it and stays within the bound;
  6. fused_experts never asks for the unreserved "moe_gg" workspace, whose first use inside a capture raises.

Measured on one H100 80GB HBM3 at a 700 W power limit: the module runs in about 8 s (16 s with the interpreter start)
and reserves at most 3.5 GB of device memory; the worst err / bound of any block over the replays is 0.41."""
import gc

import pytest
import torch

import torch_ref as R
from test_attn_decode_dispatch_gpu import attn_plan, gqa_splits, plan_honoured, mla_num_splits
from test_engine_steps_gpu import FLOOR_SEEDS, bound, check_append, kept_rows, rel_err, ulp_perturb

BF, F16, F8, F64 = torch.bfloat16, torch.float16, torch.float8_e4m3fn, torch.float64
DEV = "cuda:0"
MAX_REQS = 32
ORDER = (3, 1, 16, 8, 32)                                   # arrival order of the decode batch sizes
SCHEDULE = (8, 32, 1, 16, 3, 32, 8, 1, 16, 3, 32, 16)       # the interleaved replays
EPS = 1e-6


def fresh_workspaces():
    """No graph of an earlier test is alive here: start from no buffer at all."""
    gc.collect()
    torch.cuda.synchronize()
    from chitu_b200 import workspace
    workspace.clear()
    torch.cuda.empty_cache()


def tag_state():
    from chitu_b200 import workspace
    return {tag: (buf.data_ptr(), buf.numel()) for (tag, _), buf in workspace._ws.items()}


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8),
                                                                     b.contiguous().view(torch.uint8))


def rand(shape, gen, scale=1.0, dtype=BF):
    return (torch.randn(shape, generator=gen, device=DEV) * scale).to(dtype)


def norm_weight(n, gen):
    return (0.5 + torch.rand(n, generator=gen, device=DEV)).to(BF)


def increment_check(ref_fn, h_in, h_out, gen, what):
    """err of the block increment h_out - h_in against the fp64 reference from h_in, and its bound (floor: the reference
    against itself with h_in moved by one bf16 ulp)."""
    ref = ref_fn(h_in)
    d_ref = ref.double() - h_in.double()
    err = rel_err(h_out.double() - h_in.double(), d_ref)
    floor = 0.0
    for _ in range(FLOOR_SEEDS):
        hp = ulp_perturb(h_in, gen)
        floor = max(floor, rel_err(ref_fn(hp).double() - hp.double(), d_ref))
    return err, bound(floor), (f"{what}: err {err:.3e} > bound {bound(floor):.3e}" if err > bound(floor) else None)


def paged_lens(page):
    """Start lengths of the MAX_REQS requests: at, just before and just after page boundaries, and some long ones."""
    base = (page - 6, 1, page - 3, 2 * page - 4, 0, 3 * page - 8, 2 * page - 1, page - 12)
    return torch.tensor([base[b % 8] + b // 8 for b in range(MAX_REQS)], dtype=torch.int32, device=DEV)


# ---------------------------------------------------------------------------------------------------- stand-ins
class Llama:
    """Two LLaMA decode layers (bf16 and e4m3 KV caches) and one MLP block per quantised linear module."""
    dim, Hq, Hkv, D, F, page, pages = 512, 4, 1, 128, 1024, 256, 4
    reserve_shapes = dict(heads=4, head_dim_v=128)              # the stand-in's attention: GQA rows of 128

    def __init__(self):
        from chitu_b200.attn_backend import B200AttnBackend
        from chitu_b200.quantize.fp8 import Fp8Linear
        from chitu_b200.quantize.w4a16 import W4A16Linear
        from chitu_b200.quantize.w8a8 import W8A8Linear
        g = torch.Generator(device=DEV).manual_seed(1)
        d, D, F = self.dim, self.D, self.F
        self.layers = [dict(attn_norm=norm_weight(d, g), ffn_norm=norm_weight(d, g),
                            wqkv=rand(((self.Hq + 2 * self.Hkv) * D, d), g, d ** -0.5),
                            wo=rand((d, self.Hq * D), g, (self.Hq * D) ** -0.5),
                            w13=rand((2 * F, d), g, d ** -0.5), w2=rand((d, F), g, F ** -0.5)) for _ in range(2)]
        nb = MAX_REQS * self.pages
        shape = (nb, self.page, self.Hkv, D)
        self.caches = [rand(shape, g), rand(shape, g), rand(shape, g, 2.0).float().clamp(-448, 448).to(F8),
                       rand(shape, g, 2.0).float().clamp(-448, 448).to(F8)]
        self.bt = torch.randperm(nb, generator=torch.Generator().manual_seed(2)).view(MAX_REQS, self.pages).int().to(DEV)
        self.lens = paged_lens(self.page)
        inv = 1.0 / (500000.0 ** (torch.arange(0, D, 2, dtype=F64) / D))
        ang = torch.outer(torch.arange(self.page * self.pages, dtype=F64), inv)
        self.cos_t, self.sin_t = ang.cos().float().to(DEV), ang.sin().float().to(DEV)
        self.be = B200AttnBackend(max_reqs=MAX_REQS, n_local_heads=self.Hq)
        self.quant = []
        for cls in (W4A16Linear, Fp8Linear, W8A8Linear):
            lin = [torch.nn.Linear(k, n, bias=False, device=DEV) for n, k in ((2 * F, d), (d, F))]
            for m in lin:
                torch.nn.init.normal_(m.weight, std=m.in_features ** -0.5, generator=g)
            self.quant.append((cls.from_float(lin[0]), cls.from_float(lin[1]), norm_weight(d, g)))
        self.h = {B: torch.empty(B, d, dtype=BF, device=DEV) for B in ORDER}

    def new_inputs(self, B, seed):
        self.h[B].copy_(rand((B, self.dim), torch.Generator(device=DEV).manual_seed(seed)))

    def prepare(self, B):
        pass

    def advance(self, B):
        self.lens[:B] += 1

    def layer(self, li, h, lens, bt, kc, vc):
        from chitu_b200 import ops
        L, B, Hq, Hkv, D = self.layers[li], h.shape[0], self.Hq, self.Hkv, self.D
        qkv = ops.linear(ops.rms_norm(h, L["attn_norm"], EPS), L["wqkv"])
        q = qkv[:, : Hq * D].reshape(B, Hq, D)
        k = qkv[:, Hq * D: (Hq + Hkv) * D].reshape(B, Hkv, D)
        v = qkv[:, (Hq + Hkv) * D:].reshape(B, 1, Hkv, D)
        pos = lens.long()
        q, k = ops.apply_rotary_pos_emb(q, k, self.cos_t[pos], self.sin_t[pos], rotary_type="llama")
        o = self.be.attn_with_kvcache(q.view(B, 1, Hq, D), kc, vc, k.view(B, 1, Hkv, D), v, cache_seqlens=lens,
                                      block_table=bt)
        h = h + ops.linear(o.reshape(B, Hq * D), L["wo"])
        gu = ops.linear(ops.rms_norm(h, L["ffn_norm"], EPS), L["w13"])
        return h + ops.linear(ops.silu_and_mul(gu), L["w2"])

    def body(self, B, caches):
        from chitu_b200 import ops
        h, lens, bt = self.h[B], self.lens[:B], self.bt[:B]
        hs = [h]
        for li in range(2):
            h = self.layer(li, h, lens, bt, caches[2 * li], caches[2 * li + 1])
            hs.append(h)
        for up, down, w in self.quant:
            h = h + down(ops.silu_and_mul(up(ops.rms_norm(h, w, EPS)))).to(BF)
            hs.append(h)
        return hs

    @staticmethod
    def qlin_ref(m, x):
        """The quantised module's arithmetic in fp64 (activation quantisation in fp32, as the kernels do it)."""
        from chitu_b200.quantize.fp8 import Fp8Linear, MIN_SCALE
        from chitu_b200.quantize.w4a16 import W4A16Linear
        if isinstance(m, W4A16Linear):
            return (x.double() @ m.dequantized_weight().double().T).to(m.dtype)
        xf = x.float()
        if isinstance(m, Fp8Linear):
            s = (xf.abs().amax(dim=-1) / 448.0).clamp(min=MIN_SCALE)
            q = (xf * (1.0 / s)[:, None]).clamp(-448, 448).to(F8)
            y = (q.double() @ m.weight.double().T) * s.double()[:, None] * m.weight_scale.double()
            return y.to(BF)
        s = xf.abs().amax(dim=-1).clamp(min=1e-5) / 127.0                       # W8A8Linear
        q = torch.round(xf / s[:, None])
        return ((q.double() @ m.weight.double().T) * s.double()[:, None] * m.scale_channel.double()).to(F16)

    def check(self, B, out, before, after, gen):
        lens, bt = self.lens[:B], self.bt[:B]
        pos = lens.long()
        fails, worst, kv = [], 0.0, 0.0
        for li in range(2):
            lw = self.layers[li]
            pair = before[2 * li: 2 * li + 2]

            def ref(h, keep=None):
                caches = [c.clone() for c in pair]
                y = R.llama_layer(lw, h, caches[0], caches[1], lens, bt, self.cos_t[pos], self.sin_t[pos], self.Hq,
                                  self.Hkv, EPS, compute_dtype=F64)
                if keep is not None:
                    keep.extend(caches)
                return y
            err, bnd, f = increment_check(ref, out[li], out[li + 1], gen, f"layer {li}")
            worst, fails = max(worst, err / bnd), fails + [f] * (f is not None)
            ref_caches = []
            ref(out[li], ref_caches)
            for a, b4, r in zip(after[2 * li: 2 * li + 2], pair, ref_caches):
                kv = max(kv, check_append(a, b4, r, bt, lens, self.page))
        for i, (up, down, w) in enumerate(self.quant):
            def ref(h):
                u = self.qlin_ref(up, R.rms_norm(h, w, EPS, F64))
                return h + self.qlin_ref(down, R.silu_and_mul(u.double()).to(u.dtype)).to(BF)
            err, bnd, f = increment_check(ref, out[2 + i], out[3 + i], gen, type(up).__name__)
            worst, fails = max(worst, err / bnd), fails + [f] * (f is not None)
        if kv > 1.0:
            fails.append(f"an appended KV value is {kv:.2f} roundings from the reference's")
        return worst, fails

    def grow(self):
        """GQA attention at twice the reserved batch: "attn" outgrows its reservation."""
        B = 2 * MAX_REQS
        g = torch.Generator(device=DEV).manual_seed(7)
        q = rand((B, 1, self.Hq, self.D), g)
        kc, vc = (rand((B, self.page, self.Hkv, self.D), g) for _ in range(2))
        bt = torch.arange(B, dtype=torch.int32, device=DEV).view(B, 1)
        lens = torch.full((B,), 100, dtype=torch.int32, device=DEV)
        self.be.attn_with_kvcache(q, kc, vc, cache_seqlens=lens, block_table=bt)
        return ("attn",)


class Mixtral:
    """One Mixtral sparse-MoE block: the softmax top-2 gate with renormalisation and bf16 fused experts."""
    dim, E, topk, F = 512, 8, 2, 512
    reserve_shapes = None                                        # plugin.install(max_reqs) covers it

    def __init__(self):
        g = torch.Generator(device=DEV).manual_seed(21)
        d, F = self.dim, self.F
        self.norm = norm_weight(d, g)
        self.gate_w = rand((self.E, d), g, d ** -0.5)
        self.w1 = rand((self.E, 2 * F, d), g, d ** -0.5)
        self.w2 = rand((self.E, d, F), g, F ** -0.5)
        self.caches = []
        self.h = {B: torch.empty(B, d, dtype=BF, device=DEV) for B in ORDER}

    new_inputs, prepare = Llama.new_inputs, Llama.prepare

    def advance(self, B):
        pass

    def moe(self, x):
        from chitu_b200 import fused_moe, ops
        xn = ops.rms_norm(x, self.norm, EPS)
        w, idx = fused_moe.moe_gate(xn, self.gate_w, None, self.topk, 1, 1, "softmax_renorm", 1.0)
        return x + fused_moe.fused_experts(xn, self.w1, self.w2, w, idx), idx

    def body(self, B, caches):
        y, idx = self.moe(self.h[B])
        return [self.h[B], y, idx]

    def check(self, B, out, before, after, gen):
        h, y, idx = out
        xn = R.rms_norm(h, self.norm, EPS, F64)
        probs = torch.softmax(xn.double() @ self.gate_w.double().T, dim=-1)
        kept_rows(idx, [(probs.topk(self.topk, dim=-1)[1], probs)], self.topk)

        def ref(hh):
            x = R.rms_norm(hh, self.norm, EPS, F64)
            p = torch.softmax(x.double() @ self.gate_w.double().T, dim=-1).gather(1, idx)
            return hh + R.fused_experts(x, self.w1, self.w2, p / p.sum(dim=-1, keepdim=True), idx, compute_dtype=F64)
        err, bnd, f = increment_check(ref, h, y, gen, "moe")
        return err / bnd, [f] * (f is not None)

    def grow(self):
        """The gate and the experts over 2048 tokens: "moe_gate" and "moe" outgrow their reservations."""
        self.moe(rand((2048, self.dim), torch.Generator(device=DEV).manual_seed(8)))
        return ("moe_gate", "moe")


class DeepSeek:
    """One DeepSeek-V3 layer at the tp8 shard: fp8 / soft-fp8 linears, absorbed MLA over the paged latent cache, the
    sigmoid grouped gate and fp8 fused experts with the shared expert as expert 256."""
    dim, H, C, Rr, page, pages = 7168, 16, 512, 64, 64, 8
    E, topk, groups, topk_groups, N1, route_scale = 256, 8, 8, 4, 512, 2.5
    scale = 192 ** -0.5
    reserve_shapes = None

    def __init__(self):
        from chitu_b200.attn_backend import B200AttnBackend
        g = torch.Generator(device=DEV).manual_seed(31)
        d, H, C, Rr = self.dim, self.H, self.C, self.Rr
        self.n1, self.n2 = norm_weight(d, g), norm_weight(d, g)
        self.wq = self.fp8_weight((H * (C + Rr), d), g)
        self.wkv = self.fp8_weight((640, d), g)                 # C + R = 576 columns used, N padded to whole blocks
        self.wo = self.fp8_weight((d, H * C), g)
        self.wq_d, self.wo_d = self.deq(*self.wq), self.deq(*self.wo)
        self.wkv_bf = R.weight_dequant(*self.wkv)
        self.gate_w = rand((self.E, d), g, d ** -0.5)
        self.gate_b = (torch.randn(self.E, generator=g, device=DEV) * 0.05).float()
        Ne = self.E + 1
        self.w1 = torch.empty(Ne, self.N1, d, dtype=F8, device=DEV)
        self.w2 = torch.empty(Ne, d, self.N1 // 2, dtype=F8, device=DEV)
        for e in range(Ne):
            self.w1[e] = torch.randn(self.N1, d, generator=g, device=DEV).to(F8)
            self.w2[e] = torch.randn(d, self.N1 // 2, generator=g, device=DEV).to(F8)
        self.w1s = (0.5 + torch.rand(Ne, self.N1 // 128, d // 128, generator=g, device=DEV)) * d ** -0.5
        self.w2s = (0.5 + torch.rand(Ne, d // 128, self.N1 // 256, generator=g, device=DEV)) * (self.N1 // 2) ** -0.5
        nb = MAX_REQS * self.pages
        self.caches = [rand((nb, self.page, C + Rr), g)]
        self.bt = torch.randperm(nb, generator=torch.Generator().manual_seed(32)).view(MAX_REQS, self.pages).int().to(DEV)
        self.lens = paged_lens(self.page)
        self.lens_incl = self.lens + 1
        self.be = B200AttnBackend(max_seq_len=self.page * self.pages, max_reqs=MAX_REQS, n_local_heads=H)
        self.h = {B: torch.empty(B, d, dtype=BF, device=DEV) for B in ORDER}

    @staticmethod
    def fp8_weight(shape, g):
        N, K = shape
        s = (0.5 + torch.rand(-(-N // 128), K // 128, generator=g, device=DEV)) * K ** -0.5
        return torch.randn(shape, generator=g, device=DEV).to(F8), s

    @staticmethod
    def deq(q, s):
        N, K = q.shape[-2:]
        return q.double() * s.double().repeat_interleave(128, -2)[..., :N, :].repeat_interleave(128, -1)[..., :K]

    new_inputs = Llama.new_inputs

    def prepare(self, B):
        self.be.prepare_metadata_for_decode(self.lens[:B], self.lens_incl[:B], self.bt[:B], self.page)

    def advance(self, B):
        self.lens[:B] += 1
        self.lens_incl.copy_(self.lens + 1)

    def attention(self, h, kv_cache, lens, incl, bt):
        from chitu_b200 import ops
        B, H, C = h.shape[0], self.H, self.C
        xn = ops.rms_norm(h, self.n1, EPS)
        q = ops.linear_deepseek_v3(xn, *self.wq, soft_fp8=False).view(B, H, C + self.Rr)
        kv = ops.linear_deepseek_v3(xn, *self.wkv, soft_fp8=True)[:, : C + self.Rr].contiguous()
        o = self.be.mla_attn_with_kvcache(q[..., :C].contiguous(), q[..., C:].contiguous(), kv_cache, kv, lens, incl,
                                          bt, softmax_scale=self.scale)
        return h + ops.linear_deepseek_v3(o.reshape(B, H * C), *self.wo, soft_fp8=False)

    def moe(self, h):
        from chitu_b200 import fused_moe, ops
        xn = ops.rms_norm(h, self.n2, EPS)
        w, idx = fused_moe.moe_gate(xn, self.gate_w, self.gate_b, self.topk, self.groups, self.topk_groups, "sigmoid",
                                    self.route_scale)
        ids = torch.cat([idx, torch.full_like(idx[:, :1], self.E)], dim=1)
        w = torch.cat([w, torch.ones_like(w[:, :1])], dim=1)
        y = fused_moe.fused_experts(xn, self.w1, self.w2, w, ids, use_fp8_w8a8=True, w1_scale=self.w1s,
                                    w2_scale=self.w2s, block_shape=[128, 128])
        return h + y, idx

    def body(self, B, caches):
        h = self.h[B]
        h2 = self.attention(h, caches[0], self.lens[:B], self.lens_incl[:B], self.bt[:B])
        h3, idx = self.moe(h2)
        return [h, h2, h3, idx]

    def fp8_ref(self, x, w_d):
        xq, xs = R.act_quant(x.contiguous())
        return ((xq.double() * xs.double().repeat_interleave(128, -1)) @ w_d.T).to(BF)

    def attention_ref(self, h, kv_cache, lens, bt):
        B, H, C = h.shape[0], self.H, self.C
        xn = R.rms_norm(h, self.n1, EPS, F64)
        q = self.fp8_ref(xn, self.wq_d).view(B, H, C + self.Rr)
        kv = (xn.double() @ self.wkv_bf.double().T).to(BF)[:, : C + self.Rr].contiguous()
        o = R.mla_attn_with_kvcache(q[..., :C].contiguous(), q[..., C:].contiguous(), kv_cache, kv, lens, bt, self.scale,
                                    F64)
        return h + self.fp8_ref(o.reshape(B, H * C), self.wo_d)

    def experts_ref(self, x, ids, w):
        """fp8 fused_experts in fp64 with the kernel's roundings (R.fused_experts, each expert dequantised once)."""
        xq, xs = R.group_quant(x)
        c3 = torch.zeros(x.shape[0], ids.shape[1], x.shape[1], dtype=BF, device=DEV)
        act = lambda q, s: q.double() * s.double().repeat_interleave(128, -1)
        for e in torch.unique(ids).tolist():
            tok, slot = (ids == e).nonzero(as_tuple=True)
            h1 = (act(xq[tok], xs[tok]) @ self.deq(self.w1[e], self.w1s[e]).T).to(BF)
            aq, a_s = R.group_quant(R.silu_and_mul(h1))
            y = act(aq, a_s) @ self.deq(self.w2[e], self.w2s[e]).T
            c3[tok, slot] = (y * w[tok, slot].double()[:, None]).to(BF)
        return c3.double().sum(dim=1).to(BF)

    def check(self, B, out, before, after, gen):
        h, h2, h3, idx = out
        lens, bt = self.lens[:B], self.bt[:B]
        fails, worst = [], 0.0
        keep = []

        def attn_ref(hh, keep=None):
            cache = before[0].clone()
            y = self.attention_ref(hh, cache, lens, bt)
            if keep is not None:
                keep.append(cache)
            return y
        err, bnd, f = increment_check(attn_ref, h, h2, gen, "attention")
        worst, fails = max(worst, err / bnd), fails + [f] * (f is not None)
        attn_ref(h, keep)
        kv = check_append(after[0], before[0], keep[0], bt, lens, self.page, 2.0 ** -5)
        if kv > 1.0:
            fails.append(f"an appended latent value is {kv:.2f} roundings from the reference's")
        xn = R.rms_norm(h2, self.n2, EPS, F64)
        _, ref_idx, masked = R.moe_gate(xn.double(), self.gate_w.double(), self.gate_b.double(), self.topk, self.groups,
                                        self.topk_groups, "sigmoid", self.route_scale)
        cfg = type("Cfg", (), dict(n_expert_groups=self.groups, n_limited_groups=self.topk_groups))
        margin = R._group_margin(xn.double(), self.gate_w.double(), self.gate_b.double(), cfg)
        kept_rows(idx, [(ref_idx, masked, margin)], self.topk)
        ids = torch.cat([idx, torch.full_like(idx[:, :1], self.E)], dim=1)

        def moe_ref(hh):
            x = R.rms_norm(hh, self.n2, EPS, F64)
            s = torch.sigmoid(x.double() @ self.gate_w.double().T).gather(1, idx)
            w = torch.cat([s / s.sum(dim=-1, keepdim=True) * self.route_scale, torch.ones_like(s[:, :1])], dim=1)
            return hh + self.experts_ref(x, ids, w)
        err, bnd, f = increment_check(moe_ref, h2, h3, gen, "moe")
        return max(worst, err / bnd), fails + [f] * (f is not None)

    def grow(self):
        """The gate over 1024 tokens: "moe_gate" outgrows its reservation."""
        from chitu_b200 import fused_moe
        x = rand((1024, self.dim), torch.Generator(device=DEV).manual_seed(9))
        fused_moe.moe_gate(x, self.gate_w, self.gate_b, self.topk, self.groups, self.topk_groups, "sigmoid", 1.0)
        return ("moe_gate",)


FAMILIES = {"llama": Llama, "mixtral": Mixtral, "deepseek": DeepSeek}


def reserve(fam):
    from chitu_b200 import plugin, workspace
    if fam.reserve_shapes is None:
        plugin.install(max_reqs=MAX_REQS, device=torch.device(DEV))
    else:
        workspace.reserve_decode(torch.device(DEV), MAX_REQS, **fam.reserve_shapes)


def replay(fam, graphs, B, seed):
    fam.new_inputs(B, seed)
    fam.prepare(B)
    graphs[B][0].replay()
    torch.cuda.synchronize()
    return [o.clone() for o in graphs[B][1]], [c.clone() for c in fam.caches]


@pytest.mark.gpu
@pytest.mark.parametrize("family", list(FAMILIES))
def test_arrival_order_graphs(family):
    from chitu_b200 import workspace
    fresh_workspaces()
    fam = FAMILIES[family]()
    reserve(fam)
    held = tag_state()
    assert set(held) == {"attn", "linear", "moe", "moe_gate"}, held

    # 1. capture in arrival order; the only eager step runs at the first batch size
    fam.new_inputs(ORDER[0], 0)
    fam.prepare(ORDER[0])
    fam.body(ORDER[0], [c.clone() for c in fam.caches])
    torch.cuda.synchronize()
    graphs = {}
    for B in ORDER:
        fam.new_inputs(B, B)
        fam.prepare(B)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fam.body(B, fam.caches)
        graphs[B] = (g, out)
    torch.cuda.synchronize()
    assert tag_state() == held, "a workspace buffer moved while the graphs were captured"
    assert workspace.retired_bytes() == 0

    # 2. interleaved replays: graph == eager on a cloned state, bit for bit, and within the fp64 bound
    gen = torch.Generator(device=DEV).manual_seed(12)
    fails, worst = [], 0.0
    for t, B in enumerate(SCHEDULE):
        fam.new_inputs(B, 1000 + t)
        fam.prepare(B)
        before = [c.clone() for c in fam.caches]
        mine = [c.clone() for c in before]
        eager = fam.body(B, mine)
        graphs[B][0].replay()
        torch.cuda.synchronize()
        out = graphs[B][1]
        for i, (e, o) in enumerate(zip(eager, out)):
            assert same_bits(e, o), f"step {t} (B = {B}): output {i} of the replay differs from the eager run"
        for i, (e, c) in enumerate(zip(mine, fam.caches)):
            assert same_bits(e, c), f"step {t} (B = {B}): cache {i} of the replay differs from the eager run"
        w, f = fam.check(B, out, before, fam.caches, gen)
        worst = max(worst, w)
        fails += [f"step {t} (B = {B}): {x}" for x in f]
        fam.advance(B)
    print(f"{family}: worst err / bound over {len(SCHEDULE)} replays {worst:.3f}")
    assert not fails, "\n".join(fails)
    assert tag_state() == held and workspace.retired_bytes() == 0

    # 3. an eager call outgrows a tag the graphs hold: the old buffer is retired and the graphs replay as before
    state = list(fam.caches) + [t for t in (getattr(fam, "lens", None), getattr(fam, "lens_incl", None)) if t is not None]
    snap = [t.clone() for t in state]

    def restore():
        for t, s in zip(state, snap):
            t.copy_(s)
    first = {}
    for B in ORDER:
        restore()
        first[B] = replay(fam, graphs, B, 5000 + B)
    grown = fam.grow()
    torch.cuda.synchronize()
    now = tag_state()
    assert all(now[t] != held[t] for t in grown), (grown, held, now)
    assert workspace.retired_bytes() > 0, "an outgrown buffer the graphs hold was not retired"
    traps = [torch.full((b.numel(),), 0xFF, dtype=torch.uint8, device=DEV) for b in workspace._retired]
    for B in ORDER:
        restore()
        outs, caches = replay(fam, graphs, B, 5000 + B)
        assert all(same_bits(a, b) for a, b in zip(outs, first[B][0])), f"B = {B}: replay changed after the growth"
        assert all(same_bits(a, b) for a, b in zip(caches, first[B][1])), f"B = {B}: caches changed after the growth"
    del traps, graphs
    fresh_workspaces()


def gqa_case(B, L, pages, seed, page=256, Hq=4, Hkv=1, D=128):
    g = torch.Generator(device=DEV).manual_seed(seed)
    kc, vc = (rand((B * pages, page, Hkv, D), g) for _ in range(2))
    return dict(q=rand((B, 1, Hq, D), g), kc=kc, vc=vc, k=rand((B, 1, Hkv, D), g), v=rand((B, 1, Hkv, D), g),
                lens=torch.full((B,), L, dtype=torch.int32, device=DEV),
                bt=torch.arange(B * pages, dtype=torch.int32, device=DEV).view(B, pages))


def gqa_call(be, c, kc, vc):
    return be.attn_with_kvcache(c["q"], kc, vc, c["k"], c["v"], cache_seqlens=c["lens"], block_table=c["bt"])


def gqa_err(c, out, gen):
    """(err, bound) of a GQA decode output against the fp64 reference (floor: q moved by one bf16 ulp)."""
    def ref(q):
        return R.gqa_paged_decode(q, c["kc"].clone(), c["vc"].clone(), c["k"], c["v"], c["lens"], c["bt"],
                                  compute_dtype=F64)
    want = ref(c["q"])
    floor = max(rel_err(ref(ulp_perturb(c["q"], gen)), want) for _ in range(FLOOR_SEEDS))
    return rel_err(out, want), bound(floor)


@pytest.mark.gpu
def test_growth_during_capture_raises_and_leaves_the_buffer():
    """Capturing at a batch above the reservation raises the workspace error naming the tag; the buffer stays where it
    was, and the next eager call at that batch is correct."""
    from chitu_b200 import workspace
    from chitu_b200.attn_backend import B200AttnBackend
    fresh_workspaces()
    workspace.reserve_decode(torch.device(DEV), 8, heads=4, head_dim_v=128)
    held = tag_state()
    be = B200AttnBackend(max_reqs=8, n_local_heads=4)
    c = gqa_case(16, 300, 2, 41)
    kc, vc = c["kc"].clone(), c["vc"].clone()
    warm = gqa_case(2, 300, 2, 42)
    gqa_call(be, warm, warm["kc"], warm["vc"])                        # loads the kernels
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="workspace 'attn'"):
        with torch.cuda.graph(g):
            gqa_call(be, c, kc, vc)
    del g
    torch.cuda.synchronize()
    assert tag_state() == held, "the failed capture moved a workspace buffer"
    assert torch.equal(kc.view(torch.uint8), c["kc"].view(torch.uint8)), "the failed capture ran the append"
    out = gqa_call(be, c, kc, vc)
    torch.cuda.synchronize()
    err, bnd = gqa_err(c, out, torch.Generator(device=DEV).manual_seed(43))
    assert err <= bnd, (err, bnd)
    assert tag_state()["attn"][1] > held["attn"][1]
    fresh_workspaces()


@pytest.mark.gpu
def test_plan_tail_of_the_attention_workspace():
    """prepare_metadata_for_decode's split plan in the tail of "attn": a GQA call at the largest split count leaves it
    unchanged, its words equal the host model, and an MLA replay at another batch size refuses it and stays within the
    bound (the replay at the plan's own batch size honours it)."""
    from chitu_b200 import _lib, plugin
    from chitu_b200.attn_backend import B200AttnBackend
    fresh_workspaces()
    plugin.install(max_reqs=MAX_REQS, device=torch.device(DEV))
    H, C, Rr, page, pages = 16, 512, 64, 64, 8
    hint = page * pages
    be = B200AttnBackend(max_seq_len=hint, max_reqs=MAX_REQS, n_local_heads=H)
    g = torch.Generator(device=DEV).manual_seed(51)
    kv_cache = rand((MAX_REQS * pages, page, C + Rr), g)
    bt = torch.randperm(MAX_REQS * pages, generator=torch.Generator().manual_seed(52)).view(MAX_REQS, pages).int().to(DEV)
    lens = paged_lens(page)
    incl = lens + 1
    static = {B: dict(q_nope=rand((B, H, C), g), q_pe=rand((B, H, Rr), g), kv=rand((B, C + Rr), g)) for B in (8, 16)}

    def mla(B, cache, q_nope=None):
        s = static[B]
        return be.mla_attn_with_kvcache(s["q_nope"] if q_nope is None else q_nope, s["q_pe"], cache, s["kv"], lens[:B],
                                        incl[:B], bt[:B], softmax_scale=192 ** -0.5)

    be.prepare_metadata_for_decode(lens[:8], incl[:8], bt[:8], page)
    mla(8, kv_cache.clone())                                       # load the kernels
    torch.cuda.synchronize()
    graphs = {}
    for B in (8, 16):
        be.prepare_metadata_for_decode(lens[:B], incl[:B], bt[:B], page)
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            out = mla(B, kv_cache)
        graphs[B] = (gr, out)

    be.prepare_metadata_for_decode(lens[:8], incl[:8], bt[:8], page)
    torch.cuda.synchronize()
    ws, n = be._ws(8, H, C, DEV)
    plan = be.last_plan()
    assert plan.data_ptr() == ws.data_ptr() + n - _lib.ATTN_PLAN_BYTES
    want = attn_plan(incl[:8].tolist(), H, page, hint, n)
    assert plan[:7].tolist() == [want[w] for w in range(7)], "plan words differ from the host model"
    plan_before = plan.clone()

    # GQA at its largest split count (one request, one KV head, 40 pages of 256 keys) shares the buffer
    c = gqa_case(1, 40 * 256 - 8, 40, 54)
    assert gqa_splits("tc", 1, 4, 1, 128, 40 * 256, n) == 64
    gb = B200AttnBackend(max_reqs=MAX_REQS, n_local_heads=4)
    out = gqa_call(gb, c, c["kc"].clone(), c["vc"].clone())
    torch.cuda.synchronize()
    assert be._ws(1, 4, 128, DEV)[0].data_ptr() == ws.data_ptr(), "GQA did not run in the same attention workspace"
    assert torch.equal(plan, plan_before), "the GQA partials overwrote the split plan in the workspace tail"
    err, bnd = gqa_err(c, out, torch.Generator(device=DEV).manual_seed(55))
    assert err <= bnd, ("gqa", err, bnd)

    gen = torch.Generator(device=DEV).manual_seed(56)
    for B in (8, 16):                                      # the plan was made for B = 8
        splits = mla_num_splits(B, H, hint, n)
        honoured = [plan_honoured(want, B, H, L, splits) for L in incl[:B].tolist()]
        assert all(k is not None for k in honoured) if B == 8 else all(k is None for k in honoured), (B, honoured)
        before = kv_cache.clone()
        graphs[B][0].replay()
        torch.cuda.synchronize()
        got = graphs[B][1]
        s = static[B]

        def ref(q_nope):
            return R.mla_attn_with_kvcache(q_nope, s["q_pe"], before.clone(), s["kv"], lens[:B], bt[:B], 192 ** -0.5,
                                           F64)
        want_o = ref(s["q_nope"])
        floor = max(rel_err(ref(ulp_perturb(s["q_nope"], gen)), want_o) for _ in range(FLOOR_SEEDS))
        err = rel_err(got.view(B, H, C), want_o)
        assert err <= bound(floor), (B, err, bound(floor))
        assert torch.equal(plan, plan_before), "an MLA replay changed the plan"
        kv_cache.copy_(before)
    del graphs
    fresh_workspaces()


@pytest.mark.gpu
def test_grouped_gemm_workspace_is_off_the_decode_path(monkeypatch):
    """fused_experts never asks for "moe_gg" (invoke_fused_moe_kernel's workspace, left unreserved), and a first
    invoke_fused_moe_kernel inside a capture raises instead of growing it."""
    from chitu_b200 import fused_moe, plugin, workspace
    fresh_workspaces()
    plugin.install(max_reqs=MAX_REQS, device=torch.device(DEV))
    fam = Mixtral()
    asked, get = [], workspace.get
    monkeypatch.setattr(workspace, "get", lambda tag, n, dev: asked.append(tag) or get(tag, n, dev))
    monkeypatch.setattr(fused_moe, "invoke_fused_moe_kernel", None)
    fam.new_inputs(16, 61)
    fam.body(16, [])
    torch.cuda.synchronize()
    assert "moe_gg" not in asked and "moe" in asked, asked
    monkeypatch.undo()

    g = torch.Generator(device=DEV).manual_seed(62)
    T, topk, E, N, K = 4, 2, 8, 256, 128
    A, B = rand((T, K), g), rand((E, N, K), g, K ** -0.5)
    ids = torch.randint(0, E, (T, topk), generator=g, device=DEV, dtype=torch.int32)
    w = torch.rand(T, topk, generator=g, device=DEV)
    sorted_ids, expert_ids, npad = fused_moe.moe_align_block_size(ids, 16, E)
    Cout = torch.empty(T, topk, N, dtype=BF, device=DEV)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="workspace 'moe_gg'"):
        with torch.cuda.graph(gr):
            fused_moe.invoke_fused_moe_kernel(A, B, Cout, None, None, None, w, ids, sorted_ids, expert_ids, npad, False,
                                              topk, {"BLOCK_SIZE_M": 16})
    del gr
    assert "moe_gg" not in tag_state()
    fresh_workspaces()
