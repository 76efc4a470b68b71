"""Layer-level golden vectors: run the REAL reference transformer blocks (a thu-pacman/chitu checkout at $CHITU_REFERENCE)
on CPU with small dimensions and record inputs, weights and outputs.

    python oracle/gen_golden_models.py            (authoring container only; writes tests/golden/block_*.npz)

* `TransformerBlockLlama` (models/model_llama.py:160-185) with `RefAttnBackend` (attn_backend.py:245-501) over a
  contiguous KV cache: pins the assembly the oracle's `llama_decode_step` restates (norm placement, separate
  wq/wk/wv, interleaved rotary, in-place append, residuals, SwiGLU).
* `TransformerBlockDeepSeekV3` decode (models/model_deepseek_v3.py): see gen_deepseek_block().
The reference's Triton kernels run under TRITON_INTERPRET=1 (SURVEY.md Appendix A).
"""
import os
import sys
import types
from types import SimpleNamespace

os.environ["TRITON_INTERPRET"] = "1"
os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
os.environ.setdefault("MASTER_PORT", "29578")
os.environ.setdefault("RANK", "0")
os.environ.setdefault("WORLD_SIZE", "1")
REF = os.environ.get("CHITU_REFERENCE", "reference")   # checkout of thu-pacman/chitu
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import numpy as np
import torch
from oracle.golden_inputs import compact  # noqa: E402

sys.modules["chitu_backend"] = types.ModuleType("chitu_backend")
for name in ("w8a8gemm", "w8a8gemv"):
    sys.modules[name] = types.ModuleType(name)
import chitu.device_type as D  # noqa: E402

D._device_name = "cpu"
torch.cuda.synchronize = lambda *a, **k: None

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")


def bits(t):
    if not torch.is_tensor(t):
        return np.asarray(t)
    if t.dtype == torch.bfloat16:
        return t.contiguous().view(torch.int16).numpy().view(np.uint16)
    if t.dtype == torch.float8_e4m3fn:
        return t.contiguous().view(torch.uint8).numpy()
    return t.contiguous().numpy()


def save(name, **arrs):
    """Writes the stored form (oracle/golden_inputs.compact): large seeded inputs as SHA-256, near-copies as deltas."""
    full = {k: bits(v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **compact(name, full))
    print("wrote", name, {k: tuple(v.shape) for k, v in full.items()})


def bootstrap():
    import torch.distributed as dist
    if not dist.is_initialized():
        dist.init_process_group("gloo", rank=0, world_size=1)
    from chitu import global_vars
    if global_vars._GLOBAL_TIMERS is None:
        global_vars._set_timers()


class ContiguousCache:
    """What Attention.decode_forward needs from KVCacheManager (cache_manager.py): per-layer (k, v) of shape
    [B, max_len, Hkv, D] and the lengths before this decode."""

    def __init__(self, k, v, seqlens):
        self.k, self.v, self.seqlens = k, v, seqlens

    def get_cache_decode(self, layer_id):
        return self.k, self.v

    def get_gpu_seq_lens_excl_this_decode(self):
        return self.seqlens


def gen_llama_block():
    bootstrap()
    from chitu.attn_backend import RefAttnBackend
    from chitu.models.model_llama import TransformerBlockLlama

    torch.manual_seed(21)
    torch.set_default_dtype(torch.bfloat16)
    args = SimpleNamespace(dim=256, n_heads=8, n_kv_heads=2, multiple_of=64, ffn_dim_multiplier=None, norm_eps=1e-5)
    B, max_len, D, Hkv = 3, 48, 32, 2
    seqlens = torch.tensor([17, 40, 5], dtype=torch.long)
    k = torch.randn(B, max_len, Hkv, D)
    v = torch.randn(B, max_len, Hkv, D)
    cache = ContiguousCache(k.clone(), v.clone(), seqlens)
    blk = TransformerBlockLlama(0, args, cache, RefAttnBackend(), "torch")
    with torch.no_grad():
        for n, p in blk.named_parameters():
            if "norm" in n:
                p.copy_(1.0 + 0.1 * torch.randn_like(p))
            else:
                p.copy_(torch.randn_like(p) * 0.05)
    x = torch.randn(B, 1, args.dim)
    ang = torch.rand(B, D // 2, dtype=torch.float32) * 6.28
    cos, sin = torch.cos(ang), torch.sin(ang)
    with torch.no_grad():
        y = blk(x.clone(), cos, sin)
    torch.set_default_dtype(torch.float32)
    sd = {n.replace(".", "__"): p.detach() for n, p in blk.named_parameters()}
    save("block_llama", x=x, cos=cos, sin=sin, k_cache=k, v_cache=v, seqlens=seqlens, y=y,
         k_after=cache.k, v_after=cache.v, cfg=np.array([args.dim, args.n_heads, args.n_kv_heads]), **sd)


def gen_deepseek_blocks():
    """TransformerBlockDeepSeekV3.forward in paged decode mode (model_deepseek_v3.py:1100-1114, 672-699, 475-536,
    755-771, 921-1011) with mla_absorb = "absorb-without-precomp", merged qkv / gate-up weights, FP8 block-scaled
    linears (act_quant + fp8 GEMM Triton kernels), the Triton MLA decode kernels and the Triton fused experts."""
    bootstrap()
    from chitu import global_vars, ops
    from chitu.attn_backend import TritonAttnBackend
    from chitu.cache_manager import PagedKVCacheManager
    from chitu.models.model_deepseek_v3 import TransformerBlockDeepSeekV3

    # the autotuner cannot benchmark on CPU: keep one configuration per autotuned reference kernel
    import triton
    import chitu.fused_moe as _fm
    import chitu.triton_decode_attention as _tda
    import chitu.triton_kernels as _tk
    for mod in (_fm, _tda, _tk):
        for name in dir(mod):
            obj = getattr(mod, name)
            if isinstance(obj, triton.runtime.autotuner.Autotuner):
                obj.configs = obj.configs[:1]
                print("autotuner pinned:", mod.__name__, name, obj.configs[0])

    from oracle.synth_blocks import deepseek_args
    margs = deepseek_args()
    if global_vars._GLOBAL_ARGS is None:
        global_vars.set_global_args(SimpleNamespace(
            infer=SimpleNamespace(soft_fp8=False, tp_size=1, mla_absorb="absorb-without-precomp"), models=margs))

    class Fp32MLABackend(TritonAttnBackend):
        """bf16 `tl.dot` is broken in the Triton CPU interpreter (SURVEY.md 8c caveat 1): the reference kernels
        are fed fp32 tensors holding the same bf16 values; the append itself happens on the bf16 cache."""

        def mla_attn_with_kvcache(self, q_nope, q_pe, kv_cache, kv, cache_seqlens_excl_this_decode,
                                  cache_seqlens_incl_this_decode, block_table, softmax_scale=None, **kw):
            ops.append_to_paged_kv_cache(kv_cache, block_table, kv, cache_seqlens_excl_this_decode)
            out = super().mla_attn_with_kvcache(
                q_nope.float(), q_pe.float(), kv_cache.float(), kv.float(),
                cache_seqlens_excl_this_decode=cache_seqlens_excl_this_decode,
                cache_seqlens_incl_this_decode=cache_seqlens_incl_this_decode, block_table=block_table,
                softmax_scale=softmax_scale)
            return out.to(q_nope.dtype)

    class PagedStub(PagedKVCacheManager):
        def __init__(self, cache, table, seqlens):
            self.cache, self.table, self.excl = cache, table, seqlens
            self.incl = seqlens + 1

        def get_gpu_block_table(self):
            return self.table

        def get_gpu_seq_lens_excl_this_decode(self):
            return self.excl

        def get_gpu_seq_lens_incl_this_decode(self):
            return self.incl

        def get_paged_kv_cache(self, layer_id):
            return self.cache

    from oracle.synth_blocks import checksum, synth_deepseek_block

    for layer_id, tag, seed in ((0, "dense", 31), (1, "moe", 32)):
        P, I = synth_deepseek_block(margs, layer_id, seed)
        page = I["kv_cache"].shape[1]
        stub = PagedStub(I["kv_cache"].clone(), I["table"], I["seqlens"])
        backend = Fp32MLABackend()
        backend.prepare_metadata_for_decode(stub.excl, stub.incl, I["table"], page)
        torch.set_default_dtype(torch.bfloat16)      # the reference runs with bf16 as default dtype (backend.py:119);
        blk = TransformerBlockDeepSeekV3(layer_id, margs, stub, backend, "torch", mla_absorb="absorb-without-precomp",
                                         merge_qkv_gate_up=True)
        params = dict(blk.named_parameters())
        assert set(params) == set(P), (sorted(set(params) ^ set(P)))
        with torch.no_grad():
            for n, p in params.items():
                assert p.shape == P[n].shape and p.dtype == P[n].dtype, (n, p.shape, p.dtype, P[n].shape, P[n].dtype)
                p.data = P[n].clone()
            cap = {}
            blk.ffn_norm.register_forward_pre_hook(lambda m, inp: cap.__setitem__("h_mid", inp[0].clone()))
            if layer_id >= margs.n_dense_layers:
                blk.ffn.gate.register_forward_hook(lambda m, inp, out: cap.__setitem__("route", (out[0].clone(), out[1].clone())))
            y = blk(I["x"].clone(), I["cos"], I["sin"])   # fp8_gemm_deepseek_v3 allocates its output in the default dtype
        torch.set_default_dtype(torch.float32)
        assert y.dtype == torch.bfloat16
        B = y.shape[0]
        rows = torch.stack([stub.cache[int(I["table"][b, int(I["seqlens"][b]) // page]), int(I["seqlens"][b]) % page]
                            for b in range(B)])
        untouched = stub.cache.clone()
        for b in range(B):
            L = int(I["seqlens"][b])
            untouched[int(I["table"][b, L // page]), L % page] = I["kv_cache"][int(I["table"][b, L // page]), L % page]
        assert torch.equal(untouched, I["kv_cache"])
        extra = {}
        if "route" in cap:
            extra = dict(route_w=cap["route"][0], route_idx=cap["route"][1])
        save(f"block_deepseek_{tag}", y=y, h_mid=cap["h_mid"], kv_new_rows=rows, **extra, seed=np.array([seed]), layer_id=np.array([layer_id]),
             checksum=checksum(P, I), softmax_scale=np.array([blk.attn.softmax_scale], dtype=np.float64))

def gen_mixtral_moe():
    """SparseMoeBlockHFMixtral.forward (models/model_hf_mixtral.py:51-96): softmax(fp32) -> top-2 -> renormalise ->
    per-expert gather / SwiGLU FeedForward / weighted index_add_.  Pure torch (no Triton kernel on this path)."""
    bootstrap()
    from chitu.models.model_hf_mixtral import SparseMoeBlockHFMixtral

    torch.manual_seed(41)
    torch.set_default_dtype(torch.bfloat16)
    dim, hidden, E, topk, T = 256, 384, 8, 2, 7
    blk = SparseMoeBlockHFMixtral(dim, hidden, E, topk, op_impl="torch", merge_gate_up=True)
    with torch.no_grad():
        for n, p in blk.named_parameters():
            p.copy_(torch.randn_like(p) * (0.3 if "gate.weight" in n else 0.06))
    x = torch.randn(T, dim)
    with torch.no_grad():
        y = blk(x.clone())
    torch.set_default_dtype(torch.float32)
    w1 = torch.stack([blk.experts[e].gate_up_proj.weight.detach() for e in range(E)])
    w2 = torch.stack([blk.experts[e].down_proj.weight.detach() for e in range(E)])
    save("block_mixtral_moe", x=x, y=y, gate_w=blk.gate.weight.detach(), w1=w1, w2=w2, cfg=np.array([E, topk]))


if __name__ == "__main__":
    which = sys.argv[1:] or ["llama"]
    if "llama" in which:
        gen_llama_block()
    if "mixtral" in which:
        gen_mixtral_moe()
    if "deepseek" in which:
        gen_deepseek_blocks()
