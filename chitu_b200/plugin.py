"""`install()` patches this library's operators into an importable reference `chitu` package so that
`chitu.executor` / `cache_manager` / the model files run unchanged (SURVEY.md §8b):

  * `sys.modules["chitu_backend"]`      <- chitu_b200.chitu_backend      (csrc/binding.cpp:11-19)
  * `sys.modules["w8a8gemm" / "w8a8gemv"]` <- chitu_b200.quantize.*        (quantize/w8a8.py:4-5)
  * names in `chitu.ops`, and in every module that imported them BY NAME
    (`chitu.attn_backend`, `chitu.models.model`, `chitu.models.model_deepseek_v3`, ...)  are rebound
  * `chitu.fused_moe.{moe_align_block_size, per_token_group_quant_fp8, fused_experts}` are rebound
  * `chitu.attn_backend.B200AttnBackend` is added; `chitu.backend.Backend.build` selects it for
    `infer.attn_type == "b200"` through the one-line `elif` shown in INTEGRATION.md.

Call it BEFORE `chitu.backend.Backend.build` (ideally before importing chitu.models.*).
"""
from __future__ import annotations

import importlib
import sys

_OPS = ["append_to_paged_kv_cache", "apply_rotary_pos_emb", "apply_rotary_pos_emb_triton", "act_quant_deepseek_v3",
        "weight_dequant_deepseek_v3", "weight_dequant_soft_fp8_deepseek_v3", "fp8_gemm_deepseek_v3",
        "soft_fp8_gemm_deepseek_v3"]
_MOE = ["moe_align_block_size", "per_token_group_quant_fp8", "fused_experts", "invoke_fused_moe_kernel"]


def install(verbose: bool = False, max_reqs: int = 0, device=None):
    """`max_reqs` > 0 (infer.max_reqs): size every persistent workspace once for the largest decode batch, so that
    the reference's per-batch-size CUDA graphs (models/model.py:537-622) never see a workspace move."""
    from . import attn_backend, chitu_backend, fused_moe, ops, workspace
    if max_reqs > 0:
        import torch
        workspace.reserve_decode(device if device is not None else torch.device("cuda", torch.cuda.current_device()),
                                 max_reqs)
    from .quantize import w8a8gemm, w8a8gemv

    sys.modules.setdefault("chitu_backend", chitu_backend)
    sys.modules["chitu_backend"] = chitu_backend
    sys.modules["w8a8gemm"] = w8a8gemm
    sys.modules["w8a8gemv"] = w8a8gemv
    patched = []
    try:
        ref_ops = importlib.import_module("chitu.ops")
    except ModuleNotFoundError as e:
        # only "there is no reference package here" degrades to shims; a reference that is present but fails to
        # import is a real integration failure and must not be hidden
        if e.name is None or e.name.split(".")[0] != "chitu":
            raise
        if verbose:
            print(f"chitu_b200.install: reference package not importable ({e}); installed module shims only")
        return patched
    for name in _OPS:
        setattr(ref_ops, name, getattr(ops, name))
        patched.append(f"chitu.ops.{name}")
    ref_moe = importlib.import_module("chitu.fused_moe")
    for name in _MOE:
        setattr(ref_moe, name, getattr(fused_moe, name))
        patched.append(f"chitu.fused_moe.{name}")
    ref_attn = importlib.import_module("chitu.attn_backend")
    ref_attn.B200AttnBackend = attn_backend.B200AttnBackend
    # modules that did `from .ops import x` hold their own reference: rebind there too
    for modname, mod in list(sys.modules.items()):
        if not modname.startswith("chitu.") or mod is None:
            continue
        for name in _OPS + _MOE:
            if hasattr(mod, name) and modname not in ("chitu.ops", "chitu.fused_moe"):
                src = ops if name in _OPS else fused_moe
                setattr(mod, name, getattr(src, name))
                patched.append(f"{modname}.{name}")
    if verbose:
        print("chitu_b200.install: patched", len(patched), "names")
    return patched
