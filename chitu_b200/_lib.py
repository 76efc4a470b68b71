"""ctypes binding of libchitu_b200.so (the C ABI declared in include/chitu_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, a
RuntimeError is raised (SURVEY.md §8b "Errors": the reference's native code exit()s; here the
status code + chitu_b200_last_error() become a Python exception).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import threading
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("CHITU_B200_LIB") or os.path.join(_HERE, "libchitu_b200.so")   # CHITU_B200_LIB: profiling build
CSRC_DIR = os.path.join(_HERE, "csrc")

# dtype codes (include/chitu_b200.h)
CB_BF16, CB_F16, CB_F32, CB_FP8_E4M3, CB_I8, CB_U8, CB_I16, CB_I32, CB_I64 = range(9)
# split-KV attention workspace (csrc/splitkv.cuh): the kernels split the keys at most ATTN_MAX_SPLITS ways, and the
# last ATTN_PLAN_BYTES bytes hold the device-side split plan
ATTN_MAX_SPLITS, ATTN_PLAN_BYTES = 128, 256

_lock = threading.Lock()
_lib = None

P, I, L, F = c_void_p, c_int, c_int64, c_float

# name -> (restype, argtypes); must list every symbol of include/chitu_b200.h
SIGNATURES = {
    "chitu_b200_last_error": (c_char_p, []),
    "chitu_b200_version": (I, []),
    "chitu_b200_launch_count": (L, []),
    "chitu_b200_append_paged_kv": (I, [P, P, P, P, I, I, I, I, L, P]),
    "chitu_b200_append_paged_kv_e4m3": (I, [P, P, P, P, I, I, I, I, P]),
    "chitu_b200_scatter_kv": (I, [P, P, P, L, P, L, P, P, P, I, I, L, I, I, I, I, I, I, P]),
    "chitu_b200_moe_align_block_size": (I, [P, I, L, I, I, P, P, P, P, P]),
    "chitu_b200_moe_gate_workspace_bytes": (L, [I, I]),
    "chitu_b200_moe_gate": (I, [P, P, P, I, I, I, I, I, I, I, I, F, P, P, I, P, L, P]),
    "chitu_b200_rotary_interleaved": (I, [P, P, P, P, P, P, I, I, I, I, L, L, L, L, I, P]),
    "chitu_b200_rotary_half": (I, [P, P, P, P, I, I, I, I, P]),
    "chitu_b200_rotary_half_strided": (I, [P, L, P, P, P, I, I, I, I, P]),
    "chitu_b200_rmsnorm": (I, [P, P, P, I, I, F, I, P]),
    "chitu_b200_rmsnorm_strided": (I, [P, P, P, I, I, L, L, F, I, P]),
    "chitu_b200_rmsnorm_quant_fp8": (I, [P, P, P, P, P, I, I, L, L, F, P]),
    "chitu_b200_silu_mul_quant_fp8": (I, [P, P, P, L, I, P]),
    "chitu_b200_silu_and_mul": (I, [P, P, L, I, I, P]),
    "chitu_b200_act_quant_fp8": (I, [P, P, P, L, I, I, I, F, I, P]),
    "chitu_b200_quant_act_int8": (I, [P, P, P, L, I, I, P]),
    "chitu_b200_quant_fp8_rowwise": (I, [P, P, P, L, I, P, P, P]),
    "chitu_b200_rmsnorm_quant_fp8_rowwise": (I, [P, P, P, P, P, I, I, F, P]),
    "chitu_b200_weight_dequant_fp8": (I, [P, P, P, I, I, I, I, I, P]),
    "chitu_b200_linear_workspace_bytes": (L, [I, I]),
    "chitu_b200_linear_bf16": (I, [P, P, P, P, P, I, I, I, I, P, L, I, P]),
    "chitu_b200_linear_bf16_silu_pairs": (I, [P, P, P, I, I, I, P, L, P]),
    "chitu_b200_fp8_gemm": (I, [P, P, P, P, P, I, I, I, P, P, L, I, P]),
    "chitu_b200_soft_fp8_gemm": (I, [P, P, P, P, I, I, I, I, P, L, I, P]),
    "chitu_b200_w8a8_gemm": (I, [P, P, P, P, P, P, I, I, I, P, L, I, P]),
    "chitu_b200_w4a16_gemm": (I, [P, P, P, P, P, P, I, I, I, I, P, L, P]),
    "chitu_b200_w4a16_gemm_silu_pairs": (I, [P, P, P, P, P, I, I, I, I, P, L, P]),
    "chitu_b200_fp8_rowwise_gemm": (I, [P, P, P, P, P, P, P, I, I, I, P, L, P]),
    "chitu_b200_fp8_rowwise_gemm_silu_pairs": (I, [P, P, P, P, P, I, I, I, P, L, P]),
    "chitu_b200_attn_workspace_bytes": (L, [I, I, I, I]),
    "chitu_b200_gqa_paged_decode": (I, [P, P, P, P, P, L, L, P, P, I, I, I, I, I, I, I, F, P, P, L, I, P]),
    "chitu_b200_gqa_paged_decode_rope": (I, [P, L, P, P, P, P, L, L, P, P, P, P, I, I, I, I, I, I, I, F, P, P, L, I, P]),
    "chitu_b200_gqa_paged_prefill": (I, [P, P, P, P, P, L, L, L, L, P, P, I, I, I, I, I, I, I, I, I, I, F, P, P, L, I,
                                         P]),
    "chitu_b200_gqa_contiguous_attn": (I, [P, P, P, L, I, P, P, L, L, L, L, P, I, I, I, I, I, I, I, F, P, P, L, I, P]),
    "chitu_b200_gqa_paged_attn_fp8kv": (I, [P, L, P, P, P, P, L, L, L, L, P, P, P, P, I, I, I, I, I, I, I, I, I, I, F, P,
                                            P, L, I, P]),
    "chitu_b200_mla_decode": (I, [P, P, P, P, P, P, I, I, I, I, I, I, I, I, F, P, P, L, P]),
    "chitu_b200_mla_prefill": (I, [P, P, L, P, L, P, P, I, I, I, I, I, I, F, P, P]),
    "chitu_b200_mla_paged_prefill": (I, [P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, F, P, P, L, P]),
    "chitu_b200_mla_attn_fp8kv": (I, [P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, F, P, P, L, P]),
    "chitu_b200_debug_timeline": (I, [P]),
    "chitu_b200_debug_timeline_names": (c_char_p, []),
    "chitu_b200_debug_comm_push_area": (I, [P, P, P, P]),
    "chitu_b200_decode_prepare": (I, [P, P, P, I, P, P, P, I, I, I, P]),
    "chitu_b200_attn_plan": (I, [P, I, I, I, I, P, L, P]),
    "chitu_b200_mla_num_splits": (I, [I, I, I, L]),
    "chitu_b200_mla_absorb_o_quant": (I, [P, P, P, P, P, I, I, I, I, I, P]),
    "chitu_b200_mla_absorb_o_merge_quant": (I, [P, L, I, P, P, P, P, P, I, I, I, I, I, P]),
    "chitu_b200_mla_prep": (I, [P, P, L, P, P, P, P, P, P, P, I, I, I, I, I, I, F, P]),
    "chitu_b200_moe_workspace_bytes": (L, [I, I, I, I, I]),
    "chitu_b200_fused_experts": (I, [P, P, P, P, P, P, I, P, I, I, I, I, I, I, I, P, P, P, L, P]),
    "chitu_b200_fused_experts_w4a16": (I, [P, P, P, P, P, P, P, P, I, P, I, I, I, I, I, I, P, P, P, L, P]),
    "chitu_b200_moe_grouped_gemm_workspace_bytes": (L, [I, I, I]),
    "chitu_b200_moe_grouped_gemm": (I, [P, P, P, P, P, I, P, P, P, I, I, I, I, I, I, I, I, I, P, L, P]),
    "chitu_b200_comm_create": (I, [I, I, L, P, P]),
    "chitu_b200_comm_connect": (I, [P, P]),
    "chitu_b200_comm_destroy": (I, [P]),
    "chitu_b200_comm_status": (I, [P]),
    "chitu_b200_fp8_gemm_ar": (I, [P, P, P, P, I, I, I, P, P, L, P]),
    "chitu_b200_linear_bf16_ar": (I, [P, P, I, I, I, P, P, L, P]),
    "chitu_b200_fused_experts_ar": (I, [P, P, P, P, P, P, I, P, I, I, I, I, I, I, I, P, P, L, P]),
    "chitu_b200_allreduce_consume": (I, [P, P, P, P, P, P, P, I, I, F, P]),
    "chitu_b200_allreduce_residual_rmsnorm": (I, [P, P, P, P, P, P, P, P, I, I, F, P]),
    "chitu_b200_sample_top_k_top_p": (I, [P, L, I, I, I, P, P, P, P, P, P, P, P]),
    "chitu_b200_spec_accept_greedy": (I, [P, P, P, P, P, P, P, I, I, P]),
    "chitu_b200_spec_accept_sampled_workspace_bytes": (L, [I, I]),
    "chitu_b200_spec_accept_sampled": (I, [P, L, I, I, P, P, P, P, P, P, L, P, P, P, P, P, P, I, I, P, L, P]),
    "chitu_b200_embedding": (I, [P, P, P, I, I, L, L, I, P]),
    "chitu_b200_add": (I, [P, P, P, L, I, P]),
    "chitu_b200_argmax": (I, [P, P, I, L, I, P]),
}


def build(verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into chitu_b200/libchitu_b200.so (nvcc cross-compiles
    without a GPU)."""
    res = subprocess.run(["make", "-C", CSRC_DIR, "-j8"], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("building libchitu_b200.so failed:\n" + res.stdout[-4000:] + res.stderr[-4000:])
    if verbose:
        print(res.stdout[-2000:])
    return LIB_PATH


def load():
    """Load the library (once). Raises RuntimeError when it is missing — no CPU fallback exists."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(the CUDA extension is mandatory; there is no fallback path)"
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().chitu_b200_last_error().decode(errors="replace")
        raise RuntimeError(f"libchitu_b200 {what} failed (status {rc}): {msg}")


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def dtype_code(dt):
    import torch

    table = {
        torch.bfloat16: CB_BF16,
        torch.float16: CB_F16,
        torch.float32: CB_F32,
        torch.float8_e4m3fn: CB_FP8_E4M3,
        torch.int8: CB_I8,
        torch.uint8: CB_U8,
        torch.int16: CB_I16,
        torch.int32: CB_I32,
        torch.int64: CB_I64,
    }
    if dt not in table:
        raise TypeError(f"unsupported dtype {dt}")
    return table[dt]


def current_stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("chitu_b200 operators run on CUDA tensors only (no CPU fallback)")


def launch_count() -> int:
    return int(load().chitu_b200_launch_count())
