"""One-shot all-reduce over NVLink peer memory fused with residual add + RMSNorm (+ FP8 quant).

Host side only does the plumbing: create the symmetric buffer in the C library, exchange the CUDA IPC
handles with `torch.distributed.all_gather_object`, connect.  The reduce runs in csrc/comm.cu (SURVEY §5.8: 122
latency-bound all-reduces per DeepSeek step): `consume` after a product whose epilogue pushed its partial into every
rank's push area (`fp8_gemm_push`, `linear_push`, `experts_push`), `__call__` (the pull kernel `allreduce_norm_kernel`)
for a partial written by a product without that epilogue."""
from __future__ import annotations

import ctypes

import torch
import torch.distributed as dist

from . import _lib
from ._lib import check, current_stream, ptr


class FusedAllReduce:
    def __init__(self, group, max_rows: int, dim: int, device):
        self.lib = _lib.load()
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        assert self.world <= 8
        torch.cuda.set_device(device)
        self.handle = ctypes.c_void_p()
        ipc = (ctypes.c_uint8 * 128)()
        check(self.lib.chitu_b200_comm_create(self.rank, self.world, int(max_rows) * int(dim) * 2, ctypes.byref(self.handle),
                                              ipc), "comm_create")
        mine = bytes(ipc)
        gathered = [None] * self.world
        dist.all_gather_object(gathered, mine, group=group)
        blob = b"".join(gathered)
        buf = (ctypes.c_uint8 * len(blob)).from_buffer_copy(blob)
        check(self.lib.chitu_b200_comm_connect(self.handle, buf), "comm_connect")
        dist.barrier(group)

    def __call__(self, partial, residual, h_out, norm_w, y, q, q_scales, rows, dim, eps):
        check(self.lib.chitu_b200_allreduce_residual_rmsnorm(self.handle, ptr(partial), ptr(residual), ptr(h_out), ptr(norm_w),
                                                             ptr(y), ptr(q), ptr(q_scales), rows, dim, float(eps),
                                                             current_stream()), "allreduce_residual_rmsnorm")

    # ---- push mode: the producing kernel's epilogue stores its partial into every rank's push area (csrc/comm.cu) ----
    def fp8_gemm_push(self, xq, xs, w, w_s, M, lin_ws) -> None:
        """fp8 row-parallel linear whose epilogue starts the all-reduce (finish it with `consume`)."""
        N, K = w.shape
        check(self.lib.chitu_b200_fp8_gemm_ar(ptr(xq), ptr(xs), ptr(w), ptr(w_s), M, N, K, self.handle, ptr(lin_ws), lin_ws.numel(),
                                              current_stream()), "fp8_gemm_ar")

    def linear_push(self, x, w, M, lin_ws) -> None:
        N, K = w.shape
        check(self.lib.chitu_b200_linear_bf16_ar(ptr(x), ptr(w), M, N, K, self.handle, ptr(lin_ws), lin_ws.numel(),
                                                 current_stream()), "linear_bf16_ar")

    def experts_push(self, x, w1, w2, w1_s, w2_s, topk_w, topk_w_code, topk_ids, ids_code, T, topk, E, N1, K1, wmode,
                     moe_ws) -> None:
        check(self.lib.chitu_b200_fused_experts_ar(ptr(x), ptr(w1), ptr(w2), ptr(w1_s), ptr(w2_s), ptr(topk_w), topk_w_code,
                                                   ptr(topk_ids), ids_code, T, topk, E, N1, K1, wmode, self.handle, ptr(moe_ws),
                                                   moe_ws.numel(), current_stream()), "fused_experts_ar")

    def consume(self, residual, h_out, norm_w, y, q, q_scales, rows, dim, eps):
        """reduce the partials every rank pushed (same outputs as __call__)"""
        check(self.lib.chitu_b200_allreduce_consume(self.handle, ptr(residual), ptr(h_out), ptr(norm_w), ptr(y),
                                                    ptr(q), ptr(q_scales), rows, dim, float(eps), current_stream()),
              "allreduce_consume")

    def status(self) -> int:
        return int(self.lib.chitu_b200_comm_status(self.handle))

    def close(self):
        if self.handle:
            self.lib.chitu_b200_comm_destroy(self.handle)
            self.handle = None
