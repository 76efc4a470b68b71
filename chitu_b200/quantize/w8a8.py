"""Host-side drop-in for the module the reference registers under `quant=simple_w8a8` (SURVEY a17,
`chitu/quantize/w8a8.py`): `W8A8Linear` with per-channel int8 weights and per-token int8 activations.

What must match the reference so that its checkpoints and its quantizer walk (`quantize/quantizer.py:117-145`)
work unchanged: the buffer names and dtypes (`weight` int8 [N, K], `scale_channel` fp32 [N], `bias` fp16 [N] or
None), the constructor / `from_float` parameters, and the dispatch rule of `forward` ([bs <= 4, seq, K] inputs go
to `w8a8gemv.mv`, everything else to `w8a8gemm.mm`).  The arithmetic runs in the H100 kernels behind those two
shims and in `chitu_b200_quant_act_int8`."""
from __future__ import annotations

import torch
from torch import nn

from .. import _lib
from .._lib import check, current_stream, dtype_code, ptr, require_cuda
from . import w8a8gemm, w8a8gemv

_INT8_MAX = 127.0
_MIN_ABSMAX = 1e-5          # clamp of the reference's scale computation
_GEMV_MAX_BATCH = 4         # 3-D inputs with at most this many sequences take the GEMV entry point


@torch.no_grad()
def quant_act(act):
    """Per-token symmetric int8 quantisation (reference `quant_act`): scale = max(absmax, 1e-5) / 127 per row of the
    flattened [rows, K] view, q = round(x / scale).  One CUDA kernel; returns (q int8 [rows, K], scale fp32 [rows])."""
    require_cuda(act)
    rows_by_k = act.reshape(-1, act.shape[-1]).contiguous()
    n_rows, k = rows_by_k.shape
    q = torch.empty((n_rows, k), dtype=torch.int8, device=act.device)
    scale = torch.empty((n_rows,), dtype=torch.float32, device=act.device)
    check(_lib.load().chitu_b200_quant_act_int8(ptr(rows_by_k), ptr(q), ptr(scale), n_rows, k, dtype_code(act.dtype),
                                                current_stream()), "quant_act_int8")
    return q, scale


@torch.no_grad()
def quant_weight(w):
    """Per-output-channel symmetric int8 quantisation of an [N, K] weight (load time, plain torch):
    returns (int8 [N, K], fp32 scale [N]) with scale = max(absmax, 1e-5) / 127."""
    absmax = w.abs().amax(dim=-1, keepdim=True).to(torch.float32).clamp_(min=_MIN_ABSMAX)
    scale = absmax / _INT8_MAX
    return torch.round(w / scale).to(torch.int8), scale.flatten()


class W8A8Linear(nn.Module):
    def __init__(self, in_features, out_features, bias=True, quantize_output=False, pre_norm=None):
        super().__init__()
        self.in_features, self.out_features, self.pre_norm = in_features, out_features, pre_norm
        buffers = {
            "weight": torch.zeros(out_features, in_features, dtype=torch.int8),
            "scale_channel": torch.ones(out_features, dtype=torch.float32),
            "bias": torch.zeros(out_features, dtype=torch.float16) if bias else None,
        }
        for name, tensor in buffers.items():
            self.register_buffer(name, tensor)
        self.act_quant_name, self.act_quant = "per_token", quant_act
        self.output_quant_name = self.act_quant_name if quantize_output else "None"
        self.output_quant = self.act_quant if quantize_output else (lambda t: t)

    @torch.no_grad()
    def forward(self, x):
        lead = tuple(x.shape[:-1])
        q_x, tok_scale = self.act_quant(x)
        if x.dim() == 3 and lead[0] <= _GEMV_MAX_BATCH:
            y = w8a8gemv.mv(q_x.view(*lead, q_x.shape[-1]), self.weight, tok_scale, self.scale_channel)
        else:
            y = torch.empty((q_x.shape[0], self.out_features), dtype=torch.float16, device=x.device)
            w8a8gemm.mm(y, q_x, self.weight, tok_scale, self.scale_channel, None)
            y = y.view(*lead, self.out_features)
        if self.bias is not None:
            y += self.bias
        return y

    @staticmethod
    def from_float(module, weight_quant="per_channel", act_quant="per_token", quantize_output=False,
                   model_arch_only=False):
        has_bias = module.bias is not None
        q = W8A8Linear(module.in_features, module.out_features, has_bias, quantize_output=quantize_output)
        if model_arch_only:
            return q
        q.weight, q.scale_channel = quant_weight(module.weight)
        if has_bias:
            q.bias = module.bias
        return q

    def extra_repr(self):
        return f"{self.in_features}, {self.out_features}, bias={self.bias is not None}"
