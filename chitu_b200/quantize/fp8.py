"""FP8 (e4m3) W8A8 linears with a per-output-channel weight scale and a per-token activation scale: the format of
vLLM / compressed-tensors `FP8` and `FP8_DYNAMIC` checkpoints and of fbgemm's rowwise FP8 (Meta's Llama-3.1 FP8
releases).

The device layout of a weight W[N, K] (include/chitu_b200.h, chitu_b200_fp8_rowwise_gemm):
  weight e4m3 [N, K] row-major;   weight_scale fp32 [N];   W[n, k] = weight[n, k] * weight_scale[n].
Activations are quantised per token by `quant_act_fp8` (vLLM QuantFP8(GroupShape.PER_TOKEN).forward_native), the
tensor cores multiply the two e4m3 operands, every 128 K-elements are added into an fp32 accumulator, and
y = bf16((acc * a_s[m]) * weight_scale[n] (+ bias)).  `forward` runs the sm_90a kernels; there is no other path."""
from __future__ import annotations

import torch
from torch import nn

from .. import _lib, workspace
from .._lib import check, current_stream, ptr

E4M3 = torch.float8_e4m3fn
FP8_MAX = 448.0
MIN_SCALE = 1.0 / (FP8_MAX * 512.0)     # vLLM's _FP8_MIN_SCALING_FACTOR: the scale of an all-zero row
ALIGN = 16                              # K multiple: the TMA row pitch of the e4m3 operands


def _check_k(K):
    if K % ALIGN != 0:
        raise ValueError(f"FP8 rowwise linears need in_features % {ALIGN} == 0, not {K}")


def _cuda_scalar(v, device):
    """None, a float or a one-element tensor -> None or an fp32 [1] tensor on `device`."""
    if v is None:
        return None
    t = torch.as_tensor(v, dtype=torch.float32).reshape(-1)
    if t.numel() != 1:
        raise ValueError(f"a static activation scale or an upper bound is one value, not {t.numel()}")
    return t.to(device)


@torch.no_grad()
def quant_act_fp8(x: torch.Tensor, scale=None, scale_ub=None):
    """Per-token e4m3 quantisation of bf16 x [..., K] -> (q e4m3 [..., K], s fp32 [rows]), rows = x.numel() // K.
    Dynamic (scale None): s = max(min(max|x_row|, scale_ub) / 448, 1 / (448 * 512)); static: s = scale for every row.
    q = e4m3(clamp(x * (1 / s), +-448)).  One launch of chitu_b200_quant_fp8_rowwise."""
    if x.dtype != torch.bfloat16:
        raise ValueError(f"quant_act_fp8 takes bf16 activations, not {x.dtype}")
    if not x.is_cuda:
        raise ValueError("quant_act_fp8 runs on CUDA tensors only")
    if scale is not None and scale_ub is not None:
        raise ValueError("quant_act_fp8: an upper bound belongs to the dynamic mode, not to a static scale")
    K = x.shape[-1]
    _check_k(K)
    x2 = x.reshape(-1, K).contiguous()
    q = torch.empty(x2.shape, dtype=E4M3, device=x.device)
    s = torch.empty(x2.shape[0], dtype=torch.float32, device=x.device)
    sc, ub = _cuda_scalar(scale, x.device), _cuda_scalar(scale_ub, x.device)
    check(_lib.load().chitu_b200_quant_fp8_rowwise(ptr(x2), ptr(q), ptr(s), x2.shape[0], K, ptr(sc), ptr(ub),
                                                   current_stream()), "quant_fp8_rowwise")
    return q.view(x.shape), s


@torch.no_grad()
def quantize_weight(w: torch.Tensor):
    """Per-output-channel e4m3 quantisation of a float weight [N, K]: s[n] = max|w[n]| / 448 in fp32 (1 for an all-zero
    row), q = e4m3_rn(clamp(w / s, +-448)).  Returns (q e4m3 [N, K], s fp32 [N]) on w's device."""
    _check_k(w.shape[-1])
    wf = w.float()
    amax = wf.abs().amax(dim=-1)
    s = amax / torch.full_like(amax, FP8_MAX)          # a tensor divisor: IEEE division on every device
    s = torch.where(s > 0, s, torch.ones_like(s))
    q = (wf / s[:, None]).clamp_(-FP8_MAX, FP8_MAX).to(E4M3)
    return q.contiguous(), s.contiguous()


def dequantize(q, s):
    """The weight W = q * s[n], fp32 [N, K] (one rounding; the kernel never forms W, it scales the fp32 sum)."""
    return q.float() * s.float()[:, None]


class Fp8Linear(nn.Module):
    """y = x W^T (+ bias) with W as e4m3 [N, K] and a per-channel fp32 scale, x bf16 [..., K] quantised per token.

    Buffers: weight e4m3 [N, K], weight_scale fp32 [N], input_scale fp32 [1] (static activation scale) or None,
    input_scale_ub fp32 [1] (upper bound of the dynamic scale's amax) or None, bias bf16 [N] or None."""

    def __init__(self, in_features, out_features, bias=False):
        super().__init__()
        _check_k(in_features)
        self.in_features, self.out_features = in_features, out_features
        self.register_buffer("weight", torch.zeros(out_features, in_features, dtype=E4M3))
        self.register_buffer("weight_scale", torch.ones(out_features, dtype=torch.float32))
        self.register_buffer("input_scale", None)
        self.register_buffer("input_scale_ub", None)
        self.register_buffer("bias", torch.zeros(out_features, dtype=torch.bfloat16) if bias else None)

    @torch.no_grad()
    def forward(self, x):
        if x.dtype != torch.bfloat16:
            raise ValueError(f"Fp8Linear runs bf16 activations, not {x.dtype}")
        tensors = (x, self.weight, self.weight_scale, self.input_scale, self.input_scale_ub, self.bias)
        if not all(t.is_cuda for t in tensors if t is not None):
            raise ValueError("Fp8Linear runs on CUDA tensors only (no CPU fallback)")
        lead, K, N = tuple(x.shape[:-1]), self.in_features, self.out_features
        if x.shape[-1] != K:
            raise ValueError(f"Fp8Linear({K}, {N}) got inputs of width {x.shape[-1]}")
        q, s = quant_act_fp8(x, self.input_scale, self.input_scale_ub)
        M = s.shape[0]
        y = torch.empty(M, N, dtype=torch.bfloat16, device=x.device)
        lib = _lib.load()
        ws = workspace.get("linear", lib.chitu_b200_linear_workspace_bytes(max(M, 1), N), x.device)
        check(lib.chitu_b200_fp8_rowwise_gemm(ptr(q), ptr(s), ptr(self.weight), ptr(self.weight_scale), ptr(self.bias),
                                              None, ptr(y), M, N, K, ptr(ws), ws.numel(), current_stream()),
              "fp8_rowwise_gemm")
        return y.view(*lead, N)

    def dequantized_weight(self):
        """W [N, K] fp32, q * s rounded once (`dequantize`)."""
        return dequantize(self.weight, self.weight_scale)

    @classmethod
    def _from_layout(cls, weight, weight_scale, bias=None, input_scale=None, input_scale_ub=None):
        if weight.dtype != E4M3:
            raise ValueError(f"Fp8Linear takes e4m3 (torch.float8_e4m3fn) weights, not {weight.dtype}")
        if weight.dim() != 2:
            raise ValueError(f"Fp8Linear takes a 2-D weight, not {tuple(weight.shape)}")
        N, K = weight.shape
        ws = torch.as_tensor(weight_scale).to(device=weight.device, dtype=torch.float32)
        if ws.numel() == 1:                                  # per-tensor scale: the same for every channel
            ws = ws.reshape(1).expand(N)
        elif tuple(ws.shape) not in ((N,), (N, 1)):
            raise ValueError(f"weight_scale must be [N, 1], [N] or one value for N = {N}, not {tuple(ws.shape)}")
        m = cls(K, N, bias=bias is not None)
        m.weight = weight.contiguous()
        m.weight_scale = ws.reshape(N).contiguous()
        if bias is not None:
            m.bias = bias.to(device=weight.device, dtype=torch.bfloat16).contiguous()
        m.input_scale = _cuda_scalar(input_scale, weight.device)
        m.input_scale_ub = _cuda_scalar(input_scale_ub, weight.device)
        return m

    @classmethod
    @torch.no_grad()
    def from_float(cls, linear):
        """Per-channel e4m3 quantisation (`quantize_weight`) of an nn.Linear; activations quantised dynamically."""
        q, s = quantize_weight(linear.weight.detach())
        return cls._from_layout(q, s, None if linear.bias is None else linear.bias.detach())

    @classmethod
    @torch.no_grad()
    def from_compressed_tensors(cls, weight, weight_scale, input_scale=None, bias=None):
        """compressed-tensors `FP8` (static: input_scale is the per-tensor activation scale) and `FP8_DYNAMIC`
        (input_scale None): weight e4m3 [N, K], weight_scale [N, 1] (channel strategy), [N] or one value (tensor
        strategy, expanded to every channel)."""
        return cls._from_layout(weight, weight_scale, bias, input_scale=input_scale)

    @classmethod
    @torch.no_grad()
    def from_fbgemm(cls, weight, weight_scale, input_scale_ub=None, bias=None):
        """fbgemm rowwise FP8 (Llama-3.1 FP8): weight e4m3 [N, K], weight_scale fp32 [N, 1], input_scale_ub the upper
        bound on each token's amax (dynamic per-token activation scales)."""
        return cls._from_layout(weight, weight_scale, bias, input_scale_ub=input_scale_ub)

    def extra_repr(self):
        mode = "static" if self.input_scale is not None else "dynamic"
        return f"{self.in_features}, {self.out_features}, bias={self.bias is not None}, activations={mode}"
