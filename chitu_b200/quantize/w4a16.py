"""4-bit weight-only linears (W4A16, groups of 128 along K) for GPTQ / AWQ checkpoints.

The device layout of a weight W[N, K] (include/chitu_b200.h, chitu_b200_w4a16_gemm):
  qweight uint8 [N, K/2]: element k of row n in byte k/2, low nibble for even k, high nibble for odd k;
  scales  [N, K/128] in the io dtype;   zeros uint8 [N, K/128], 0..15.
The weight element is io((q - z) * s), one rounding; the GEMM accumulates in fp32 and rounds once to the io dtype.

`from_gptq` / `from_awq` repack the two checkpoint layouts into it and `from_float` quantises a float weight; all three
are host torch, run once at load time.  `forward` runs the sm_90a kernel; there is no other path.  `pack_experts` stacks
per-expert modules into the layout of `fused_moe.fused_experts(use_int4_w4a16=True)`."""
from __future__ import annotations

import torch
from torch import nn

from .. import _lib, workspace
from .._lib import check, current_stream, dtype_code, ptr, require_cuda

GROUP = 128
_AWQ_ORDER = (0, 2, 4, 6, 1, 3, 5, 7)      # AWQ GEMM packing: nibble i of a word holds column 8c + _AWQ_ORDER[i]


def _check_k(K):
    if K % GROUP != 0:
        raise ValueError(f"W4A16 needs in_features % {GROUP} == 0, not {K}")


def _group_size(K, groups):
    if groups * GROUP != K:
        raise ValueError(f"W4A16 is built for groups of {GROUP} only: {K} inputs in {groups} groups")


def pack_rows(q):
    """q [N, K] integers 0..15 -> the device's uint8 [N, K/2] (even k in the low nibble)."""
    q = q.to(torch.uint8)
    return (q[:, 0::2] | (q[:, 1::2] << 4)).contiguous()


def unpack_rows(qweight):
    """The device's uint8 [..., N, K/2] -> q [..., N, K] (uint8, 0..15)."""
    lo, hi = qweight & 0xF, qweight >> 4
    return torch.stack((lo, hi), dim=-1).reshape(*qweight.shape[:-1], -1)


def dequantize(qweight, scales, zeros):
    """The element values the kernel multiplies: io((q - z) * s) [..., N, K] in scales' dtype (leading dims: a stack of
    experts; zeros None: every zero is 8).  (q - z) * s is exact in fp32 (a 5-bit integer times a 16-bit float), so the
    cast is the one rounding."""
    q = unpack_rows(qweight).float()
    z = 8.0 if zeros is None else zeros.float().repeat_interleave(GROUP, dim=-1)
    s = scales.float().repeat_interleave(GROUP, dim=-1)
    return ((q - z) * s).to(scales.dtype)


@torch.no_grad()
def quantize_rtn(w, dtype=torch.bfloat16):
    """Round-to-nearest asymmetric group-128 quantisation of a float weight [N, K] (GPTQ's min / max quantiser without
    the error feedback): per row and group, with lo = min(min w, 0) and hi = max(max w, 0),
    s = io(max(hi - lo, 1e-4 * 15) / 15), z = clamp(round(-lo / s), 0, 15), q = clamp(round(w / s) + z, 0, 15).
    Returns (qweight, scales, zeros) in the device layout."""
    N, K = w.shape
    _check_k(K)
    g = w.float().reshape(N, K // GROUP, GROUP)
    lo, hi = g.amin(dim=-1).clamp(max=0), g.amax(dim=-1).clamp(min=0)
    s = ((hi - lo).clamp(min=1e-4 * 15) / 15).to(dtype)
    sf = s.float()
    z = torch.round(-lo / sf).clamp_(0, 15)
    q = (torch.round(g / sf[..., None]) + z[..., None]).clamp_(0, 15)
    return pack_rows(q.reshape(N, K)), s.contiguous(), z.to(torch.uint8).contiguous()


def _unpack_cols(packed, order=None):
    """int32 [R, C/8] packed along the columns (column 8c + order[i] in bits 4i; order None = natural) -> [R, C]."""
    order = tuple(range(8)) if order is None else order
    shifts = torch.empty(8, dtype=torch.int32)
    for i, col in enumerate(order):
        shifts[col] = 4 * i
    shifts = shifts.to(packed.device)
    vals = (packed.to(torch.int32)[:, :, None] >> shifts) & 0xF
    return vals.reshape(packed.shape[0], -1)


class W4A16Linear(nn.Module):
    """y = x W^T (+ bias) with W held as 4-bit groups of 128 (see the module docstring); x [..., K] in `dtype`."""

    def __init__(self, in_features, out_features, bias=True, dtype=torch.bfloat16):
        super().__init__()
        _check_k(in_features)
        if dtype not in (torch.bfloat16, torch.float16):
            raise ValueError(f"W4A16Linear runs bf16 or fp16 activations, not {dtype}")
        self.in_features, self.out_features, self.dtype = in_features, out_features, dtype
        G = in_features // GROUP
        self.register_buffer("qweight", torch.zeros(out_features, in_features // 2, dtype=torch.uint8))
        self.register_buffer("scales", torch.ones(out_features, G, dtype=dtype))
        self.register_buffer("zeros", torch.full((out_features, G), 8, dtype=torch.uint8))
        self.register_buffer("bias", torch.zeros(out_features, dtype=dtype) if bias else None)

    @torch.no_grad()
    def forward(self, x):
        require_cuda(x, self.qweight, self.scales, self.zeros, self.bias)
        if x.dtype != self.dtype:
            raise TypeError(f"W4A16Linear({self.dtype}) got {x.dtype} activations")
        lead = tuple(x.shape[:-1])
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        M, N, K = x2.shape[0], self.out_features, self.in_features
        y = torch.empty(M, N, dtype=self.dtype, device=x.device)
        lib = _lib.load()
        ws = workspace.get("linear", lib.chitu_b200_linear_workspace_bytes(max(M, 1), N), x.device)
        check(lib.chitu_b200_w4a16_gemm(ptr(x2), ptr(self.qweight), ptr(self.scales), ptr(self.zeros), None, ptr(y), M,
                                        N, K, dtype_code(self.dtype), ptr(ws), ws.numel(), current_stream()),
              "w4a16_gemm")
        y = y.view(*lead, N)
        if self.bias is not None:
            y += self.bias
        return y

    def dequantized_weight(self):
        """W [N, K] in the io dtype: the exact element values the kernel multiplies."""
        return dequantize(self.qweight, self.scales, self.zeros)

    @classmethod
    def _from_layout(cls, qweight, scales, zeros, bias):
        N, K = qweight.shape[0], qweight.shape[1] * 2
        m = cls(K, N, bias=bias is not None, dtype=scales.dtype)
        m.qweight, m.scales, m.zeros = qweight.contiguous(), scales.contiguous(), zeros.to(torch.uint8).contiguous()
        if bias is not None:
            m.bias = bias.to(scales.dtype).contiguous()
        return m

    @classmethod
    @torch.no_grad()
    def from_float(cls, linear, dtype=torch.bfloat16):
        """Round-to-nearest group-128 asymmetric quantisation (`quantize_rtn`) of an nn.Linear."""
        q, s, z = quantize_rtn(linear.weight.detach(), dtype)
        return cls._from_layout(q, s, z, None if linear.bias is None else linear.bias.detach())

    @classmethod
    @torch.no_grad()
    def from_gptq(cls, qweight, qzeros, scales, g_idx=None, bias=None):
        """AutoGPTQ's layout: qweight int32 [K/8, N] packed along K (element 8r + i of column n in bits 4i of
        qweight[r, n]), qzeros int32 [K/128, N/8] packed along N storing zero - 1 (read back as (v + 1) & 15, as
        AutoGPTQ's kernels do), scales fp16 [K/128, N].  Act-order (a g_idx other than k // 128) is refused."""
        K, N = qweight.shape[0] * 8, qweight.shape[1]
        _check_k(K)
        _group_size(K, scales.shape[0])
        if g_idx is not None and not torch.equal(g_idx.to(torch.int64).cpu(), torch.arange(K) // GROUP):
            raise ValueError("act-order GPTQ (g_idx other than k // 128) is not supported")
        q = _unpack_cols(qweight.T.contiguous()).reshape(N, K)        # [N, K/8] words along K -> [N, K]
        z = (_unpack_cols(qzeros)[:, :N] + 1) & 0xF                     # [K/128, N]
        return cls._from_layout(pack_rows(q), scales.T.contiguous(), z.T.contiguous(), bias)

    @classmethod
    @torch.no_grad()
    def from_awq(cls, qweight, qzeros, scales, bias=None):
        """AWQ's GEMM layout: qweight int32 [K, N/8] and qzeros int32 [K/128, N/8], both packed along N with nibble i
        holding column 8c + [0, 2, 4, 6, 1, 3, 5, 7][i]; scales fp16 [K/128, N]."""
        K, N = qweight.shape[0], qweight.shape[1] * 8
        _check_k(K)
        _group_size(K, scales.shape[0])
        q = _unpack_cols(qweight, _AWQ_ORDER)                           # [K, N]
        z = _unpack_cols(qzeros, _AWQ_ORDER)                            # [K/128, N]
        return cls._from_layout(pack_rows(q.T), scales.T.contiguous(), z.T.contiguous(), bias)

    def extra_repr(self):
        return f"{self.in_features}, {self.out_features}, bias={self.bias is not None}, dtype={self.dtype}"


@torch.no_grad()
def pack_experts(gate, up, down):
    """Stack per-expert W4A16Linear modules (from `from_gptq` / `from_awq` / `from_float`) into the expert layout of
    `fused_moe.fused_experts(use_int4_w4a16=True)`: gate / up / down are lists of E modules (Mixtral's w1 / w3 / w2), and
    the result is (w1, w1_scale, w1_zp, w2, w2_scale, w2_zp) with
      w1 uint8 [E, 2F, K/2] = each expert's [gate ; up] rows,  w2 uint8 [E, K, F/2] = down,
      w*_scale bf16 [E, N, K/128],  w*_zp uint8 [E, N, K/128].
    The MoE path computes in bf16, so the scales are cast to bf16.  GPTQ and AWQ store fp16 scales: that cast is one
    rounding of each scale that the fp16 checkpoint does not have (about 2^-9 relative).  Biases are not carried (the
    expert linears of Mixtral have none); a module with a bias is refused."""
    if not (len(gate) == len(up) == len(down)) or not gate:
        raise ValueError(f"pack_experts needs the same number (> 0) of gate, up and down modules, not "
                         f"{len(gate)}, {len(up)}, {len(down)}")
    if any(m.bias is not None for m in (*gate, *up, *down)):
        raise ValueError("pack_experts: the fused experts take no bias")

    def stack(mods):
        return tuple(torch.stack([getattr(m, name) for m in mods]).contiguous() for name in ("qweight", "scales", "zeros"))

    w1 = [torch.cat(pair, dim=1) for pair in zip(stack(gate), stack(up))]
    w2 = list(stack(down))
    if w1[0].shape[-1] * 2 != w2[0].shape[1] or w2[0].shape[-1] * 4 != w1[0].shape[1]:
        raise ValueError(f"pack_experts: gate / up [{w1[0].shape[1] // 2}, {w1[0].shape[-1] * 2}] and down "
                         f"[{w2[0].shape[1]}, {w2[0].shape[-1] * 2}] do not chain")
    w1[1], w2[1] = w1[1].to(torch.bfloat16), w2[1].to(torch.bfloat16)
    return w1[0], w1[1], w1[2], w2[0], w2[1], w2[2]
