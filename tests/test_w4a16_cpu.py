"""W4A16 without a GPU: the GPTQ / AWQ repacks into the device layout (chitu_b200/quantize/w4a16.py) against each
format's own dequantisation written out from its bit positions, the refusals of the Python constructors, and the
argument checks of the two C entries (chitu_b200_w4a16_gemm[_silu_pairs]), which refuse before touching the device."""
import numpy as np
import pytest
import torch

from chitu_b200.quantize import W4A16Linear
from chitu_b200.quantize import w4a16 as W

F16 = torch.float16


def _edge_ints(shape, gen):
    """Random 0..15 with the first row and column pinned to the extremes 0 and 15."""
    v = torch.randint(0, 16, shape, generator=gen, dtype=torch.int64)
    v[0, :] = 0
    v[:, 0] = 15
    v[-1, -1] = 0
    return v


def _pack_u32(nibbles):
    """[..., 8] nibbles -> int32 words with nibble i at bits 4i (bit 31 set where nibble 7 >= 8)."""
    n = nibbles.numpy().astype(np.uint32)
    w = np.zeros(n.shape[:-1], dtype=np.uint32)
    for i in range(8):
        w |= n[..., i] << np.uint32(4 * i)
    return torch.from_numpy(w.view(np.int32))


def _scales(shape, gen):
    return (torch.rand(shape, generator=gen) * 0.02 + 1e-3).to(F16)


def _gptq_tensors(K, N, seed):
    """AutoGPTQ's layout written from its bit positions.  q [K, N], zero [K/128, N] in 0..15; qzeros stores
    (zero - 1) & 15 (zero 0 wraps to 15)."""
    g = torch.Generator().manual_seed(seed)
    q, z, s = _edge_ints((K, N), g), _edge_ints((K // 128, N), g), _scales((K // 128, N), g)
    qweight = _pack_u32(q.view(K // 8, 8, N).permute(0, 2, 1))                 # element 8r + i of column n: bits 4i
    qzeros = _pack_u32(((z - 1) & 15).view(K // 128, N // 8, 8))               # packed along N, natural order
    return q, z, s, qweight, qzeros


def _gptq_dequant(qweight, qzeros, scales):
    """The GPTQ format's own dequantisation: w[k, n] = fp16((q - ((stored zero + 1) & 15)) * s), as [N, K]."""
    K, N = qweight.shape[0] * 8, qweight.shape[1]
    qw = qweight.numpy().view(np.uint32)
    qz = qzeros.numpy().view(np.uint32)
    q = np.zeros((K, N), dtype=np.int64)
    for k in range(K):
        q[k] = (qw[k // 8] >> np.uint32(4 * (k % 8))) & 15
    z = np.zeros((K // 128, N), dtype=np.int64)
    for n in range(N):
        z[:, n] = ((qz[:, n // 8] >> np.uint32(4 * (n % 8))) & 15) + 1
    z &= 15
    zk = np.repeat(z, 128, axis=0)
    sk = np.repeat(scales.float().numpy(), 128, axis=0)
    return torch.from_numpy(((q - zk) * sk).astype(np.float32)).to(F16).T.contiguous()


AWQ_ORDER = [0, 2, 4, 6, 1, 3, 5, 7]


def _awq_tensors(K, N, seed):
    g = torch.Generator().manual_seed(seed)
    q, z, s = _edge_ints((K, N), g), _edge_ints((K // 128, N), g), _scales((K // 128, N), g)
    qweight = _pack_u32(q.view(K, N // 8, 8)[:, :, AWQ_ORDER])                 # nibble i = column 8c + ORDER[i]
    qzeros = _pack_u32(z.view(K // 128, N // 8, 8)[:, :, AWQ_ORDER])
    return q, z, s, qweight, qzeros


def _awq_dequant(qweight, qzeros, scales):
    """AWQ's own dequantisation: w[k, n] = fp16((q - z) * s), nibbles in the order [0, 2, 4, 6, 1, 3, 5, 7]."""
    K, N = qweight.shape[0], qweight.shape[1] * 8
    qw, qz = qweight.numpy().view(np.uint32), qzeros.numpy().view(np.uint32)
    q = np.zeros((K, N), dtype=np.int64)
    z = np.zeros((K // 128, N), dtype=np.int64)
    for i, col in enumerate(AWQ_ORDER):
        q[:, col::8] = (qw >> np.uint32(4 * i)) & 15
        z[:, col::8] = (qz >> np.uint32(4 * i)) & 15
    zk, sk = np.repeat(z, 128, axis=0), np.repeat(scales.float().numpy(), 128, axis=0)
    return torch.from_numpy(((q - zk) * sk).astype(np.float32)).to(F16).T.contiguous()


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("K,N", [(128, 8), (384, 64), (1024, 200)])
def test_gptq_repack_matches_the_format_dequant(K, N):
    q, z, s, qweight, qzeros = _gptq_tensors(K, N, seed=K + N)
    m = W4A16Linear.from_gptq(qweight, qzeros, s, g_idx=torch.arange(K, dtype=torch.int32) // 128)
    assert m.qweight.shape == (N, K // 2) and m.qweight.dtype == torch.uint8
    assert m.scales.shape == (N, K // 128) and m.scales.dtype == F16 and m.zeros.dtype == torch.uint8
    assert torch.equal(W.unpack_rows(m.qweight).long(), q.T)
    assert torch.equal(m.zeros.long(), z.T)                                   # the zero - 1 convention undone
    assert int(m.zeros.min()) == 0 and int(m.zeros.max()) == 15
    assert _same_bits(m.dequantized_weight(), _gptq_dequant(qweight, qzeros, s))


@pytest.mark.parametrize("K,N", [(128, 8), (384, 64), (1024, 200)])
def test_awq_repack_matches_the_format_dequant(K, N):
    q, z, s, qweight, qzeros = _awq_tensors(K, N, seed=3 * K + N)
    m = W4A16Linear.from_awq(qweight, qzeros, s)
    assert torch.equal(W.unpack_rows(m.qweight).long(), q.T)
    assert torch.equal(m.zeros.long(), z.T)
    assert _same_bits(m.dequantized_weight(), _awq_dequant(qweight, qzeros, s))


def test_nibble_orders_agree_with_vllm():
    """vLLM's gptq_pack / awq_pack are an independent statement of the two packings."""
    qu = pytest.importorskip("vllm.model_executor.layers.quantization.utils.quant_utils")
    K, N = 256, 64
    q, z, s, qweight, qzeros = _gptq_tensors(K, N, seed=5)
    assert torch.equal(qu.gptq_pack(q.to(torch.int32), 4, K, N), qweight)
    q, z, s, qweight, qzeros = _awq_tensors(K, N, seed=6)
    assert torch.equal(qu.awq_pack(q.to(torch.int32), 4, K, N), qweight)
    assert torch.equal(qu.awq_pack(z.to(torch.int32), 4, K // 128, N), qzeros)


def test_device_layout_packs_even_k_low():
    q = torch.tensor([[1, 2, 15, 0]], dtype=torch.uint8)
    assert W.pack_rows(q).tolist() == [[0x21, 0x0F]]
    assert torch.equal(W.unpack_rows(W.pack_rows(q)), q)


@pytest.mark.parametrize("dtype", [torch.bfloat16, F16])
def test_from_float_round_to_nearest(dtype):
    """from_float: every dequantised element within one quantisation step of the input (half a step from rounding q,
    up to half more where the rounded zero shifts the group's grid past its extreme), the io rounding on top."""
    g = torch.Generator().manual_seed(1)
    lin = torch.nn.Linear(256, 48, bias=True)
    with torch.no_grad():
        lin.weight.copy_(torch.randn(48, 256, generator=g) * 0.05)
        lin.weight[3, :128] = 0.25                                               # a constant group
    m = W4A16Linear.from_float(lin, dtype)
    assert m.scales.dtype == dtype and m.bias.dtype == dtype and m.dtype == dtype
    w = m.dequantized_weight().float()
    step = m.scales.float().repeat_interleave(128, dim=1)
    err = (w - lin.weight.detach().float()).abs()
    assert bool((err <= step * (1 + 2 ** -6) + 2 ** -8 * lin.weight.detach().abs().float()).all())
    assert float(err.mean()) < 0.3 * float(step.mean())


# ------------------------------------------------------------------------------------------------------- refusals
def test_act_order_and_group_size_are_refused():
    K, N = 256, 16
    _, _, s, qweight, qzeros = _gptq_tensors(K, N, seed=9)
    act_order = torch.arange(K, dtype=torch.int32).flip(0) // 128
    with pytest.raises(ValueError, match="act-order"):
        W4A16Linear.from_gptq(qweight, qzeros, s, g_idx=act_order)
    s64 = s.repeat_interleave(2, dim=0)                                          # 4 groups of 64
    with pytest.raises(ValueError, match="groups of 128"):
        W4A16Linear.from_gptq(qweight, qzeros, s64)
    _, _, s, qweight, qzeros = _awq_tensors(K, N, seed=10)
    with pytest.raises(ValueError, match="groups of 128"):
        W4A16Linear.from_awq(qweight, qzeros, s64)


def test_k_not_a_multiple_of_128_is_refused():
    with pytest.raises(ValueError):
        W4A16Linear(200, 64)
    with pytest.raises(ValueError):
        W.quantize_rtn(torch.randn(8, 192))
    with pytest.raises(ValueError):
        W4A16Linear.from_gptq(torch.zeros(24, 8, dtype=torch.int32), torch.zeros(2, 1, dtype=torch.int32),
                              torch.ones(2, 8, dtype=F16))                       # K = 192


def test_cpu_tensors_raise():
    m = W4A16Linear(128, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(2, 128, dtype=torch.bfloat16))


def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def test_c_entries_refuse_bad_arguments_and_launch_nothing():
    from chitu_b200._lib import CB_BF16, CB_F16, CB_F32, launch_count
    lib = _lib()
    A = 1 << 20                                  # 16-byte aligned stand-ins: every case is refused before a dereference
    x, qw, sc, zr, y, ws = A, 2 * A, 3 * A, 4 * A, 5 * A, 6 * A

    def plain(**kw):
        a = dict(x=x, qw=qw, sc=sc, zr=zr, res=None, y=y, M=4, N=64, K=256, dtype=CB_BF16)
        a.update(kw)
        return lib.chitu_b200_w4a16_gemm(a["x"], a["qw"], a["sc"], a["zr"], a["res"], a["y"], a["M"], a["N"], a["K"],
                                         a["dtype"], ws, 1 << 20, None), "chitu_b200_w4a16_gemm"

    def pairs(**kw):
        a = dict(x=x, qw=qw, sc=sc, zr=zr, y=y, M=4, N=64, K=256, dtype=CB_BF16)
        a.update(kw)
        return lib.chitu_b200_w4a16_gemm_silu_pairs(a["x"], a["qw"], a["sc"], a["zr"], a["y"], a["M"], a["N"], a["K"],
                                                    a["dtype"], ws, 1 << 20, None), "chitu_b200_w4a16_gemm_silu_pairs"

    before = launch_count()
    bad = [dict(x=None), dict(qw=None), dict(sc=None), dict(zr=None), dict(y=None), dict(x=x + 8), dict(qw=qw + 4),
           dict(sc=sc + 2), dict(zr=zr + 1), dict(y=y + 8), dict(K=192), dict(K=64), dict(dtype=CB_F32),
           dict(dtype=7), dict(M=-1), dict(N=0)]
    for call in (plain, pairs):
        for kw in bad:
            rc, name = call(**kw)
            assert rc < 0, (name, kw)
            assert name in lib.chitu_b200_last_error().decode(), (name, kw)
    for kw in (dict(res=A + 8),):
        rc, name = plain(**kw)
        assert rc < 0 and name in lib.chitu_b200_last_error().decode()
    rc, name = pairs(N=66 + 1)
    assert rc < 0 and name in lib.chitu_b200_last_error().decode()
    for call in (plain, pairs):                  # M = 0: nothing to do, fp16 too
        for dt in (CB_BF16, CB_F16):
            assert call(M=0, dtype=dt)[0] == 0
    assert launch_count() == before


def test_engine_refuses_w4a16_with_a_process_group():
    from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
    with pytest.raises(ValueError, match="w4a16"):
        LlamaDecodeEngine(LLAMA3_8B, max_reqs=1, max_seq_len=256, device="cpu", tp_size=2, process_group=object(),
                          weight_format="w4a16")
    with pytest.raises(ValueError, match="weight_format"):
        LlamaDecodeEngine(LLAMA3_8B, max_reqs=1, max_seq_len=256, device="cpu", weight_format="int3")
