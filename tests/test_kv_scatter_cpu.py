"""chitu_b200_scatter_kv without a GPU: every refusal of the C entry returns a negative status naming it before anything
is launched (fake device pointers are never dereferenced), an empty batch returns 0 without a launch, and
ops.scatter_kv_to_cache refuses CPU tensors."""
import pytest
import torch

from chitu_b200 import _lib as L
from chitu_b200 import ops

A = 4096          # a fake, 16-byte aligned device pointer


def _scatter(cache0=A, cache1=A, src0=A, src0_st=1024, src1=A, src1_st=1024, cu=A, starts=A, bt=A, bt_stride=4,
             page=256, cache_sb=0, cache_rows=0, B=2, total=8, n=1024, src_dtype=L.CB_BF16, cache_dtype=L.CB_BF16):
    return L.load().chitu_b200_scatter_kv(cache0, cache1, src0, src0_st, src1, src1_st, cu, starts, bt, bt_stride, page,
                                          cache_sb, cache_rows, B, total, n, src_dtype, cache_dtype, None)


CONTIG = dict(bt=None, bt_stride=0, page=0, cache_sb=100 * 1024, cache_rows=100)
E4M3 = dict(cache_dtype=L.CB_FP8_E4M3)

REFUSED = [
    ("null cache0", dict(cache0=None)),
    ("null src0", dict(src0=None)),
    ("null cu_seqlens", dict(cu=None)),
    ("cache1 without src1", dict(src1=None)),
    ("src1 without cache1", dict(cache1=None)),
    ("fp32 rows", dict(src_dtype=L.CB_F32, cache_dtype=L.CB_F32)),
    ("bf16 rows into an fp16 cache", dict(cache_dtype=L.CB_F16)),
    ("bf16 rows into an int8 cache", dict(cache_dtype=L.CB_I8)),
    ("e4m3 rows", dict(src_dtype=L.CB_FP8_E4M3, cache_dtype=L.CB_FP8_E4M3)),
    ("e4m3 into a contiguous cache", dict(CONTIG, **E4M3)),
    ("page_size 0", dict(page=0)),
    ("negative page_size", dict(page=-64)),
    ("bt_stride 0", dict(bt_stride=0)),
    ("e4m3 row not a multiple of 8", dict(E4M3, n=1020, src0_st=1024, src1_st=1024)),
    ("e4m3 source misaligned", dict(E4M3, src0=A + 8)),
    ("e4m3 second source misaligned", dict(E4M3, src1=A + 2)),
    ("e4m3 source stride not a multiple of 8", dict(E4M3, src0_st=1028)),
    ("e4m3 cache misaligned", dict(E4M3, cache1=A + 4)),
    ("contiguous batch stride below cache_rows x n", dict(CONTIG, cache_sb=99 * 1024)),
    ("contiguous batch stride not a multiple of n", dict(CONTIG, cache_sb=100 * 1024 + 8)),
    ("negative cache_rows", dict(CONTIG, cache_rows=-1)),
    ("negative B", dict(B=-1)),
    ("negative total_rows", dict(total=-1)),
    ("n == 0", dict(n=0)),
]


def test_scatter_entry_refuses_before_any_launch():
    before = L.launch_count()
    for what, kw in REFUSED:
        assert _scatter(**kw) < 0, what
        assert "scatter_kv" in L.load().chitu_b200_last_error().decode(), what
    assert L.launch_count() == before


def test_scatter_entry_accepts_what_it_builds_and_an_empty_batch_launches_nothing():
    """The same fake pointers with B == 0 or total_rows == 0 return 0: every argument passed the checks, and nothing was
    launched (a launch would have failed on them)."""
    before = L.launch_count()
    for kw in (dict(), dict(E4M3), dict(CONTIG), dict(cache1=None, src1=None, n=576, src0_st=576),
               dict(E4M3, cache1=None, src1=None, n=576, src0_st=640, page=64), dict(starts=None),
               dict(src0=A + 2, src0_st=1023), dict(page=1)):
        assert _scatter(B=0, **kw) == 0, kw
        assert _scatter(total=0, **kw) == 0, kw
    assert L.launch_count() == before


def test_scatter_op_refuses_cpu_tensors():
    k_cache = torch.zeros(4, 16, 2, 64, dtype=torch.bfloat16)
    k = torch.zeros(10, 2, 64, dtype=torch.bfloat16)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    bt = torch.zeros(2, 4, dtype=torch.int32)
    with pytest.raises(RuntimeError):
        ops.scatter_kv_to_cache(k_cache, k_cache.clone(), k, k.clone(), cu, bt)
    with pytest.raises(RuntimeError):
        ops.scatter_kv_to_cache(k_cache[:, :, 0], None, k[:, 0], None, cu, bt)
