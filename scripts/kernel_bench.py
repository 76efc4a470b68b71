"""Per-kernel microbenchmarks (dev tool): warm CUDA-event timing of the hot kernels at the bench shapes.

Every case rotates over enough distinct copies of its HBM-resident operands (weights / KV pages) that a call never
finds them in the 50 MB L2 — the honest way to defeat the cache: a memset-style flush leaves dirty lines whose
write-back is charged to the next kernel.

    python scripts/kernel_bench.py gemm | mla | gqa | moe | all        (needs an H100)
"""
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from chitu_b200 import fused_moe, ops  # noqa: E402
from chitu_b200.attn_backend import B200AttnBackend  # noqa: E402

DEV = "cuda"
L2 = 126 << 20


def timed(fn, n_sets, iters=5):
    """All `n_sets` calls (one per operand set) are captured in ONE CUDA graph and the replay is timed: per-call device
    time without the host's launch cost (an eager loop of 20 us kernels measures ctypes + cuTensorMapEncode, not the GPU)."""
    for i in range(min(n_sets, 3)):
        fn(i)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn(0)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(n_sets):
            fn(i)
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / n_sets)
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def sets_for(nbytes):
    return max(2, math.ceil(3 * L2 / max(nbytes, 1)))


def bench_gemm():
    """the dense decode linears of LLaMA-3-8B (bf16) and of one DeepSeek-R1 tp=8 rank (fp8 block-scaled), M = 1 / 16"""
    shapes = [("llama wqkv", 6144, 4096, "bf16"), ("llama wo", 4096, 4096, "bf16"), ("llama w13", 28672, 4096, "bf16"),
              ("llama w2", 4096, 14336, "bf16"), ("llama head", 128256, 4096, "bf16"),
              ("ds wqkv_a", 2112, 7168, "fp8"), ("ds wq_b", 3072, 1536, "fp8"), ("ds wo", 7168, 2048, "fp8"),
              ("ds gate", 256, 7168, "bf16"), ("ds dense w13", 4608, 7168, "fp8"), ("ds dense w2", 7168, 2304, "fp8"),
              ("ds shared w13", 512, 7168, "fp8"), ("ds shared w2", 7168, 256, "fp8"), ("ds head", 16160, 7168, "bf16")]
    for name, N, K, kind in shapes:
        for M in (1, 16):
            elem = 2 if kind == "bf16" else 1
            n = min(sets_for(N * K * elem), 48)
            if kind == "bf16":
                ws = [torch.randn(N, K, device=DEV, dtype=torch.bfloat16) * 0.02 for _ in range(n)]
                x = torch.randn(M, K, device=DEV, dtype=torch.bfloat16)
                fn = lambda i: ops.linear(x, ws[i])
            else:
                ws = [torch.randint(-60, 60, (N, K), device=DEV, dtype=torch.int8).view(torch.float8_e4m3fn) for _ in range(n)]
                ss = [torch.rand((N + 127) // 128, (K + 127) // 128, device=DEV) * 0.01 + 0.001 for _ in range(n)]
                xq, xs = ops.act_quant_deepseek_v3(torch.randn(M, K, device=DEV, dtype=torch.bfloat16))
                fn = lambda i: ops.fp8_gemm_deepseek_v3(xq, xs, ws[i], ss[i])
            med, mn = timed(fn, n)
            mb = N * K * elem / 1e6
            print(f"gemm  {name:14s} {kind} M={M:2d} N={N:6d} K={K:5d}  {med:7.1f} us (min {mn:6.1f})  {mb:7.1f} MB  "
                  f"{mb / med * 1e-3 * 1e3:5.2f} TB/s  fixed-cost est {med - mb / 5.6:5.1f} us", flush=True)
            del ws


def bench_gqa():
    for B, ctx, Hq, Hkv in ((16, 4096, 32, 8), (1, 4096, 32, 8), (16, 4096, 4, 1), (64, 1024, 32, 8)):
        D, page = 128, 256
        per = (ctx + page) // page
        nbytes = B * ctx * Hkv * D * 2 * 2
        n = min(sets_for(nbytes), 24)
        caches = [(torch.randn(B * per, page, Hkv, D, device=DEV, dtype=torch.bfloat16),
                   torch.randn(B * per, page, Hkv, D, device=DEV, dtype=torch.bfloat16)) for _ in range(n)]
        bt = torch.randperm(B * per, device=DEV, dtype=torch.int32).view(B, per).contiguous()
        seqlens = torch.full((B,), ctx - 1, device=DEV, dtype=torch.int32)
        q = torch.randn(B, 1, Hq, D, device=DEV, dtype=torch.bfloat16)
        kn = torch.randn(B, 1, Hkv, D, device=DEV, dtype=torch.bfloat16)
        vn = torch.randn(B, 1, Hkv, D, device=DEV, dtype=torch.bfloat16)
        be = B200AttnBackend(max_seq_len=ctx)
        fn = lambda i: be.attn_with_kvcache(q, caches[i][0], caches[i][1], kn, vn, cache_seqlens=seqlens, block_table=bt)
        med, mn = timed(fn, n)
        print(f"gqa   B={B:2d} ctx={ctx} Hq={Hq} Hkv={Hkv}  {med:7.1f} us (min {mn:6.1f})  {nbytes / 1e6:7.1f} MB  "
              f"{nbytes / med / 1e6:5.2f} TB/s", flush=True)
        del caches


def bench_mla():
    for B, ctx, H in ((16, 4096, 16), (1, 4096, 16), (64, 1024, 16), (16, 4096, 128)):
        C, R, page = 512, 64, 64
        per = (ctx + page) // page
        nbytes = B * ctx * (C + R) * 2
        n = min(sets_for(nbytes), 32)
        caches = [torch.randn(B * per, page, C + R, device=DEV, dtype=torch.bfloat16) for _ in range(n)]
        bt = torch.randperm(B * per, device=DEV, dtype=torch.int32).view(B, per).contiguous()
        excl = torch.full((B,), ctx - 1, device=DEV, dtype=torch.int32)
        q_nope = torch.randn(B, H, C, device=DEV, dtype=torch.bfloat16)
        q_pe = torch.randn(B, H, R, device=DEV, dtype=torch.bfloat16)
        kv = torch.randn(B, 1, 1, C + R, device=DEV, dtype=torch.bfloat16)
        be = B200AttnBackend(max_seq_len=ctx, max_reqs=B, n_local_heads=H)
        be.prepare_metadata_for_decode(excl, excl + 1, bt, page)
        fn = lambda i: be.mla_attn_with_kvcache(q_nope, q_pe, caches[i], kv, excl, excl + 1, bt, softmax_scale=0.1352)
        med, mn = timed(fn, n)
        print(f"mla   B={B:2d} ctx={ctx} H={H:3d}  {med:7.1f} us (min {mn:6.1f})  {nbytes / 1e6:7.1f} MB  "
              f"{nbytes / med / 1e6:5.2f} TB/s   (decode + split merge)", flush=True)
        del caches


def bench_moe():
    E, N1, K1, inter = 257, 512, 7168, 256
    n = 4
    sets = []
    for _ in range(n):
        w1 = torch.randint(-60, 60, (E, N1, K1), device=DEV, dtype=torch.int8).view(torch.float8_e4m3fn)
        w2 = torch.randint(-60, 60, (E, K1, inter), device=DEV, dtype=torch.int8).view(torch.float8_e4m3fn)
        sets.append((w1, w2, torch.rand(E, N1 // 128, K1 // 128, device=DEV) * 0.01 + 0.001,
                     torch.rand(E, K1 // 128, inter // 128, device=DEV) * 0.01 + 0.001))
    for T in (1, 4, 16, 64):
        x = torch.randn(T, K1, device=DEV, dtype=torch.bfloat16)
        ids = torch.stack([torch.cat([torch.randperm(256, device=DEV)[:8], torch.tensor([256], device=DEV)])
                           for _ in range(T)]).to(torch.int64)
        tw = torch.rand(T, 9, device=DEV, dtype=torch.float32)
        fn = lambda i: fused_moe.fused_experts(x, sets[i][0], sets[i][1], tw, ids, use_fp8_w8a8=True, w1_scale=sets[i][2],
                                               w2_scale=sets[i][3], block_shape=[128, 128])
        med, mn = timed(fn, n)
        nd = ids.unique().numel()
        mb = nd * (N1 * K1 + K1 * inter) / 1e6
        print(f"moe   T={T:3d} distinct experts {nd:3d}  {med:7.1f} us (min {mn:6.1f})  {mb:6.0f} MB  {mb / med * 1e-3 * 1e3:5.2f} TB/s",
              flush=True)


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "all"
    for name, fn in (("gemm", bench_gemm), ("gqa", bench_gqa), ("mla", bench_mla), ("moe", bench_moe)):
        if what in (name, "all"):
            fn()
