"""Absorbed-MLA prefill attention on one GPU: the sm_90a kernel behind B200AttnBackend.attn_varlen_func against the
previous path (flash_attn / torch SDPA per sequence, B200AttnBackend._attn_varlen_library) on the same inputs.

For H in {16, 128} (tp = 8, 1) and causal batches 1x4096, 4x1024, 16x512, 1x16384 it records the kernel time (CUDA
events over warmed-up repeats), the previous path's time when it fits in memory, both outputs' max_rel against each
other, the achieved TFLOP/s from the causal FLOP count 2 * 1088 * H * L (L + 1) / 2 per sequence and its share of the
989 TFLOP/s dense-bf16 figure of the H100 SXM data sheet (a share of a data-sheet rate, not of a measured peak), and
the bytes of K and V the CTAs stage from L2 (each 64-row tile reads every key tile it needs).

  python scripts/prefill_bench.py --out DIR          writes DIR/prefill_bench.json

Reads the device name and power limit (nvidia-smi --query-gpu, a query only); changes no device setting.
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from chitu_b200.attn_backend import B200AttnBackend  # noqa: E402
from paged_prefill_bench import gpu_info  # noqa: E402

QK, DV = 576, 512
DATASHEET_BF16_TFLOPS = 989.0
BATCHES = [(1, 4096), (4, 1024), (16, 512), (1, 16384)]


def causal_flops(H, lens):
    return sum(2.0 * (QK + DV) * H * L * (L + 1) / 2 for L in lens)


def staged_kv_bytes(H, lens):
    """K + V bytes the kernel's CTAs stage (64 query rows per CTA, 64-key tiles, causal)."""
    total = 0
    for L in lens:
        rows = L * H
        for r0 in range(0, rows, 64):
            last = min(r0 + 64, rows) - 1
            total += math.ceil((last // H + 1) / 64) * 64 * (QK + DV) * 2
    return total


def time_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--old-reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prefill_bench.py measures on a CUDA device; none is visible")
    os.makedirs(args.out, exist_ok=True)
    be = B200AttnBackend()
    res = {"gpu": gpu_info(), "datasheet_bf16_tflops": DATASHEET_BF16_TFLOPS, "causal": True, "cases": []}
    for H in (16, 128):
        for nb, L in BATCHES:
            lens = [L] * nb
            g = torch.Generator(device="cpu").manual_seed(H * 100003 + nb * L)
            T = nb * L
            case = {"H": H, "batch": f"{nb}x{L}"}
            try:
                q = (torch.randn(T, H, QK, generator=g) * 2.0).bfloat16().cuda()
                kv = torch.randn(T, 1, QK, generator=g).bfloat16().cuda()
            except torch.OutOfMemoryError:
                case["skipped"] = "inputs do not fit"
                res["cases"].append(case)
                continue
            k, v = kv, kv[..., :DV]
            cu = torch.tensor([i * L for i in range(nb + 1)], dtype=torch.int32, device="cuda")
            new = lambda: be.attn_varlen_func(q, k, v, cu, cu, L, L, causal=True)   # noqa: E731
            out_new = new()
            ms = time_ms(new, 3, args.reps)
            fl = causal_flops(H, lens)
            kvb = staged_kv_bytes(H, lens)
            case.update(kernel_ms=ms, tflops=fl / ms / 1e9, share_of_datasheet_bf16=fl / ms / 1e9 / DATASHEET_BF16_TFLOPS,
                        staged_kv_gb=kvb / 1e9, staged_kv_tb_per_s=kvb / ms / 1e9,
                        unique_kv_and_q_gb=(T * (QK + DV) + T * H * (QK + DV)) * 2 / 1e9)
            old = lambda: be._attn_varlen_library(q, k, v, cu, cu, L, L, causal=True)   # noqa: E731
            try:
                out_old = old()
                torch.cuda.synchronize()
                a, b = out_new.double(), out_old.double()
                case["max_rel_vs_previous"] = ((a - b).abs().max() / b.abs().max().clamp(min=1e-30)).item()
                del out_old, a, b
                case["previous_ms"] = time_ms(old, 1, args.old_reps)
                case["speedup"] = case["previous_ms"] / ms
            except torch.OutOfMemoryError:
                case["previous_ms"] = None
                case["previous_skipped"] = "out of memory"
            torch.cuda.empty_cache()
            print(json.dumps(case), flush=True)
            res["cases"].append(case)
            del q, kv, k, v, out_new
            torch.cuda.empty_cache()
    with open(os.path.join(args.out, "prefill_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
