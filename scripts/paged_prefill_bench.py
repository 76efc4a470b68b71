"""GQA attention over the paged KV cache with seqlen_q > 1 on one GPU: the sm_90a kernel behind
B200AttnBackend.attn_with_kvcache (chitu_b200_gqa_paged_prefill) against, in the same process,
  torch       append by index, gather the pages, scaled_dot_product_attention with enable_gqa and the bottom-right mask
  flash_attn  flash_attn.flash_attn_with_kvcache on the same paged cache, when it can be imported (recorded either way)
LLaMA-3-8B layer shapes (32 / 8 heads, head dim 128, 256-token pages, bf16, causal, new k / v appended):
  chunked prefill at B = 1, (prefix, chunk) in (0, 512) (0, 2048) (0, 8192) (4096, 512) (4096, 2048) (16384, 2048);
  speculative verification at B in {1, 16}, sq in {2, 4, 8}, context 4096;
plus one Mixtral tp = 4 (8 / 2 heads) chunk.  Repeating a call is idempotent (the append rewrites the same positions
with the same values), so the caches are not restored between repeats.

For every case and path: the median, min and max over 5 CUDA-event windows of 20 calls each after 3 warm-up calls;
the causal FLOPs 4 * D * Hq * sum_i (prefix + i + 1) and the unique K / V bytes 2 * 2 * Lk * Hkv * D per request,
TFLOP/s and TB/s, the share of the H100 SXM data-sheet figures (989 TFLOP/s dense bf16, 3.35 TB/s) of the least time
either bound allows and which bound it is, and max_rel against each comparator.

  python scripts/paged_prefill_bench.py --out DIR          writes DIR/paged_prefill_bench.json

Reads the device name, power limit and max SM clock (nvidia-smi --query-gpu, a query only); changes no device setting.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chitu_b200.attn_backend import B200AttnBackend  # noqa: E402

D, PAGE = 128, 256
DATASHEET_BF16_TFLOPS = 989.0
DATASHEET_TB_S = 3.35
CASES = ([("llama3-8b", 32, 8, 1, prefix, chunk)
          for prefix, chunk in [(0, 512), (0, 2048), (0, 8192), (4096, 512), (4096, 2048), (16384, 2048)]]
         + [("llama3-8b", 32, 8, B, 4096, sq) for B in (1, 16) for sq in (2, 4, 8)]
         + [("mixtral-tp4", 8, 2, 1, 4096, 2048)])


def time_ms(fn, warmup, reps, windows):
    """Mean ms per call in each of `windows` CUDA-event windows of `reps` calls, after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(windows):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(reps):
            fn()
        end.record()
        torch.cuda.synchronize()
        res.append(start.elapsed_time(end) / reps)
    return res


def spread(ts):
    ts = sorted(ts)
    return {"median": ts[len(ts) // 2], "min": ts[0], "max": ts[-1]}


def gpu_info():
    info = {"device": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv"],
                           capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e!r}"
    return info


def max_rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-30)).item()


def make_inputs(Hq, Hkv, B, prefix, sq, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    Lk = prefix + sq
    per = math.ceil(Lk / PAGE)
    nb = B * per + 4
    kc = torch.randn(nb, PAGE, Hkv, D, generator=g).bfloat16().cuda()
    vc = torch.randn(nb, PAGE, Hkv, D, generator=g).bfloat16().cuda()
    bt = torch.randperm(nb, generator=g)[:B * per].view(B, per).int().cuda()
    q = torch.randn(B, sq, Hq, D, generator=g).bfloat16().cuda()
    k = torch.randn(B, sq, Hkv, D, generator=g).bfloat16().cuda()
    v = torch.randn(B, sq, Hkv, D, generator=g).bfloat16().cuda()
    seqlens = torch.full((B,), prefix, dtype=torch.int32, device="cuda")
    return q, kc, vc, k, v, seqlens, bt


def torch_path(q, kc, vc, k, v, prefix, bt, scale):
    B, sq, Hq, _ = q.shape
    Lk = prefix + sq
    pos = torch.arange(prefix, Lk, device=q.device)
    blk = bt[:, pos // PAGE].long()                                  # [B, sq]
    kc[blk, pos % PAGE] = k
    vc[blk, pos % PAGE] = v
    pos = torch.arange(Lk, device=q.device)
    blk = bt[:, pos // PAGE].long()
    kk = kc[blk, pos % PAGE].transpose(1, 2)                         # [B, Hkv, Lk, D]
    vv = vc[blk, pos % PAGE].transpose(1, 2)
    mask = torch.ones(sq, Lk, dtype=torch.bool, device=q.device).tril(diagonal=Lk - sq)
    o = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), kk, vv, attn_mask=mask, scale=scale,
                                                         enable_gqa=Hq != kk.shape[1])
    return o.transpose(1, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("paged_prefill_bench.py measures on a CUDA device; none is visible")
    os.makedirs(args.out, exist_ok=True)
    try:
        from flash_attn import flash_attn_with_kvcache
    except ImportError:
        flash_attn_with_kvcache = None
    be = B200AttnBackend()
    res = {"gpu": gpu_info(), "datasheet_bf16_tflops": DATASHEET_BF16_TFLOPS, "datasheet_tb_s": DATASHEET_TB_S,
           "flash_attn_available": flash_attn_with_kvcache is not None, "cases": []}
    for n, (model, Hq, Hkv, B, prefix, sq) in enumerate(CASES):
        q, kc, vc, k, v, seqlens, bt = make_inputs(Hq, Hkv, B, prefix, sq, seed=n)
        scale = 1.0 / math.sqrt(D)
        new = lambda: be.attn_with_kvcache(q, kc, vc, k, v, seqlens, block_table=bt, causal=True)  # noqa: E731
        out_new = new()
        t_new = spread(time_ms(new, 3, args.reps, args.windows))
        ms = t_new["median"]
        flops = B * 4.0 * D * Hq * (sq * prefix + sq * (sq + 1) / 2)
        kv_bytes = B * 2 * 2 * (prefix + sq) * Hkv * D
        t_flops, t_bytes = flops / (DATASHEET_BF16_TFLOPS * 1e12), kv_bytes / (DATASHEET_TB_S * 1e12)
        case = {"model": model, "Hq": Hq, "Hkv": Hkv, "B": B, "prefix": prefix, "sq": sq, "kernel_ms": ms,
                "kernel_ms_spread": t_new,
                "causal_gflop": flops / 1e9, "kv_mb": kv_bytes / 1e6, "tflops": flops / ms / 1e9,
                "tb_per_s": kv_bytes / ms / 1e9, "bound": "compute" if t_flops >= t_bytes else "memory",
                "share_of_datasheet_bound": max(t_flops, t_bytes) * 1e3 / ms}
        old = lambda: torch_path(q, kc, vc, k, v, prefix, bt, scale)  # noqa: E731
        out_old = old()
        case["max_rel_vs_torch"] = max_rel(out_new, out_old)
        t_old = spread(time_ms(old, 3, args.reps, args.windows))
        case["torch_ms"], case["torch_ms_spread"] = t_old["median"], t_old
        case["speedup_vs_torch"] = case["torch_ms"] / ms
        case["speedup_vs_torch_worst"] = t_old["min"] / t_new["max"]
        del out_old
        if flash_attn_with_kvcache is not None:
            fa = lambda: flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=seqlens, block_table=bt,  # noqa: E731
                                                 softmax_scale=scale, causal=True)
            case["max_rel_vs_flash_attn"] = max_rel(out_new, fa())
            t_fa = spread(time_ms(fa, 3, args.reps, args.windows))
            case["flash_attn_ms"], case["flash_attn_ms_spread"] = t_fa["median"], t_fa
            case["speedup_vs_flash_attn"] = case["flash_attn_ms"] / ms
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
        del q, kc, vc, k, v, out_new
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "paged_prefill_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
