"""GQA attention over the NON-paged KV cache on one GPU: the sm_90a kernels behind
B200AttnBackend.attn_with_kvcache(block_table=None) (chitu_b200_gqa_contiguous_attn) against, in the same process,
  paged       the paged kernels (chitu_b200_gqa_paged_decode / _prefill) on the same data in 256-token pages: an identity
              block table over the same memory, the same max_seqlen_hint and so the same split count
  flash_attn  flash_attn.flash_attn_with_kvcache without a block table, when it can be imported (recorded either way)
  torch       append by slice, scaled_dot_product_attention with enable_gqa (and the bottom-right mask for sq > 1) over
              the [B, Lk] prefix of the cache
Shapes: LLaMA-3-8B (32 / 8 heads) and Mixtral tp = 4 (8 / 2 heads), head dim 128, bf16, causal, new k / v appended:
  decode (sq = 1) at B in {1, 16, 64} and S in {4096, 10240, 16384} with Lk = S - 1;
  speculative verification at sq in {2, 4, 8}, B in {1, 16}, after a 4096-token context (S = 8192);
  chunked prefill of 512 and 2048 tokens after a 4096-token prefix at B = 1 (S = 8192).
Repeating a call is idempotent (the append rewrites the same positions with the same values), so the caches are not
restored between repeats.

For every case and path: the median, min and max over 5 CUDA-event windows of 20 calls each after 3 warm-up calls
(and, for this kernel and the paged one, the same over replays of a CUDA graph of 20 calls, which leaves out the
host's launch cost: graph_ms is per call, its spread per replay);
the causal FLOPs 4 * D * Hq * sum_i (prefix + i + 1) and the unique K / V bytes 2 * 2 * Lk * Hkv * D per request,
TFLOP/s and TB/s, the share of the H100 SXM data-sheet figures (989 TFLOP/s dense bf16, 3.35 TB/s) of the least time
either bound allows and which bound it is, and max_rel against each comparator.

  python scripts/contiguous_kvcache_bench.py --out DIR          writes DIR/contiguous_kvcache_bench.json

Reads the device name, power limit and max SM clock (nvidia-smi --query-gpu, a query only); changes no device setting.
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
from paged_prefill_bench import gpu_info, max_rel, spread, time_ms  # noqa: E402

D, PAGE = 128, 256
DATASHEET_BF16_TFLOPS = 989.0
DATASHEET_TB_S = 3.35
MODELS = [("llama3-8b", 32, 8), ("mixtral-tp4", 8, 2)]
CASES = ([("decode", m, Hq, Hkv, B, S, S - 2, 1) for m, Hq, Hkv in MODELS for B in (1, 16, 64)
          for S in (4096, 10240, 16384)]
         + [("verify", m, Hq, Hkv, B, 8192, 4096, sq) for m, Hq, Hkv in MODELS for B in (1, 16) for sq in (2, 4, 8)]
         + [("chunk", m, Hq, Hkv, 1, 8192, 4096, sq) for m, Hq, Hkv in MODELS for sq in (512, 2048)])


def make_inputs(Hq, Hkv, B, S, sq, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kc = torch.randn(B, S, Hkv, D, generator=g, device="cuda").bfloat16()
    vc = torch.randn(B, S, Hkv, D, generator=g, device="cuda").bfloat16()
    q = torch.randn(B, sq, Hq, D, generator=g, device="cuda").bfloat16()
    k = torch.randn(B, sq, Hkv, D, generator=g, device="cuda").bfloat16()
    v = torch.randn(B, sq, Hkv, D, generator=g, device="cuda").bfloat16()
    return q, kc, vc, k, v


def graph_ms(fn, reps, windows):
    """time_ms over CUDA-graph replays of `reps` captured calls: the device time without the host's launch cost."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    return time_ms(g.replay, 3, 1, windows)                         # ms per replay of `reps` calls


def torch_path(q, kc, vc, k, v, prefix, scale):
    B, sq, Hq, _ = q.shape
    Lk = prefix + sq
    kc[:, prefix:Lk] = k
    vc[:, prefix:Lk] = v
    kk, vv = kc[:, :Lk].transpose(1, 2), vc[:, :Lk].transpose(1, 2)         # [B, Hkv, Lk, D]
    mask = None
    if sq > 1:
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
        sys.exit("contiguous_kvcache_bench.py measures on a CUDA device; none is visible")
    os.makedirs(args.out, exist_ok=True)
    try:
        from flash_attn import flash_attn_with_kvcache
    except ImportError:
        flash_attn_with_kvcache = None
    be = B200AttnBackend()
    res = {"gpu": gpu_info(), "datasheet_bf16_tflops": DATASHEET_BF16_TFLOPS, "datasheet_tb_s": DATASHEET_TB_S,
           "flash_attn_available": flash_attn_with_kvcache is not None, "cases": []}
    for n, (kind, model, Hq, Hkv, B, S, prefix, sq) in enumerate(CASES):
        q, kc, vc, k, v = make_inputs(Hq, Hkv, B, S, sq, seed=n)
        seqlens = torch.full((B,), prefix, dtype=torch.int32, device="cuda")
        scale = 1.0 / math.sqrt(D)
        new = lambda: be.attn_with_kvcache(q, kc, vc, k, v, seqlens, causal=True)  # noqa: E731
        out_new = new()
        t_new = spread(time_ms(new, 3, args.reps, args.windows))
        ms = t_new["median"]
        flops = B * 4.0 * D * Hq * (sq * prefix + sq * (sq + 1) / 2)
        kv_bytes = B * 2 * 2 * (prefix + sq) * Hkv * D
        t_flops, t_bytes = flops / (DATASHEET_BF16_TFLOPS * 1e12), kv_bytes / (DATASHEET_TB_S * 1e12)
        case = {"kind": kind, "model": model, "Hq": Hq, "Hkv": Hkv, "B": B, "S": S, "prefix": prefix, "sq": sq,
                "kernel_ms": ms, "kernel_ms_spread": t_new, "causal_gflop": flops / 1e9, "kv_mb": kv_bytes / 1e6,
                "tflops": flops / ms / 1e9, "tb_per_s": kv_bytes / ms / 1e9,
                "bound": "compute" if t_flops >= t_bytes else "memory",
                "share_of_datasheet_bound": max(t_flops, t_bytes) * 1e3 / ms}

        kp, vp = kc.view(B * S // PAGE, PAGE, Hkv, D), vc.view(B * S // PAGE, PAGE, Hkv, D)
        bt = torch.arange(B * S // PAGE, dtype=torch.int32, device="cuda").view(B, S // PAGE)
        paged = lambda: be.attn_with_kvcache(q, kp, vp, k, v, seqlens, block_table=bt, causal=True)  # noqa: E731
        out_paged = paged()
        case["bit_identical_to_paged"] = torch.equal(out_new.view(torch.int16), out_paged.view(torch.int16))
        case["max_rel_vs_paged"] = max_rel(out_new, out_paged)
        t_p = spread(time_ms(paged, 3, args.reps, args.windows))
        case["paged_ms"], case["paged_ms_spread"] = t_p["median"], t_p
        case["speedup_vs_paged"] = t_p["median"] / ms
        case["speedup_vs_paged_worst"] = t_p["min"] / t_new["max"]
        g_new, g_p = spread(graph_ms(new, args.reps, args.windows)), spread(graph_ms(paged, args.reps, args.windows))
        case["graph_ms"], case["graph_ms_spread"] = g_new["median"] / args.reps, g_new
        case["paged_graph_ms"], case["paged_graph_ms_spread"] = g_p["median"] / args.reps, g_p
        case["graph_speedup_vs_paged"] = g_p["median"] / g_new["median"]

        if flash_attn_with_kvcache is not None:
            fa = lambda: flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=seqlens,  # noqa: E731
                                                 softmax_scale=scale, causal=True)
            case["max_rel_vs_flash_attn"] = max_rel(out_new, fa())
            t_fa = spread(time_ms(fa, 3, args.reps, args.windows))
            case["flash_attn_ms"], case["flash_attn_ms_spread"] = t_fa["median"], t_fa
            case["speedup_vs_flash_attn"] = t_fa["median"] / ms

        old = lambda: torch_path(q, kc, vc, k, v, prefix, scale)  # noqa: E731
        case["max_rel_vs_torch"] = max_rel(out_new, old())
        t_old = spread(time_ms(old, 3, args.reps, args.windows))
        case["torch_ms"], case["torch_ms_spread"] = t_old["median"], t_old
        case["speedup_vs_torch"] = t_old["median"] / ms
        case["speedup_vs_torch_worst"] = t_old["min"] / t_new["max"]
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
        del q, kc, vc, k, v, kp, vp, out_new, out_paged
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "contiguous_kvcache_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
