"""Absorbed-MLA attention over the paged latent cache with seqlen_q > 1 on one GPU: the sm_90a kernel behind
B200AttnBackend.mla_attn_with_kvcache with a 4-D q_nope (chitu_b200_mla_paged_prefill) against, in the same process
and on the same cache and inputs,
  decode      sq successive one-token decode calls (chitu_b200_mla_decode), the only native route before it
  gather      append by index, gather the pages into a contiguous copy, attn_varlen_func (the sm_90a MLA prefill kernel)
DeepSeek-V3 local head counts H in {8 (tp = 16), 16 (tp = 8), 128 (tp = 1)}, 64-token pages, bf16, causal, new latent
rows appended:
  multi-token-prediction verification: sq in {2, 4}, B in {1, 16, 64}, prefix in {1024, 4096, 16384};
  chunked prefill: sq in {512, 2048} on a 4096-token prefix at B = 1.
Repeating a call is idempotent (the append rewrites the same positions with the same values), so the cache is not
restored between repeats.

For every case and path: the median, min and max over 5 CUDA-event windows of 20 calls each after 3 warm-up calls;
the causal FLOPs 2 * 1088 * H * sum of visible keys and the unique K bytes Lk * 1152 per request, TFLOP/s and TB/s,
the share of the H100 SXM data-sheet figures (989 TFLOP/s dense bf16, 3.35 TB/s) of the least time either bound
allows and which bound it is, and max_rel of the new path against each comparator.

  python scripts/mla_paged_prefill_bench.py --out DIR          writes DIR/mla_paged_prefill_bench.json

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

C, R, PAGE = 512, 64, 64
ROW = C + R
DATASHEET_BF16_TFLOPS = 989.0
DATASHEET_TB_S = 3.35
CASES = ([("mtp", H, B, prefix, sq) for H in (8, 16, 128) for sq in (2, 4) for B in (1, 16, 64)
          for prefix in (1024, 4096, 16384)]
         + [("chunk", H, 1, 4096, sq) for H in (8, 16, 128) for sq in (512, 2048)])


def make_inputs(H, B, prefix, sq, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    per = math.ceil((prefix + sq) / PAGE)
    nb = B * per + 4
    kc = torch.randn(nb, PAGE, ROW, generator=g).bfloat16().cuda()
    bt = torch.randperm(nb, generator=g)[:B * per].view(B, per).int().cuda()
    q_nope = torch.randn(B, sq, H, C, generator=g).bfloat16().cuda()
    q_pe = torch.randn(B, sq, H, R, generator=g).bfloat16().cuda()
    kv = torch.randn(B, sq, ROW, generator=g).bfloat16().cuda()
    seq_excl = torch.full((B,), prefix, dtype=torch.int32, device="cuda")
    return q_nope, q_pe, kc, kv, seq_excl, bt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mla_paged_prefill_bench.py measures on a CUDA device; none is visible")
    os.makedirs(args.out, exist_ok=True)
    be = B200AttnBackend()
    scale = 1.0 / math.sqrt(be.qk_nope_head_dim + be.qk_rope_head_dim)
    res = {"gpu": gpu_info(), "datasheet_bf16_tflops": DATASHEET_BF16_TFLOPS, "datasheet_tb_s": DATASHEET_TB_S,
           "cases": []}
    for n, (kind, H, B, prefix, sq) in enumerate(CASES):
        q_nope, q_pe, kc, kv, seq_excl, bt = make_inputs(H, B, prefix, sq, seed=n)
        Lk = prefix + sq
        new = lambda: be.mla_attn_with_kvcache(q_nope, q_pe, kc, kv, seq_excl, None, bt, causal=True)  # noqa: E731
        out_new = new()
        t_new = spread(time_ms(new, 3, args.reps, args.windows))
        ms = t_new["median"]
        flops = B * 2.0 * (ROW + C) * H * (sq * prefix + sq * (sq + 1) / 2)
        k_bytes = B * Lk * ROW * 2
        t_flops, t_bytes = flops / (DATASHEET_BF16_TFLOPS * 1e12), k_bytes / (DATASHEET_TB_S * 1e12)
        case = {"kind": kind, "H": H, "B": B, "prefix": prefix, "sq": sq, "kernel_ms": ms, "kernel_ms_spread": t_new,
                "causal_gflop": flops / 1e9, "k_mb": k_bytes / 1e6, "tflops": flops / ms / 1e9,
                "tb_per_s": k_bytes / ms / 1e9, "bound": "compute" if t_flops >= t_bytes else "memory",
                "share_of_datasheet_bound": max(t_flops, t_bytes) * 1e3 / ms}

        # sq successive decode calls: token i appends its row and attends to prefix + i + 1 keys
        steps = [(q_nope[:, i].contiguous(), q_pe[:, i].contiguous(), kv[:, i].contiguous(), seq_excl + i)
                 for i in range(sq)]

        def decode():
            return [be.mla_attn_with_kvcache(qn, qp, kc, k, s, None, bt) for qn, qp, k, s in steps]

        case["max_rel_vs_decode"] = max_rel(out_new, torch.cat(decode(), dim=1))
        t_dec = spread(time_ms(decode, 3, args.reps, args.windows))
        case["decode_ms"], case["decode_ms_spread"] = t_dec["median"], t_dec
        case["speedup_vs_decode"] = t_dec["median"] / ms
        case["speedup_vs_decode_worst"] = t_dec["min"] / t_new["max"]
        del steps

        # append by index, gather the pages into a contiguous copy, attn_varlen_func on it
        new_pos = torch.arange(prefix, Lk, device="cuda")
        new_blk, new_off = bt[:, new_pos // PAGE].long(), new_pos % PAGE
        pos = torch.arange(Lk, device="cuda")
        blk, off = bt[:, pos // PAGE].long(), pos % PAGE
        cu_q = torch.arange(0, (B + 1) * sq, sq, dtype=torch.int32, device="cuda")
        cu_k = torch.arange(0, (B + 1) * Lk, Lk, dtype=torch.int32, device="cuda")

        def gather():
            kc[new_blk, new_off] = kv
            k = kc[blk, off].view(B * Lk, 1, ROW)
            q = torch.cat([q_nope, q_pe], dim=-1).view(B * sq, H, ROW)
            return be.attn_varlen_func(q, k, k[..., :C], cu_q, cu_k, sq, Lk, causal=True, softmax_scale=scale)

        case["max_rel_vs_gather"] = max_rel(out_new, gather().view(B, sq, H, C))
        t_g = spread(time_ms(gather, 3, args.reps, args.windows))
        case["gather_ms"], case["gather_ms_spread"] = t_g["median"], t_g
        case["speedup_vs_gather"] = t_g["median"] / ms
        case["speedup_vs_gather_worst"] = t_g["min"] / t_new["max"]
        print(json.dumps(case), flush=True)
        res["cases"].append(case)
        del q_nope, q_pe, kc, kv, out_new
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "mla_paged_prefill_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
