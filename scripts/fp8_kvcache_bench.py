"""GQA attention over an fp8 (e4m3fn) paged KV cache on one GPU: B200AttnBackend.attn_with_kvcache with e4m3 caches
(chitu_b200_gqa_paged_attn_fp8kv) against the same call over bf16 caches, in the same process, on the same values
(the e4m3 cache holds the bf16 cache rounded to e4m3; new k / v rows are bf16 and the fp8 path stores them rounded).
  decode   sq = 1 at B in {1, 16, 64} and S in {4096, 16384} (Lk = S), LLaMA-3-8B (32 / 8 heads) and Mixtral tp = 4
           (8 / 2 heads)
  multi    the sq > 1 cases of scripts/paged_prefill_bench.py (chunked prefill and speculative verification)
  engine   the LLaMA-3-8B decode step (CUDA graph, fused rotary) at bs = 16 and 64, seq 4096, kv_dtype bf16 and fp8
Head dim 128, 256-token pages, causal, new k / v appended.

Attention cases: 3 warm-up calls per path, then 5 CUDA-event windows of 20 calls per path, the bf16 and fp8 windows
alternating; median, min and max per path.  The KV bytes model is the unique K / V bytes a call reads,
2 * Lk * Hkv * D * (2 B bf16 | 1 B e4m3) per request, and TB/s is that over the median.  max_rel is each path's output
against the fp32 reference over its own cache values (torch SDPA in fp32 over the decoded caches with the stored new
rows).  Engine: per kv_dtype an engine is built, its step captured, 5 steps warmed up and 3 windows of 20 graph replays
timed; the bf16 and fp8 engines are built in turn, twice, so their windows alternate (both do not fit in memory at
bs = 64); ms per step is the median over all windows of a dtype, with min and max.

  python scripts/fp8_kvcache_bench.py --out DIR          writes DIR/fp8_kvcache_bench.json

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
from paged_prefill_bench import CASES as MULTI_CASES  # noqa: E402
from paged_prefill_bench import gpu_info, max_rel, spread, time_ms  # noqa: E402

D, PAGE = 128, 256
E4M3 = torch.float8_e4m3fn
MODELS = [("llama3-8b", 32, 8), ("mixtral-tp4", 8, 2)]
CASES = ([("decode", m, Hq, Hkv, B, S, 1) for m, Hq, Hkv in MODELS for B in (1, 16, 64) for S in (4096, 16384)]
         + [("multi", m, Hq, Hkv, B, prefix, sq) for m, Hq, Hkv, B, prefix, sq in MULTI_CASES])


def quant(x):
    return x.float().clamp(-448.0, 448.0).to(E4M3)


def make_inputs(Hq, Hkv, B, prefix, sq, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    per = math.ceil((prefix + sq) / PAGE)
    nb = B * per + 4
    kc = torch.randn(nb, PAGE, Hkv, D, generator=g).bfloat16().cuda()
    vc = torch.randn(nb, PAGE, Hkv, D, generator=g).bfloat16().cuda()
    bt = torch.randperm(nb, generator=g)[:B * per].view(B, per).int().cuda()
    q = torch.randn(B, sq, Hq, D, generator=g).bfloat16().cuda()
    k = torch.randn(B, sq, Hkv, D, generator=g).bfloat16().cuda()
    v = torch.randn(B, sq, Hkv, D, generator=g).bfloat16().cuda()
    seqlens = torch.full((B,), prefix, dtype=torch.int32, device="cuda")
    return q, kc, vc, k, v, seqlens, bt


def reference(q, kc, vc, k, v, prefix, bt, scale):
    """fp32 attention of every request over its first prefix + sq keys after the append (bottom-right causal)."""
    B, sq, Hq, _ = q.shape
    Lk = prefix + sq
    pos = torch.arange(Lk, device=q.device)
    mask = torch.ones(sq, Lk, dtype=torch.bool, device=q.device).tril(diagonal=Lk - sq)
    out = torch.empty(B, sq, Hq, D, dtype=torch.float32, device=q.device)
    for b in range(B):
        blk = bt[b, pos // PAGE].long()
        kk, vv = kc[blk, pos % PAGE].float(), vc[blk, pos % PAGE].float()          # [Lk, Hkv, D]
        kk[prefix:], vv[prefix:] = k[b].float(), v[b].float()
        o = torch.nn.functional.scaled_dot_product_attention(
            q[b].float().transpose(0, 1), kk.transpose(0, 1), vv.transpose(0, 1), attn_mask=mask, scale=scale,
            enable_gqa=Hq != kk.shape[1])
        out[b] = o.transpose(0, 1)
    return out


def alternate(fns, reps, windows):
    """`windows` CUDA-event windows of `reps` calls for each function in turn (3 warm-up calls each first)."""
    for fn in fns:
        time_ms(fn, 3, 1, 1)
    ts = [[] for _ in fns]
    for _ in range(windows):
        for i, fn in enumerate(fns):
            ts[i] += time_ms(fn, 0, reps, 1)
    return [spread(t) for t in ts]


def attention_cases(args, be):
    out = []
    for n, (kind, model, Hq, Hkv, B, prefix, sq) in enumerate(CASES):
        if kind == "decode":
            prefix -= 1                                            # Lk = S with the appended token
        q, kc, vc, k, v, seqlens, bt = make_inputs(Hq, Hkv, B, prefix, sq, seed=n)
        kc8, vc8 = quant(kc), quant(vc)
        scale = 1.0 / math.sqrt(D)
        bf = lambda: be.attn_with_kvcache(q, kc, vc, k, v, seqlens, block_table=bt, causal=True)  # noqa: E731
        f8 = lambda: be.attn_with_kvcache(q, kc8, vc8, k, v, seqlens, block_table=bt, causal=True)  # noqa: E731
        o_bf, o_f8 = bf(), f8()
        t_bf, t_f8 = alternate([bf, f8], args.reps, args.windows)
        Lk = prefix + sq
        bytes_bf, bytes_f8 = B * 2 * Lk * Hkv * D * 2, B * 2 * Lk * Hkv * D
        case = {"kind": kind, "model": model, "Hq": Hq, "Hkv": Hkv, "B": B, "prefix": prefix, "sq": sq,
                "bf16_ms": t_bf["median"], "bf16_ms_spread": t_bf, "fp8_ms": t_f8["median"], "fp8_ms_spread": t_f8,
                "speedup": t_bf["median"] / t_f8["median"], "speedup_worst": t_bf["min"] / t_f8["max"],
                "kv_mb_bf16": bytes_bf / 1e6, "kv_mb_fp8": bytes_f8 / 1e6,
                "bf16_tb_per_s": bytes_bf / t_bf["median"] / 1e9, "fp8_tb_per_s": bytes_f8 / t_f8["median"] / 1e9,
                "bf16_max_rel": max_rel(o_bf, reference(q, kc, vc, k, v, prefix, bt, scale)),
                "fp8_max_rel": max_rel(o_f8, reference(q, kc8, vc8, quant(k), quant(v), prefix, bt, scale))}
        print(json.dumps(case), flush=True)
        out.append(case)
        del q, kc, vc, k, v, kc8, vc8, o_bf, o_f8
        torch.cuda.empty_cache()
    return out


def engine_cases(args):
    from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
    S, out = 4096, []
    for B in (16, 64):
        ts = {"bf16": [], "fp8": []}
        for _ in range(2):
            for name, kv in (("bf16", torch.bfloat16), ("fp8", E4M3)):
                eng = LlamaDecodeEngine(LLAMA3_8B, max_reqs=B, max_seq_len=S + 512, page_size=256, kv_dtype=kv)
                eng.set_synthetic_context(S)
                eng.capture()
                ts[name] += time_ms(eng.step, 5, args.reps, 3)
                del eng
                torch.cuda.empty_cache()
        kv_bytes = 32 * B * 2 * S * 8 * D            # layers x requests x (K, V) x keys x kv heads x D, per byte/elem
        case = {"kind": "engine", "model": "llama3-8b", "B": B, "seq": S,
                "bf16_ms_per_step": spread(ts["bf16"]), "fp8_ms_per_step": spread(ts["fp8"]),
                "kv_gb_bf16": 2 * kv_bytes / 1e9, "kv_gb_fp8": kv_bytes / 1e9}
        case["speedup"] = case["bf16_ms_per_step"]["median"] / case["fp8_ms_per_step"]["median"]
        case["bf16_tok_s"] = B * 1e3 / case["bf16_ms_per_step"]["median"]
        case["fp8_tok_s"] = B * 1e3 / case["fp8_ms_per_step"]["median"]
        print(json.dumps(case), flush=True)
        out.append(case)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_kvcache_bench.py measures on a CUDA device; none is visible")
    os.makedirs(args.out, exist_ok=True)
    res = {"gpu": gpu_info(), "cases": attention_cases(args, B200AttnBackend())}
    if not args.skip_engine:
        res["engine"] = engine_cases(args)
    with open(os.path.join(args.out, "fp8_kvcache_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
