"""Absorbed-MLA attention over an fp8 (e4m3fn) paged latent cache on one GPU: B200AttnBackend.mla_attn_with_kvcache
with an e4m3 cache (chitu_b200_mla_attn_fp8kv) against the same call over the bf16 cache, in the same process, on the
same values (the e4m3 cache holds the bf16 cache rounded to e4m3; the new rows are bf16 and the fp8 path stores them
rounded).
  decode   sq = 1 at H in {8, 16, 128} (DeepSeek-R1 at tp = 16 / 8 / 1), B in {1, 16, 64}, Lk in {4096, 16384}
  verify   sq in {2, 4} (multi-token-prediction verification) at H in {16, 128}, B = 16, prefix 4096
  chunk    sq in {512, 2048} (chunked prefill on a cached prefix) at H = 16, B = 1, prefix 4096
  engine   the DeepSeek-R1 tp = 16 shard decode step (CUDA graph) at bs = 16 and 64, seq 4096, kv_dtype bf16 and fp8
64-token pages, C = 512, R = 64, causal, new rows appended.

Attention cases: 3 warm-up calls per path, then `--windows` CUDA-event windows of `--reps` calls per path, the bf16
and fp8 windows alternating; median, min and max per path.  The bytes model is the unique cache bytes a call reads,
Lk x 1152 (bf16) or Lk x 576 (e4m3) per request, and TB/s is that over the median.  max_rel is each path's output
against the fp32 reference over its own cache values (decoded cache, stored new rows), for cases small enough to
check.  Engine: per kv_dtype an engine is built, its step captured, 5 steps warmed up and 3 windows of `--reps` graph
replays timed; the bf16 and fp8 engines are built in turn, `--engine-rounds` times, so their windows alternate; ms per
step is the median over all windows of a dtype, with min and max.

  python scripts/mla_fp8_kvcache_bench.py --out DIR          writes DIR/mla_fp8_kvcache_bench.json

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
from fp8_kvcache_bench import alternate, quant  # noqa: E402
from paged_prefill_bench import gpu_info, max_rel, spread, time_ms  # noqa: E402

C, R, PAGE = 512, 64, 64
ROW = C + R
E4M3 = torch.float8_e4m3fn
SCALE = 1.0 / math.sqrt(192)
CASES = ([("decode", H, B, S - 1, 1) for H in (8, 16, 128) for B in (1, 16, 64) for S in (4096, 16384)]
         + [("verify", H, 16, 4096, sq) for H in (16, 128) for sq in (2, 4)]
         + [("chunk", 16, 1, 4096, sq) for sq in (512, 2048)])


def make_inputs(H, B, prefix, sq, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    per = math.ceil((prefix + sq) / PAGE)
    nb = B * per + 4
    kc = torch.randn(nb, PAGE, ROW, generator=g).bfloat16().cuda()
    bt = torch.randperm(nb, generator=g)[:B * per].view(B, per).int().cuda()
    qn = torch.randn(B, sq, H, C, generator=g).bfloat16().cuda()
    qp = torch.randn(B, sq, H, R, generator=g).bfloat16().cuda()
    kv = torch.randn(B, sq, ROW, generator=g).bfloat16().cuda()
    seqlens = torch.full((B,), prefix, dtype=torch.int32, device="cuda")
    return qn, qp, kc, kv, seqlens, bt


def reference(qn, qp, kc, kv, prefix, bt):
    """fp32 attention of every request over its first prefix + sq keys after the append (bottom-right causal)."""
    B, sq, H, _ = qn.shape
    Lk = prefix + sq
    pos = torch.arange(Lk, device=qn.device)
    mask = torch.ones(sq, Lk, dtype=torch.bool, device=qn.device).tril(diagonal=Lk - sq)
    out = torch.empty(B, sq, H, C, dtype=torch.float32, device=qn.device)
    for b in range(B):
        rows = kc[bt[b, pos // PAGE].long(), pos % PAGE].float()
        rows[prefix:] = kv[b].float()
        q = torch.cat([qn[b], qp[b]], dim=-1).float()                                 # [sq, H, 576]
        s = torch.einsum("ihd,jd->hij", q, rows) * SCALE
        p = torch.softmax(s.masked_fill(~mask, float("-inf")), dim=-1)
        out[b] = torch.einsum("hij,jd->ihd", p, rows[:, :C])
    return out


def attention_cases(args):
    out = []
    for n, (kind, H, B, prefix, sq) in enumerate(CASES):
        be = B200AttnBackend(max_seq_len=prefix + sq + PAGE, n_local_heads=H)
        qn, qp, kc, kv, seqlens, bt = make_inputs(H, B, prefix, sq, seed=n)
        kc8 = quant(kc)
        q3 = (qn[:, 0], qp[:, 0]) if sq == 1 else (qn, qp)
        kvc = kv[:, 0] if sq == 1 else kv
        # the append rewrites the same slots every call: the timed calls see the same cache state
        bf = lambda: be.mla_attn_with_kvcache(*q3, kc, kvc, seqlens, None, bt)  # noqa: E731
        f8 = lambda: be.mla_attn_with_kvcache(*q3, kc8, kvc, seqlens, None, bt)  # noqa: E731
        o_bf, o_f8 = bf(), f8()
        t_bf, t_f8 = alternate([bf, f8], args.reps, args.windows)
        Lk = prefix + sq
        bytes_bf, bytes_f8 = B * Lk * ROW * 2, B * Lk * ROW
        case = {"kind": kind, "H": H, "B": B, "prefix": prefix, "sq": sq, "Lk": Lk,
                "bf16_ms": t_bf["median"], "bf16_ms_spread": t_bf, "fp8_ms": t_f8["median"], "fp8_ms_spread": t_f8,
                "speedup": t_bf["median"] / t_f8["median"], "speedup_worst": t_bf["min"] / t_f8["max"],
                "cache_mb_bf16": bytes_bf / 1e6, "cache_mb_fp8": bytes_f8 / 1e6,
                "bf16_tb_per_s": bytes_bf / t_bf["median"] / 1e9, "fp8_tb_per_s": bytes_f8 / t_f8["median"] / 1e9}
        if B * H * sq * Lk <= (1 << 26):
            case["bf16_max_rel"] = max_rel(o_bf.view(B, sq, H, C), reference(qn, qp, kc, kv, prefix, bt))
            case["fp8_max_rel"] = max_rel(o_f8.view(B, sq, H, C),
                                          reference(qn, qp, kc8.float().bfloat16(), quant(kv).float().bfloat16(),
                                                    prefix, bt))
        print(json.dumps(case), flush=True)
        out.append(case)
        del qn, qp, kc, kc8, kv, o_bf, o_f8
        torch.cuda.empty_cache()
    return out


def engine_cases(args):
    from chitu_b200.engine_deepseek import DEEPSEEK_R1, DeepSeekDecodeEngine
    from dataclasses import replace
    cfg = replace(DEEPSEEK_R1, n_layers=args.layers) if args.layers else DEEPSEEK_R1
    S, out = 4096, []
    for B in (16, 64):
        ts = {"bf16": [], "fp8": []}
        for _ in range(args.engine_rounds):
            for name, kv in (("bf16", torch.bfloat16), ("fp8", E4M3)):
                eng = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 512, tp_size=16, kv_dtype=kv)
                eng.set_synthetic_context(S)
                eng.capture()
                ts[name] += time_ms(eng.step, 5, args.reps, 3)
                del eng
                torch.cuda.empty_cache()
        cache_bytes = cfg.n_layers * B * (S + 1) * ROW          # per byte of element
        case = {"kind": "engine", "model": "deepseek-r1-tp16-shard", "layers": cfg.n_layers, "B": B, "seq": S,
                "bf16_ms_per_step": spread(ts["bf16"]), "fp8_ms_per_step": spread(ts["fp8"]),
                "cache_gb_read_bf16": 2 * cache_bytes / 1e9, "cache_gb_read_fp8": cache_bytes / 1e9}
        case["speedup"] = case["bf16_ms_per_step"]["median"] / case["fp8_ms_per_step"]["median"]
        print(json.dumps(case), flush=True)
        out.append(case)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--layers", type=int, default=0, help="engine layer count (0: DeepSeek-R1's 61)")
    ap.add_argument("--engine-rounds", type=int, default=2)
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("mla_fp8_kvcache_bench.py measures on a CUDA device; none is visible")
    os.makedirs(args.out, exist_ok=True)
    res = {"gpu": gpu_info(), "cases": attention_cases(args)}
    if not args.skip_engine:
        res["engine"] = engine_cases(args)
    with open(os.path.join(args.out, "mla_fp8_kvcache_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["gpu"]))


if __name__ == "__main__":
    main()
