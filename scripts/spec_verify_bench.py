"""Cost of the LLaMA engine's speculative verify step against its decode step on one GPU, both captured as CUDA graphs
and replayed alternating in the same run.

LLaMA-3-8B (32 layers), context 4096, bs 1 / 4 / 16, k = 1 / 3 / 7 drafts per request, bf16 and fp8 weights, bf16 and
e4m3 KV caches.  For each case one engine is built with max_draft = k; its decode graph (B rows) and its verify graph
(B * (k + 1) rows, causal attention over the cache plus the k + 1 new rows, greedy acceptance) are timed with CUDA
events.  seq_lens is reset before every replay (a copy outside both graphs), so every step runs at the same context.

Reported per case: ms per decode step and per verify step (median, min, max over `--windows` windows), their ratio, and
the break-even mean accepted length ratio - 1: a verify step emits accepted + 1 tokens, so drafts that are accepted
more often than that on average make verification cheaper per token than decoding.

  python scripts/spec_verify_bench.py --out DIR          writes DIR/spec_verify_bench.json

Reads the device name, power limit and max SM clock (nvidia-smi --query-gpu, a query only); changes no device setting.
Multi-GPU (tensor-parallel) verify steps are not measured here: they need more than one GPU.
"""
import argparse
import dataclasses
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from paged_prefill_bench import gpu_info  # noqa: E402
from w4a16_bench import alternate  # noqa: E402


def case(cfg, B, k, fmt, kv, args):
    from chitu_b200.engine import LlamaDecodeEngine
    S = args.seq
    e = LlamaDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, device="cuda:0", page_size=256, weight_format=fmt,
                          kv_dtype=kv, max_draft=k)
    e.set_synthetic_context(S)
    e.n_draft.fill_(k)
    e.capture()
    e.capture_verify()
    s0 = e.seq_lens.clone()

    def replay(graph):
        def fn():
            e.seq_lens.copy_(s0)
            graph.replay()
        return fn

    t_dec, t_ver = alternate([replay(e.graph), replay(e.verify_graph)], 3, args.steps, args.windows)
    ratio = t_ver["median"] / t_dec["median"]
    out = {"weight_format": fmt, "kv": "e4m3" if kv == torch.float8_e4m3fn else "bf16", "bs": B, "k": k, "seq": S,
           "layers": cfg.n_layers, "decode_ms": t_dec, "verify_ms": t_ver, "ratio": ratio,
           "break_even_accepted": ratio - 1, "launches_decode": e.launches_per_step,
           "launches_verify": e.launches_per_verify}
    del e
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=20, help="graph replays per timing window")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--k", type=int, nargs="+", default=[1, 3, 7])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_verify_bench.py measures on a GPU; none is visible")
    from chitu_b200.engine import LLAMA3_8B
    cfg = dataclasses.replace(LLAMA3_8B, n_layers=args.layers)
    res = {"gpu": gpu_info(), "cases": []}
    print(json.dumps(res["gpu"]), flush=True)
    for fmt in ("bf16", "fp8"):
        for kv in (torch.bfloat16, torch.float8_e4m3fn):
            for B in args.bs:
                for k in args.k:
                    c = case(cfg, B, k, fmt, kv, args)
                    res["cases"].append(c)
                    print(f"{fmt:4s} kv={c['kv']:5s} bs={B:2d} k={k}  decode {c['decode_ms']['median']:7.3f} ms  "
                          f"verify {c['verify_ms']['median']:7.3f} ms  ratio {c['ratio']:.3f}  "
                          f"break-even accepted {c['break_even_accepted']:.3f}", flush=True)
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "spec_verify_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
