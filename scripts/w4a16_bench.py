"""W4A16 (4-bit weights, groups of 128) against bf16 weights on one GPU, both paths alternating in one run:

  GEMM    the LLaMA-3-8B layer shapes qkv 6144x4096, o 4096x4096, w13 28672x4096 (SiluAndMul pairs epilogue) and
          w2 4096x14336 at M = 1, 16, 64: chitu_b200_w4a16_gemm[_silu_pairs] against chitu_b200_linear_bf16[_silu_pairs]
          on the dequantised weight.  Each timed call cycles over NREP distinct weights so that none sits in L2.
          Reported: us per call, GB/s on the algorithmic bytes (packed weight + scales + zeros + x + y; bf16: weight +
          x + y) and their share of the 3.35 TB/s data-sheet HBM bandwidth, the speed-up, and max_rel of the W4 output
          against the bf16 kernel on the dequantised weight.
  engine  LLaMA-3-8B (32 layers), context 4096, bs 1 and 16, the step replayed as one CUDA graph, for
          weight_format="w4a16" and "bf16": ms per step, tok/s and the share of 3.35 TB/s that the step's algorithmic
          bytes (layer weights in their format, the bf16 head, the KV cache read) would need.

Timings: the median, min and max over `--windows` CUDA-event windows after warm-up.

  python scripts/w4a16_bench.py --out DIR          writes DIR/w4a16_bench.json

Reads the device name, power limit and max SM clock (nvidia-smi --query-gpu, a query only); changes no device setting.
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

from paged_prefill_bench import gpu_info, max_rel, spread, time_ms  # noqa: E402

from chitu_b200 import _lib  # noqa: E402
from chitu_b200._lib import check, current_stream, ptr  # noqa: E402
from chitu_b200.quantize import w4a16 as W  # noqa: E402

DATASHEET_TB_S = 3.35
SHAPES = [("qkv", 6144, 4096, False), ("o", 4096, 4096, False), ("w13_pairs", 28672, 4096, True),
          ("w2", 4096, 14336, False)]
MS = (1, 16, 64)
NREP = 8                      # distinct weights per shape: 8 x 8.4 MB (the smallest W4 weight) > the 50 MB L2
BF = torch.bfloat16


def alternate(fns, warmup, reps, windows):
    """`windows` CUDA-event windows of `reps` calls of each function in turn, after `warmup` calls of each."""
    for fn in fns:
        time_ms(fn, warmup, 1, 1)
    ts = [[] for _ in fns]
    for _ in range(windows):
        for i, fn in enumerate(fns):
            ts[i] += time_ms(fn, 0, reps, 1)
    return [spread(t) for t in ts]


def gemm_cases(args, lib):
    dev = "cuda:0"
    out = []
    for name, N, K, pairs in SHAPES:
        g = torch.Generator(device=dev).manual_seed(N + K)
        w4 = [W.quantize_rtn(torch.randn(N, K, generator=g, device=dev) * 0.02, BF) for _ in range(NREP)]
        wbf = [W.dequantize(*t) for t in w4]
        n_out = N // 2 if pairs else N
        for M in MS:
            x = (torch.randn(M, K, generator=g, device=dev)).to(BF)
            y4 = torch.empty(M, n_out, dtype=BF, device=dev)
            yb = torch.empty(M, n_out, dtype=BF, device=dev)
            ws = torch.zeros(lib.chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=dev)
            st = current_stream()

            def run_w4(i):
                q, s, z = w4[i]
                if pairs:
                    return lib.chitu_b200_w4a16_gemm_silu_pairs(ptr(x), ptr(q), ptr(s), ptr(z), ptr(y4), M, N, K,
                                                                _lib.CB_BF16, ptr(ws), ws.numel(), st)
                return lib.chitu_b200_w4a16_gemm(ptr(x), ptr(q), ptr(s), ptr(z), None, ptr(y4), M, N, K, _lib.CB_BF16,
                                                 ptr(ws), ws.numel(), st)

            def run_bf(i):
                if pairs:
                    return lib.chitu_b200_linear_bf16_silu_pairs(ptr(x), ptr(wbf[i]), ptr(yb), M, N, K, ptr(ws),
                                                                 ws.numel(), st)
                return lib.chitu_b200_linear_bf16(ptr(x), ptr(wbf[i]), None, None, ptr(yb), M, N, K, _lib.CB_BF16,
                                                  ptr(ws), ws.numel(), 2, st)

            check(run_w4(0), "w4a16"), check(run_bf(0), "linear_bf16")
            torch.cuda.synchronize()
            rel = max_rel(y4, yb)

            def cycle(fn):
                return lambda: [fn(i) for i in range(NREP)]

            t4, tb = alternate([cycle(run_w4), cycle(run_bf)], 2, args.reps, args.windows)
            us4, usb = t4["median"] * 1e3 / NREP, tb["median"] * 1e3 / NREP
            io = M * K * 2 + M * n_out * 2
            b4 = N * K // 2 + N * (K // 128) * 3 + io
            bb = N * K * 2 + io
            case = {"name": name, "M": M, "N": N, "K": K, "w4_us": us4, "bf16_us": usb, "speedup": usb / us4,
                    "w4_gb_s": b4 / us4 / 1e3, "bf16_gb_s": bb / usb / 1e3,
                    "w4_hbm_share": b4 / us4 / 1e3 / (DATASHEET_TB_S * 1e3),
                    "bf16_hbm_share": bb / usb / 1e3 / (DATASHEET_TB_S * 1e3),
                    "w4_bytes": b4, "bf16_bytes": bb, "max_rel_vs_bf16": rel,
                    "w4_ms_per_cycle": t4, "bf16_ms_per_cycle": tb}
            out.append(case)
            print(f"gemm {name:10s} M={M:3d}  w4 {us4:8.2f} us {case['w4_gb_s']:7.0f} GB/s "
                  f"({case['w4_hbm_share']:.2f})  bf16 {usb:8.2f} us {case['bf16_gb_s']:7.0f} GB/s "
                  f"({case['bf16_hbm_share']:.2f})  speed-up {case['speedup']:.2f}x  max_rel {rel:.1e}", flush=True)
        del w4, wbf
        torch.cuda.empty_cache()
    return out


def step_bytes(eng, cfg, B, S):
    layer = 0
    for lw in eng.layers:
        for name in ("wqkv", "wo", "w13", "w2"):
            t = lw[name]
            layer += sum(u.numel() * u.element_size() for u in t) if isinstance(t, tuple) else t.numel() * t.element_size()
    head = eng.head.numel() * eng.head.element_size()
    kv = 2 * cfg.n_layers * B * S * eng.Hkv * eng.D * 2
    return layer, head, kv


def engine_cases(args):
    from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
    cfg = dataclasses.replace(LLAMA3_8B, n_layers=args.layers)
    S = args.seq
    out = []
    for B in (1, 16):
        engs = {}
        for fmt in ("w4a16", "bf16"):
            e = LlamaDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, device="cuda:0", page_size=256,
                                  weight_format=fmt)
            e.set_synthetic_context(S)
            e.capture()
            engs[fmt] = e
        saved = {f: e.seq_lens.clone() for f, e in engs.items()}

        def stepper(e, s0):
            def fn():
                e.seq_lens.copy_(s0)          # the same context length every step (a copy the graph does not include)
                e.graph.replay()
            return fn

        t = alternate([stepper(engs[f], saved[f]) for f in ("w4a16", "bf16")], 3, args.steps, args.windows)
        for f, tf in zip(("w4a16", "bf16"), t):
            layer, head, kv = step_bytes(engs[f], cfg, B, S)
            ms = tf["median"]
            total = layer + head + kv
            case = {"weight_format": f, "bs": B, "seq": S, "layers": cfg.n_layers, "ms_per_step": ms,
                    "ms_spread": tf, "tok_s": B / ms * 1e3, "step_gb": total / 1e9, "layer_weight_gb": layer / 1e9,
                    "head_gb": head / 1e9, "kv_gb": kv / 1e9, "hbm_share": total / (ms * 1e-3) / (DATASHEET_TB_S * 1e12),
                    "launches_per_step": engs[f].launches_per_step}
            out.append(case)
            print(f"engine {f:6s} bs={B:2d} S={S}  {ms:7.3f} ms/step  {case['tok_s']:8.1f} tok/s  "
                  f"{case['step_gb']:.2f} GB/step  share {case['hbm_share']:.2f}", flush=True)
        del engs
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10, help="weight cycles per GEMM timing window")
    ap.add_argument("--steps", type=int, default=20, help="graph replays per engine timing window")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("w4a16_bench.py measures on a GPU; none is visible")
    lib = _lib.load()
    res = {"gpu": gpu_info(), "datasheet_tb_s": DATASHEET_TB_S, "nrep": NREP}
    print(json.dumps(res["gpu"]), flush=True)
    res["gemm"] = gemm_cases(args, lib)
    if not args.skip_engine:
        res["engine"] = engine_cases(args)
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "w4a16_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
