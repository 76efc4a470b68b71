"""FP8 rowwise (e4m3 W8A8, per-channel weight and per-token activation scales) against bf16 and W4A16 weights on one
GPU, the paths alternating in one run:

  GEMM    the LLaMA-3-8B layer shapes qkv 6144x4096, o 4096x4096, w13 28672x4096 (SiluAndMul pairs epilogue) and
          w2 4096x14336 at M = 1, 16, 64: chitu_b200_fp8_rowwise_gemm[_silu_pairs] on already quantised activations,
          chitu_b200_linear_bf16[_silu_pairs] and chitu_b200_w4a16_gemm[_silu_pairs] on weights of the same
          distribution.  Each timed call cycles over NREP distinct weights so that none sits in L2.  Reported: us per
          call, GB/s on the algorithmic bytes (fp8: e4m3 weight + scales + e4m3 x + its scales + y; bf16: weight + x +
          y; W4: packed weight + scales + zeros + x + y) and their share of the 3.35 TB/s data-sheet HBM bandwidth, the
          speed-ups over bf16, and max_rel of the fp8 output against the fp64 product of its operands.
  engine  LLaMA-3-8B (32 layers), context 4096, bs 1 and 16, the step replayed as one CUDA graph, for
          weight_format="fp8" and "bf16": ms per step, tok/s and the share of 3.35 TB/s that the step's algorithmic
          bytes (layer weights in their format, the bf16 head, the KV cache read) would need.

Timings: the median, min and max over `--windows` CUDA-event windows after warm-up.

  python scripts/fp8_linear_bench.py --out DIR          writes DIR/fp8_linear_bench.json

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
from w4a16_bench import DATASHEET_TB_S, MS, NREP, SHAPES, alternate, step_bytes  # noqa: E402

from chitu_b200 import _lib  # noqa: E402
from chitu_b200._lib import check, current_stream, ptr  # noqa: E402
from chitu_b200.quantize import fp8 as Q  # noqa: E402
from chitu_b200.quantize import w4a16 as W  # noqa: E402

BF = torch.bfloat16


def gemm_cases(args, lib):
    dev = "cuda:0"
    out = []
    for name, N, K, pairs in SHAPES:
        g = torch.Generator(device=dev).manual_seed(N + K)
        wf = [torch.randn(N, K, generator=g, device=dev) * 0.02 for _ in range(NREP)]
        w8 = [Q.quantize_weight(w) for w in wf]
        wbf = [w.to(BF) for w in wf]
        w4 = [W.quantize_rtn(w, BF) for w in wf]
        del wf
        n_out = N // 2 if pairs else N
        for M in MS:
            x = torch.randn(M, K, generator=g, device=dev).to(BF)
            xq, xs = Q.quant_act_fp8(x)
            y8, yb, y4 = (torch.empty(M, n_out, dtype=BF, device=dev) for _ in range(3))
            ws = torch.zeros(lib.chitu_b200_linear_workspace_bytes(M, N), dtype=torch.uint8, device=dev)
            st = current_stream()

            def run_fp8(i):
                q, s = w8[i]
                if pairs:
                    return lib.chitu_b200_fp8_rowwise_gemm_silu_pairs(ptr(xq), ptr(xs), ptr(q), ptr(s), ptr(y8), M, N,
                                                                      K, ptr(ws), ws.numel(), st)
                return lib.chitu_b200_fp8_rowwise_gemm(ptr(xq), ptr(xs), ptr(q), ptr(s), None, None, ptr(y8), M, N, K,
                                                       ptr(ws), ws.numel(), st)

            def run_bf(i):
                if pairs:
                    return lib.chitu_b200_linear_bf16_silu_pairs(ptr(x), ptr(wbf[i]), ptr(yb), M, N, K, ptr(ws),
                                                                 ws.numel(), st)
                return lib.chitu_b200_linear_bf16(ptr(x), ptr(wbf[i]), None, None, ptr(yb), M, N, K, _lib.CB_BF16,
                                                  ptr(ws), ws.numel(), 2, st)

            def run_w4(i):
                q, s, z = w4[i]
                if pairs:
                    return lib.chitu_b200_w4a16_gemm_silu_pairs(ptr(x), ptr(q), ptr(s), ptr(z), ptr(y4), M, N, K,
                                                                _lib.CB_BF16, ptr(ws), ws.numel(), st)
                return lib.chitu_b200_w4a16_gemm(ptr(x), ptr(q), ptr(s), ptr(z), None, ptr(y4), M, N, K, _lib.CB_BF16,
                                                 ptr(ws), ws.numel(), st)

            check(run_fp8(0), "fp8_rowwise"), check(run_bf(0), "linear_bf16"), check(run_w4(0), "w4a16")
            torch.cuda.synchronize()
            q0, s0 = w8[0]
            ref = (xq.double() * xs.double()[:, None]) @ (q0.double() * s0.double()[:, None]).T
            if pairs:
                g_, u_ = ref[:, 0::2].to(BF).double(), ref[:, 1::2].to(BF).double()
                ref = (g_ / (1 + torch.exp(-g_))).to(BF).double() * u_
            rel = max_rel(y8, ref)
            del ref

            def cycle(fn):
                return lambda: [fn(i) for i in range(NREP)]

            t8, tb, t4 = alternate([cycle(run_fp8), cycle(run_bf), cycle(run_w4)], 2, args.reps, args.windows)
            us8, usb, us4 = (t["median"] * 1e3 / NREP for t in (t8, tb, t4))
            b8 = N * K + N * 4 + M * K + M * 4 + M * n_out * 2
            bb = N * K * 2 + M * K * 2 + M * n_out * 2
            b4 = N * K // 2 + N * (K // 128) * 3 + M * K * 2 + M * n_out * 2
            share = lambda b, us: b / us / 1e3 / (DATASHEET_TB_S * 1e3)    # noqa: E731
            case = {"name": name, "M": M, "N": N, "K": K, "fp8_us": us8, "bf16_us": usb, "w4_us": us4,
                    "fp8_speedup_vs_bf16": usb / us8, "w4_speedup_vs_bf16": usb / us4,
                    "fp8_gb_s": b8 / us8 / 1e3, "bf16_gb_s": bb / usb / 1e3, "w4_gb_s": b4 / us4 / 1e3,
                    "fp8_hbm_share": share(b8, us8), "bf16_hbm_share": share(bb, usb), "w4_hbm_share": share(b4, us4),
                    "fp8_bytes": b8, "bf16_bytes": bb, "w4_bytes": b4, "fp8_max_rel_vs_fp64": rel,
                    "fp8_ms_per_cycle": t8, "bf16_ms_per_cycle": tb, "w4_ms_per_cycle": t4}
            out.append(case)
            print(f"gemm {name:10s} M={M:3d}  fp8 {us8:8.2f} us ({case['fp8_hbm_share']:.2f})  bf16 {usb:8.2f} us "
                  f"({case['bf16_hbm_share']:.2f})  w4 {us4:8.2f} us ({case['w4_hbm_share']:.2f})  "
                  f"fp8/bf16 {case['fp8_speedup_vs_bf16']:.2f}x  max_rel {rel:.1e}", flush=True)
        del w8, wbf, w4
        torch.cuda.empty_cache()
    return out


def engine_cases(args):
    from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
    cfg = dataclasses.replace(LLAMA3_8B, n_layers=args.layers)
    S = args.seq
    fmts = ("fp8", "bf16")
    out = []
    for B in (1, 16):
        engs = {}
        for fmt in fmts:
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

        t = alternate([stepper(engs[f], saved[f]) for f in fmts], 3, args.steps, args.windows)
        for f, tf in zip(fmts, t):
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
        raise SystemExit("fp8_linear_bench.py measures on a GPU; none is visible")
    lib = _lib.load()
    res = {"gpu": gpu_info(), "datasheet_tb_s": DATASHEET_TB_S, "nrep": NREP}
    print(json.dumps(res["gpu"]), flush=True)
    res["gemm"] = gemm_cases(args, lib)
    if not args.skip_engine:
        res["engine"] = engine_cases(args)
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_linear_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
