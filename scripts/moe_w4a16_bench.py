"""4-bit MoE experts (W4A16, groups of 128) against bf16 experts on one GPU, both paths alternating in one run:

  experts  fused_experts on the Mixtral-8x7B layer shape (E = 8, top-2, dim 4096, F 14336) at T = 1, 16, 64, 256:
           chitu_b200_fused_experts_w4a16 against chitu_b200_fused_experts (bf16) on the dequantised weights.  Each
           timed call cycles over NL layers' weights so that none sits in L2.  Reported: us per call, distinct experts,
           GB/s on the algorithmic bytes (each distinct expert's packed weights + scales + zeros, or bf16 weights, once,
           plus x and out) and their share of the 3.35 TB/s data-sheet HBM bandwidth, the speed-up, and max_rel of the
           W4 output against bf16 on the dequantised weights.
  engine   the full 32-layer Mixtral-8x7B in W4 at tp_size=1 on one GPU, context 4096, bs 1 and 16, the step replayed as
           one CUDA graph: ms per step, tok/s, algorithmic GB per step and its share of 3.35 TB/s, and
           torch.cuda.max_memory_allocated (building included, and over the timed steps alone).
  layers   bf16 and W4 engines with --cmp-layers layers at tp_size=1 (where both fit), alternating: the per-layer cost of
           the two formats in the same run.

Timings: the median, min and max over `--windows` CUDA-event windows after warm-up.

  python scripts/moe_w4a16_bench.py --out DIR          writes DIR/moe_w4a16_bench.json

Reads the device name, power limit and max SM clock (nvidia-smi --query-gpu, a query only); changes no device setting.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from paged_prefill_bench import gpu_info, max_rel  # noqa: E402
from w4a16_bench import DATASHEET_TB_S, alternate  # noqa: E402

from chitu_b200 import _lib  # noqa: E402
from chitu_b200._lib import check, current_stream, ptr  # noqa: E402
from chitu_b200.quantize import w4a16 as W  # noqa: E402

BF = torch.bfloat16
E, TOPK, DIM, F = 8, 2, 4096, 14336
TS = (1, 16, 64, 256)
NL = 4                        # layers' weights cycled per timed call: 4 x 0.7 GB (W4) > the 50 MB L2
DEV = "cuda:0"


def w4_bytes(n):
    return n // 2 + n // 128 * 3       # packed weight, bf16 scale and uint8 zero per group


def expert_cases(args, lib):
    g = torch.Generator(device=DEV).manual_seed(0)

    def stack(N, K):
        parts = [W.quantize_rtn(torch.randn(N, K, generator=g, device=DEV) * 0.02, BF) for _ in range(E)]
        return tuple(torch.stack(t) for t in zip(*parts))

    w4 = [(stack(2 * F, DIM), stack(DIM, F)) for _ in range(NL)]
    wbf = [(W.dequantize(*a), W.dequantize(*b)) for a, b in w4]
    out = []
    for T in TS:
        x = torch.randn(T, DIM, generator=g, device=DEV).to(BF)
        logits = torch.randn(T, E, generator=g, device=DEV)
        tw, ids = torch.topk(torch.softmax(logits, dim=-1), TOPK, dim=-1)
        tw = (tw / tw.sum(dim=-1, keepdim=True)).to(BF).contiguous()
        ids = ids.contiguous()
        distinct = len(torch.unique(ids))
        y4, yb = torch.empty(T, DIM, dtype=BF, device=DEV), torch.empty(T, DIM, dtype=BF, device=DEV)
        ws = torch.zeros(lib.chitu_b200_moe_workspace_bytes(T, TOPK, E, 2 * F, DIM), dtype=torch.uint8, device=DEV)
        st = current_stream()
        route = (ptr(tw), _lib.CB_BF16, ptr(ids), _lib.CB_I64, T, TOPK, E, 2 * F, DIM)

        def run_w4(i):
            (q1, s1, z1), (q2, s2, z2) = w4[i]
            return lib.chitu_b200_fused_experts_w4a16(ptr(x), ptr(q1), ptr(s1), ptr(z1), ptr(q2), ptr(s2), ptr(z2), *route,
                                                      ptr(y4), None, ptr(ws), ws.numel(), st)

        def run_bf(i):
            return lib.chitu_b200_fused_experts(ptr(x), ptr(wbf[i][0]), ptr(wbf[i][1]), None, None, *route, 0, ptr(yb),
                                                None, ptr(ws), ws.numel(), st)

        check(run_w4(0), "fused_experts_w4a16"), check(run_bf(0), "fused_experts")
        torch.cuda.synchronize()
        rel = max_rel(y4, yb)

        def cycle(fn):
            return lambda: [fn(i) for i in range(NL)]

        t4, tb = alternate([cycle(run_w4), cycle(run_bf)], 2, args.reps, args.windows)
        us4, usb = t4["median"] * 1e3 / NL, tb["median"] * 1e3 / NL
        io = 2 * T * DIM * 2
        b4 = distinct * w4_bytes(3 * F * DIM) + io
        bb = distinct * 3 * F * DIM * 2 + io
        case = {"T": T, "distinct_experts": distinct, "w4_us": us4, "bf16_us": usb, "speedup": usb / us4,
                "w4_gb_s": b4 / us4 / 1e3, "bf16_gb_s": bb / usb / 1e3,
                "w4_hbm_share": b4 / us4 / 1e3 / (DATASHEET_TB_S * 1e3),
                "bf16_hbm_share": bb / usb / 1e3 / (DATASHEET_TB_S * 1e3), "w4_bytes": b4, "bf16_bytes": bb,
                "max_rel_vs_bf16": rel, "w4_ms_per_cycle": t4, "bf16_ms_per_cycle": tb}
        out.append(case)
        print(f"experts T={T:3d} distinct={distinct}  w4 {us4:8.1f} us {case['w4_gb_s']:6.0f} GB/s "
              f"({case['w4_hbm_share']:.2f})  bf16 {usb:8.1f} us {case['bf16_gb_s']:6.0f} GB/s "
              f"({case['bf16_hbm_share']:.2f})  speed-up {case['speedup']:.2f}x  max_rel {rel:.1e}", flush=True)
    del w4, wbf
    torch.cuda.empty_cache()
    return out


def _engine(cfg, B, S, fmt):
    from chitu_b200.engine_mixtral import MixtralDecodeEngine
    e = MixtralDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, device=DEV, tp_size=1, weight_format=fmt)
    e.set_synthetic_context(S)
    e.capture()
    return e


def _stepper(e):
    s0 = e.seq_lens.clone()

    def fn():
        e.seq_lens.copy_(s0)              # the same context length every step (a copy the graph does not include)
        e.graph.replay()
    return fn


def _record(e, fmt, B, S, tf):
    ms = tf["median"]
    distinct = e.distinct_experts_per_layer()
    nbytes = e.algorithmic_bytes(S, distinct)
    return {"weight_format": fmt, "bs": B, "seq": S, "layers": e.cfg.n_layers, "ms_per_step": ms, "ms_spread": tf,
            "ms_per_layer": ms / e.cfg.n_layers, "tok_s": B / ms * 1e3, "distinct_experts_per_layer": distinct,
            "step_gb": nbytes / 1e9, "hbm_share": nbytes / (ms * 1e-3) / (DATASHEET_TB_S * 1e12),
            "launches_per_step": e.launches_per_step}


def full_model_cases(args):
    from chitu_b200.engine_mixtral import MIXTRAL_8X7B
    S, out = args.seq, []
    for B in (1, 16):
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        e = _engine(MIXTRAL_8X7B, B, S, "w4a16")
        peak_build = torch.cuda.max_memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        (tf,) = alternate([_stepper(e)], 3, args.steps, args.windows)
        case = _record(e, "w4a16", B, S, tf)
        case.update(max_memory_allocated_gb=peak_build / 1e9, steps_max_memory_allocated_gb=torch.cuda.max_memory_allocated() / 1e9,
                    memory_allocated_gb=torch.cuda.memory_allocated() / 1e9)
        out.append(case)
        print(f"mixtral-8x7b w4a16 32 layers tp1 bs={B:2d} S={S}  {case['ms_per_step']:7.3f} ms/step  "
              f"{case['tok_s']:8.1f} tok/s  {case['step_gb']:.2f} GB/step  share {case['hbm_share']:.2f}  "
              f"max_memory_allocated {case['max_memory_allocated_gb']:.1f} GB (steps {case['steps_max_memory_allocated_gb']:.1f})",
              flush=True)
        del e
    torch.cuda.empty_cache()
    return out


def layer_cases(args):
    from chitu_b200.engine_mixtral import MixtralConfig
    cfg = MixtralConfig(n_layers=args.cmp_layers)
    S, out = args.seq, []
    for B in (1, 16):
        engs = {f: _engine(cfg, B, S, f) for f in ("w4a16", "bf16")}
        t = alternate([_stepper(engs[f]) for f in engs], 3, args.steps, args.windows)
        for f, tf in zip(engs, t):
            case = _record(engs[f], f, B, S, tf)
            out.append(case)
            print(f"mixtral {cfg.n_layers} layers tp1 {f:6s} bs={B:2d}  {case['ms_per_step']:7.3f} ms/step "
                  f"({case['ms_per_layer']:.3f} ms/layer)  {case['step_gb']:.2f} GB/step  share {case['hbm_share']:.2f}",
                  flush=True)
        del engs
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=10, help="weight cycles per fused-experts timing window")
    ap.add_argument("--steps", type=int, default=20, help="graph replays per engine timing window")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--cmp-layers", type=int, default=8)
    ap.add_argument("--skip-engine", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_w4a16_bench.py measures on a GPU; none is visible")
    lib = _lib.load()
    res = {"gpu": gpu_info(), "datasheet_tb_s": DATASHEET_TB_S, "layers_cycled": NL}
    print(json.dumps(res["gpu"]), flush=True)
    res["experts"] = expert_cases(args, lib)
    if not args.skip_engine:
        res["full_model"] = full_model_cases(args)
        res["layers"] = layer_cases(args)
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "moe_w4a16_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
