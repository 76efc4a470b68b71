#!/usr/bin/env python
"""bench.py — decode tokens/s of the hot path (BASELINE.json metric) + roofline + CPU baseline.

    python bench.py --gpus N --steps K --warmup W            # our arm (libchitu_b200, CUDA)
    python bench.py --impl reference --gpus N --steps K ...  # the reference's CPU path (oracle port)

`value` (every N): LLaMA-3-8B bf16 paged-KV decode (BASELINE.json configs[1]), bs=16, seq=4096, tensor-parallel
over the N ranks (column/row shards + all-reduce exactly where chitu/tensor_parallel.py:166 reduces) -> strong scaling.
The SAME JSON line also carries the north-star configuration (BASELINE.json configs[3]) under the driver's clock:
    N = 1 : "deepseek_r1_shard"  ONE rank's tp=16 shard (42 GB of FP8 weights, 61 layers) without collectives: the
            smallest tensor-parallel degree at which the FP8 model fits 80 GB H100s (two 8-GPU nodes)
    N = 2/4/8: "deepseek_r1_reduced" tp=N with a reduced layer count (12 / 24 / 40 of 61 layers) so that one rank's FP8
            weights stay within ~55-62 GB of an 80 GB H100: the full 61 layers need ~85 GB per rank at tp=8
each with tokens/s, ms/step, counted distinct experts, algorithmic bytes and the step's fraction of the HBM roofline
against the measured peak (when MEASURED_PEAKS.json exists) or the H100 SXM data sheet's 3.35 TB/s, and its own clocks
record.  A "step" = one decode step of the whole model for the whole batch.

--dump-outputs DIR writes, after the timed steps, what the last timed step of every engine returned to its caller
(logits and next tokens, float32 / float64 .npy; logits over 12 MB as a fixed, seeded sample of vocabulary columns; at
most 64 MB in all; with tensor parallelism rank 0's vocabulary shard of the logits).  Inputs are seeded, so two builds
given the same arguments can be compared output for output.
"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "decode tokens/s at bs=16 (LLaMA-3-8B bf16 paged-KV, seq=4096)"
UNIT = "tokens/s"
NOMINAL_HBM_GBS = 3350.0          # H100 SXM data sheet (HBM3)


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return NOMINAL_HBM_GBS, "H100 SXM data sheet (not measured)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region.

    The query loop is started before the warm-up (nvidia-smi needs ~100 ms to initialise); a reader thread
    stamps every sample on arrival and `stop()` keeps the samples that fall into [mark_begin, mark_end].
    A window shorter than a few sampling periods is topped up by the caller with untimed replays of the SAME
    step (the same count on every rank) before `mark_end()`."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index=0):
        self.gpu, self.proc, self.samples, self.t0, self.t1, self.extended = gpu_index, None, [], None, None, False

    def start(self):
        import threading
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "50", "-i", str(self.gpu)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True, bufsize=1)
        except Exception:
            self.proc = None
            return

        def reader():
            for line in self.proc.stdout:
                self.samples.append((time.time(), line))
        self.thread = threading.Thread(target=reader, daemon=True)
        self.thread.start()

    def mark_begin(self):
        self.t0 = time.time()

    def mark_end(self):
        self.t1 = time.time()

    def in_window(self):
        return [l for (t, l) in self.samples if self.t0 is not None and t >= self.t0 and (self.t1 is None or t <= self.t1)]

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"], "samples": 0}
        lines = self.in_window()
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, smax, reasons = [], [], set()
        for line in lines:
            f = [x.strip() for x in line.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                smax.append(float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        out = {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(smax) if smax else None,
               "reasons": sorted(reasons), "samples": len(sm)}
        if self.extended:
            out["note"] = "timed region shorter than the sampling period: topped up with untimed replays of the same step"
        return out


def bytes_per_step(cfg, B, S, tp):
    """Algorithmic HBM bytes per decode step per GPU (SURVEY.md §8d): every weight byte once,
    KV rows once, bf16 head; activations ignored."""
    D = cfg.head_dim
    Hq, Hkv, F = cfg.n_heads // tp, cfg.n_kv_heads // tp, cfg.ffn_dim // tp
    w_layer = ((Hq + 2 * Hkv) * D * cfg.dim + cfg.dim * Hq * D + 3 * F * cfg.dim) * 2
    kv_layer = B * (S + 1) * 2 * Hkv * D * 2
    head = (cfg.vocab_size // tp) * cfg.dim * 2
    return cfg.n_layers * (w_layer + kv_layer) + head, w_layer, kv_layer


def dist_env():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    return world, rank, local


DUMP_BUDGET_BYTES = 64 << 20          # --dump-outputs writes at most this much in all
DUMP_LOGITS_BYTES = 12 << 20          # per logits array; larger ones are sampled


def dump_outputs(args, label, eng, next_tokens):
    """--dump-outputs: the logits and next tokens of the engine's last timed step -> DIR/<label>_*.npy.  Logits larger
    than DUMP_LOGITS_BYTES (float32) keep a fixed, seeded sample of vocabulary columns, written beside them as
    <label>_logits_cols.npy; nothing more is written once DUMP_BUDGET_BYTES is used.  With tensor parallelism the logits
    are rank 0's vocabulary shard (the next tokens are global)."""
    import numpy as np
    import torch
    if not getattr(args, "dump_outputs", None):
        return
    os.makedirs(args.dump_outputs, exist_ok=True)
    logits = eng.logits.float()
    rows, cols = logits.shape
    arrays = {}
    if rows * cols * 4 > DUMP_LOGITS_BYTES:
        k = max(1, DUMP_LOGITS_BYTES // (rows * 4))
        pick = torch.randperm(cols, generator=torch.Generator().manual_seed(0))[:k].sort().values
        arrays["logits"] = logits[:, pick.to(logits.device)].cpu().numpy()
        arrays["logits_cols"] = pick.numpy().astype(np.float64)
    else:
        arrays["logits"] = logits.cpu().numpy()
    arrays["next_tokens"] = next_tokens.cpu().numpy().astype(np.float64)
    used = getattr(args, "_dump_bytes", 0)
    for name, a in arrays.items():
        if used + a.nbytes > DUMP_BUDGET_BYTES:
            print(f"--dump-outputs: {label}_{name} skipped (the {DUMP_BUDGET_BYTES >> 20} MB budget is used)", file=sys.stderr)
            continue
        np.save(os.path.join(args.dump_outputs, f"{label}_{name}.npy"), a)
        used += a.nbytes
    args._dump_bytes = used


def time_engine(eng, B, S, args, world, dev, sampler=None, label=None):
    """W untimed warm-up steps, K device-timed steps (CUDA events between barriers, max over ranks), then K end-to-end
    steps through the public `decode()` (pinned host tokens in, host tokens out).  Returns ms/step, e2e ms/step, clocks.
    With --dump-outputs, what the last end-to-end step returned is written under `label`."""
    import torch
    import torch.distributed as dist

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    tokens_host = torch.randint(100, 1000, (B,), dtype=torch.int64,                  # gen_reqs_fake range
                                generator=torch.Generator().manual_seed(B)).pin_memory()
    eng.tokens.copy_(tokens_host)
    if sampler is not None:
        sampler.start()
    for _ in range(args.warmup):
        eng.step()
    eng.seq_lens.fill_(S)
    barrier()
    if sampler is not None:
        sampler.mark_begin()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        eng.step()
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    eng.seq_lens.fill_(S)
    for _ in range(3):
        eng.decode(tokens_host)
    eng.seq_lens.fill_(S)
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        nxt = eng.decode(tokens_host)    # H2D tokens + graph replay + D2H next tokens (sync)
    barrier()
    e2e_ms = (time.perf_counter() - t0) * 1e3
    if label is not None and args.steps > 0 and int(os.environ.get("RANK", "0")) == 0:
        dump_outputs(args, label, eng, nxt)
    t = torch.tensor([ms, e2e_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, e2e_ms = t.tolist()
    clocks = None
    # clocks: the window covers both timed regions (the same step); a window shorter than ~0.4 s is topped up with
    # the same number of untimed replays on every rank
    extra = max(0, int(400.0 / max(ms / args.steps, 1e-3)) - 2 * args.steps)
    eng.seq_lens.fill_(S)
    for i in range(extra):
        eng.step()
        if (i + 1) % 64 == 0:            # never outgrow the KV capacity the engine was built with
            eng.seq_lens.fill_(S)
    barrier()
    if sampler is not None:
        sampler.mark_end()
        sampler.extended = extra > 0
        clocks = sampler.stop()
    eng.seq_lens.fill_(S)
    return ms / args.steps, e2e_ms / args.steps, clocks


def gemm_table(eng, B, args):
    """Launch-weighted roofline of the weight-streaming GEMM template (the dominant kernel: ~2/3 of the step): each of
    the four LLaMA layer shapes is replayed over the 32 layers' DISTINCT weights (GBs, far larger than L2) inside one
    CUDA graph (so host launch cost is not in the number) and timed with CUDA events."""
    import torch

    from chitu_b200 import _lib
    from chitu_b200._lib import check, current_stream, ptr
    lib = _lib.load()
    M = B
    rows = []
    shapes = [("wqkv", eng.xn, eng.qkv), ("wo", eng.attn_out, eng.h2), ("w13", eng.xn, eng.gate_up), ("w2", eng.act, eng.h2)]
    for name, x, y in shapes:
        ws = [lw[name] for lw in eng.layers]
        N, K = ws[0].shape

        # the engine's own launch: w13 carries the SiluAndMul epilogue (interleaved gate / up rows) unless switched off
        pairs = name == "w13" and getattr(eng, "fuse_silu", False)

        def run_all():
            for w in ws:
                if pairs:
                    check(lib.chitu_b200_linear_bf16_silu_pairs(ptr(x), ptr(w), ptr(eng.act), M, N, K, ptr(eng.lin_ws),
                                                                eng.lin_ws.numel(), current_stream()), "linear_silu_pairs")
                else:
                    check(lib.chitu_b200_linear_bf16(ptr(x), ptr(w), None, None, ptr(y), M, N, K, _lib.CB_BF16,
                                                     ptr(eng.lin_ws), eng.lin_ws.numel(), args.linear_impl,
                                                     current_stream()), "linear")
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run_all()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run_all()
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 5
        k0.record()
        for _ in range(reps):
            g.replay()
        k1.record()
        torch.cuda.synchronize()
        k_ms = k0.elapsed_time(k1) / (reps * len(ws))
        rows.append(dict(name=f"linear_bf16{'_silu_pairs' if pairs else ''} {name} M={M} N={N} K={K}", ms=k_ms,
                         bytes=N * K * 2 + M * K * 2 + (M * N if pairs else M * N * 2), launches_per_step=len(ws)))
        del g
    return rows


def run_llama(args, world, rank, local, pg):
    import torch

    from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
    dev = f"cuda:{local}"
    cfg = LLAMA3_8B
    S = args.seq
    results = {}
    for B in (args.bs, 1):
        eng = LlamaDecodeEngine(cfg, max_reqs=B, max_seq_len=S + max(512, args.steps + args.warmup + 128), device=dev,
                                page_size=256, tp_rank=rank, tp_size=world, process_group=pg,
                                linear_impl=args.linear_impl, use_fused_allreduce=not args.nccl_allreduce)
        eng.set_synthetic_context(S)
        eng.capture()
        sampler = ClockSampler(local) if (B == args.bs and rank == 0) else None
        ms, e2e_ms, clocks = time_engine(eng, B, S, args, world, dev, sampler, label=f"llama3_8b_bs{B}")
        results[B] = dict(ms_per_step=ms, e2e_ms_per_step=e2e_ms, launches_per_step=eng.launches_per_step, clocks=clocks)
        if B == args.bs and world == 1:
            results["gemms"] = gemm_table(eng, B, args)
        del eng
        torch.cuda.empty_cache()
    return results


def deepseek_variant(world):
    """(label, tp, n_layers, n_dense, note) of the DeepSeek-R1 block reported at this GPU count (SURVEY §8e)."""
    if world == 1:
        return ("deepseek_r1_shard", 16, 61, 3,
                "ONE rank's tp=16 shard of the full 61-layer model on one GPU, no collectives (per-rank kernel time of the "
                "tp=16 configuration that fits 80 GB H100s; NOT a 1-GPU DeepSeek-R1)")
    # per rank: a MoE layer holds 1.42 GB x (8 / tp) of FP8 experts; the layer count keeps the weights within ~62 GB so
    # that the KV cache and workspaces fit an 80 GB H100 (61 layers at tp=8 would need ~85 GB)
    layers = {2: 12, 4: 24, 8: 40}.get(world, 8)
    return ("deepseek_r1_reduced", world, layers, 3,
            f"REDUCED model: {layers} of 61 layers (3 dense + {layers - 3} MoE) at tp={world}, sized for 80 GB per GPU — the "
            "full FP8 model needs tp >= 16 on 80 GB GPUs; tokens/s of this variant are not comparable with the 61-layer numbers")


def run_deepseek_block(args, world, rank, local, pg, tp=None, layers=None):
    """DeepSeek-R1 FP8 MLA-absorb paged decode at bs = args.bs and bs = 1 -> dict (rank 0) or None."""
    import torch

    from chitu_b200.engine_deepseek import DEEPSEEK_R1, DeepSeekDecodeEngine
    dev = f"cuda:{local}"
    label, v_tp, v_layers, n_dense, note = deepseek_variant(world)
    tp = tp or v_tp
    layers = layers or v_layers
    cfg = dataclasses.replace(DEEPSEEK_R1, n_layers=layers, n_dense_layers=min(n_dense, layers))
    S = args.seq
    peak, peak_src = peaks()
    out = {}
    for B in (args.bs, 1):
        eng = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=S + max(256, args.steps + args.warmup + 128), device=dev,
                                   tp_rank=rank if world > 1 else 0, tp_size=tp, process_group=pg,
                                   use_fused_allreduce=not args.nccl_allreduce)
        eng.set_synthetic_context(S)
        eng.capture()
        sampler = ClockSampler(local) if rank == 0 else None
        ms, e2e_ms, clocks = time_engine(eng, B, S, args, world, dev, sampler, label=f"{label}_bs{B}")
        distinct = eng.distinct_experts_per_layer()
        nbytes = eng.algorithmic_bytes(S, distinct)
        gbs = nbytes / (ms * 1e-3) / 1e9
        out[B] = {"tokens_per_s": B / (ms * 1e-3), "ms_per_step": ms, "e2e_tokens_per_s": B / (e2e_ms * 1e-3),
                  "distinct_experts_per_layer": distinct, "algorithmic_bytes_per_rank": nbytes,
                  "achieved_gbs_per_rank": gbs, "step_frac_of_measured_peak": gbs / peak,
                  "step_frac_of_datasheet_hbm": gbs / NOMINAL_HBM_GBS, "launches_per_step": int(eng.launches_per_step),
                  "clocks": clocks}
        del eng
        torch.cuda.empty_cache()
    if rank != 0:
        return None
    return {"label": label, "note": note, "model": "DeepSeek-R1 671B shapes (config/models/DeepSeek-R1.yaml), FP8 block-scaled "
            "w8a8 linears + experts, MLA absorb paged decode (page 64), synthetic weights", "tp": tp, "n_gpus": world,
            "n_layers": layers, "seq_len": S, "dtype": "fp8_e4m3 (bf16 gate/head)", "steps": args.steps, "warmup": args.warmup,
            "peak_gbs": peak, "peak_source": peak_src,
            "allreduce": "none" if world == 1 else ("nccl" if args.nccl_allreduce else
                                                     "fused one-shot NVLink peer-memory all-reduce + residual + RMSNorm + FP8 quant"),
            f"bs{args.bs}": out[args.bs], "bs1": out[1]}


def run_cuda(args):
    import torch
    import torch.distributed as dist

    from chitu_b200.engine import LLAMA3_8B

    world, rank, local = dist_env()
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    pg = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(dev))
        pg = dist.group.WORLD

    check = None
    if world > 1 and not args.no_mgpu_check:
        # witnessed by the driver's scaling run: fused all-reduce vs NCCL + torch reference math on this world size
        from scripts.mgpu_check import run_checks
        check = run_checks(rank, world, dev, engines=False)
    cfg = LLAMA3_8B
    S = args.seq
    results = run_llama(args, world, rank, local, pg)
    ds = None
    if not args.no_deepseek:
        ds = run_deepseek_block(args, world, rank, local, pg)
    if rank != 0:
        return
    B = args.bs
    r = results[B]
    total_bytes, w_layer, kv_layer = bytes_per_step(cfg, B, S, world)
    peak, peak_src = peaks()
    step_gbs = total_bytes / (r["ms_per_step"] * 1e-3) / 1e9
    roof = {"bound": "hbm", "peak": peak, "unit": "GB/s", "peak_source": peak_src,
            "step_achieved_gbs": step_gbs, "step_frac": step_gbs / peak, "step_frac_of_datasheet_hbm": step_gbs / NOMINAL_HBM_GBS,
            "step_algorithmic_bytes": total_bytes}
    if "gemms" in results:
        g = results["gemms"]
        tot_b = sum(x["bytes"] * x["launches_per_step"] for x in g)
        tot_ms = sum(x["ms"] * x["launches_per_step"] for x in g)
        best = max(g, key=lambda x: x["bytes"] / x["ms"])
        achieved = tot_b / (tot_ms * 1e-3) / 1e9
        roof.update({"kernel": "tc_gemm_kernel<bf16,16> (wgmma swap-AB weight-streaming GEMM), launch-weighted over the "
                               "four layer shapes x 32 layers (128 of the step's launches)",
                     "achieved": achieved, "frac": achieved / peak, "kernel_ms_per_step": tot_ms,
                     "kernel_share_of_step": tot_ms / r["ms_per_step"], "best_kernel": best["name"],
                     "per_shape": [{"name": x["name"], "us": x["ms"] * 1e3, "gbs": x["bytes"] / (x["ms"] * 1e-3) / 1e9,
                                    "frac": x["bytes"] / (x["ms"] * 1e-3) / 1e9 / peak, "bytes": x["bytes"]} for x in g]})
    else:
        roof.update({"kernel": "whole decode step (per-rank algorithmic bytes / step time)", "achieved": step_gbs,
                     "frac": step_gbs / peak})
    line = {
        "metric": METRIC, "value": B / (r["ms_per_step"] * 1e-3), "unit": UNIT, "n_gpus": world,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": r["ms_per_step"], "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": f"LLaMA-3-8B bf16 paged-KV decode, bs={B}, seq={S}, page=256, tp={world}",
                   "global_batch": B, "seq_len": S, "parallelism": f"tp{world}",
                   "l2": "inputs larger than L2: %.1f GB of weights+KV streamed per step vs 50 MB L2" % (total_bytes / 1e9),
                   "cuda_graph": True, "linear_impl": args.linear_impl,
                   "allreduce": "none" if world == 1 else ("nccl" if args.nccl_allreduce else "fused one-shot NVLink peer-memory all-reduce + residual + RMSNorm")},
        "bs1": {"value": 1 / (results[1]["ms_per_step"] * 1e-3), "ms_per_step": results[1]["ms_per_step"],
                "e2e_value": 1 / (results[1]["e2e_ms_per_step"] * 1e-3),
                "launches_per_step": int(results[1]["launches_per_step"]),
                "hbm_frac_of_step_roofline": (bytes_per_step(cfg, 1, S, world)[0] / (results[1]["ms_per_step"] * 1e-3) / 1e9) / peak},
        "e2e": {"value": B / (r["e2e_ms_per_step"] * 1e-3), "unit": UNIT, "h2d_bytes_per_step": B * 8,
                "d2h_bytes_per_step": B * 8},
        "gpu_launches": int(r["launches_per_step"]) * args.steps,
        "launches_per_step": int(r["launches_per_step"]),
        "clocks": r["clocks"],
        "roofline": roof,
    }
    if ds is not None:
        line[ds["label"]] = ds
    if check is not None:
        line["multi_gpu_parity"] = check
    if not args.no_cpu_baseline and world == 1:
        line["cpu_baseline"] = cpu_baseline_with_reference(B, S)
    print(json.dumps(line))


def run_deepseek(args):
    """--workload deepseek-r1: the DeepSeek block alone as the JSON line's metric (BASELINE.json configs[3])."""
    import torch
    import torch.distributed as dist

    world, rank, local = dist_env()
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    pg = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device(dev))
        pg = dist.group.WORLD
    ds = run_deepseek_block(args, world, rank, local, pg, tp=args.tp or None, layers=args.layers or None)
    if rank != 0:
        return
    B = args.bs
    r = ds[f"bs{B}"]
    line = {
        "metric": "decode tokens/s at bs=%d (DeepSeek-R1 671B FP8 MLA-absorb paged decode, tp=%d, seq=%d)" % (B, ds["tp"], args.seq),
        "value": r["tokens_per_s"], "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": r["ms_per_step"], "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
        "dtype": "fp8_e4m3", "data": "synthetic",
        "config": {"workload": "DeepSeek-R1 FP8 block-scaled w8a8, MLA absorb paged decode, bs=%d seq=%d, %d layers, tp=%d — %s"
                               % (B, args.seq, ds["n_layers"], ds["tp"], ds["note"]),
                   "global_batch": B, "seq_len": args.seq, "parallelism": f"tp{ds['tp']}", "cuda_graph": True,
                   "allreduce": ds["allreduce"], "distinct_experts_per_layer": r["distinct_experts_per_layer"],
                   "l2": "inputs larger than L2: %.1f GB streamed per step" % (r["algorithmic_bytes_per_rank"] / 1e9)},
        "bs1": ds["bs1"],
        "e2e": {"value": r["e2e_tokens_per_s"], "unit": UNIT, "h2d_bytes_per_step": B * 8, "d2h_bytes_per_step": B * 8},
        "gpu_launches": r["launches_per_step"] * args.steps, "launches_per_step": r["launches_per_step"],
        "clocks": r["clocks"],
        "roofline": {"bound": "hbm", "achieved": r["achieved_gbs_per_rank"], "peak": ds["peak_gbs"], "unit": "GB/s",
                     "frac": r["step_frac_of_measured_peak"], "traffic": None,
                     "kernel": "whole decode step (per-rank algorithmic bytes / step time)", "peak_source": ds["peak_source"],
                     "step_frac_of_datasheet_hbm": r["step_frac_of_datasheet_hbm"],
                     "step_algorithmic_bytes": r["algorithmic_bytes_per_rank"]},
    }
    print(json.dumps(line))


def run_sweep(args):
    """--workload w8a8-sweep (BASELINE.json configs[4], README.md:63-67): bs in {1,16,256} for (a) the FP8 block-scaled
    DeepSeek-R1 tp=8 shard step (reduced layers), (b) the dense FP8 linears and (c) the INT8 W8A8Linear kernels at the
    same (N,K), each with its fraction of the HBM roofline."""
    import torch

    from chitu_b200 import _lib
    from chitu_b200._lib import check, current_stream, ptr
    from chitu_b200.engine_deepseek import DEEPSEEK_R1, DeepSeekDecodeEngine, quantize_fp8_block
    world, rank, local = dist_env()
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    lib = _lib.load()
    peak, peak_src = peaks()
    S = args.seq
    shapes = [("wqkv_a", 2112, 7168), ("wq_b", 3072, 1536), ("wo", 7168, 2048), ("dense_w13", 4608, 7168), ("dense_w2", 7168, 2304)]
    out = {"label": "w8a8_sweep", "peak_gbs": peak, "peak_source": peak_src, "ops": [], "steps": []}
    nrep = 24                                             # distinct weights per shape: 24 x (4.7 .. 33 MB) >> L2 for the big ones
    for name, N, K in shapes:
        g = torch.Generator(device=dev).manual_seed(N + K)
        wq = [quantize_fp8_block(torch.randn(N, K, generator=g, device=dev) * 0.02) for _ in range(nrep)]
        wi = [(torch.randint(-127, 128, (N, K), generator=g, device=dev, dtype=torch.int32).to(torch.int8),
               torch.rand(N, generator=g, device=dev) * 0.01) for _ in range(nrep)]
        for M in (1, 16, 256):
            x = torch.randn(M, K, generator=g, device=dev).bfloat16()
            xq = torch.empty(M, K, dtype=torch.float8_e4m3fn, device=dev)
            xs = torch.empty(M, K // 128, dtype=torch.float32, device=dev)
            check(lib.chitu_b200_act_quant_fp8(ptr(x), ptr(xq), ptr(xs), M, K, 128, 0, 0.0, _lib.CB_BF16, current_stream()), "q")
            xi = torch.randint(-127, 128, (M, K), generator=g, device=dev, dtype=torch.int32).to(torch.int8)
            xis = torch.rand(M, generator=g, device=dev) * 0.01
            y = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
            yh = torch.empty(M, N, dtype=torch.float16, device=dev)
            ws = torch.zeros(max(lib.chitu_b200_linear_workspace_bytes(M, N), 256), dtype=torch.uint8, device=dev)

            def f_fp8():
                for w, s in wq:
                    check(lib.chitu_b200_fp8_gemm(ptr(xq), ptr(xs), ptr(w), ptr(s), ptr(y), M, N, K, None, ptr(ws),
                                                  ws.numel(), 0, current_stream()), "fp8")

            def f_i8():
                for w, s in wi:
                    check(lib.chitu_b200_w8a8_gemm(ptr(yh), ptr(xi), ptr(w), ptr(xis), ptr(s), None, M, N, K, ptr(ws),
                                                   ws.numel(), 0, current_stream()), "i8")
            for kind, fn in (("fp8_block", f_fp8), ("int8_w8a8", f_i8)):
                st = torch.cuda.Stream()
                st.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(st):
                    fn()
                torch.cuda.current_stream().wait_stream(st)
                torch.cuda.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    fn()
                for _ in range(3):
                    gr.replay()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(5):
                    gr.replay()
                e1.record()
                torch.cuda.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / (5 * nrep)
                nbytes = N * K + M * K + M * N * 2 + (0 if kind == "int8_w8a8" else (N // 128 + 1) * (K // 128) * 4)
                flops = 2.0 * M * N * K
                out["ops"].append({"op": name, "kind": kind, "M": M, "N": N, "K": K, "us": us, "gbs": nbytes / us / 1e3,
                                   "frac_of_hbm_peak": nbytes / us / 1e3 / peak, "tflops": flops / us / 1e6})
                del gr
        del wq, wi
        torch.cuda.empty_cache()
    layers = args.layers or 8
    cfg = dataclasses.replace(DEEPSEEK_R1, n_layers=layers, n_dense_layers=min(3, layers))
    for B in (1, 16, 256):
        eng = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=S + max(256, args.steps + args.warmup + 128), device=dev, tp_rank=0,
                                   tp_size=8, process_group=None)
        eng.set_synthetic_context(S)
        eng.capture()
        sampler = ClockSampler(local)
        ms, e2e_ms, clocks = time_engine(eng, B, S, args, 1, dev, sampler)
        distinct = eng.distinct_experts_per_layer()
        nbytes = eng.algorithmic_bytes(S, distinct)
        out["steps"].append({"bs": B, "n_layers": layers, "tp_shard": 8, "ms_per_step": ms, "tokens_per_s": B / (ms * 1e-3),
                             "distinct_experts_per_layer": distinct, "algorithmic_bytes": nbytes,
                             "step_frac_of_measured_peak": nbytes / (ms * 1e-3) / 1e9 / peak,
                             "launches_per_step": int(eng.launches_per_step), "clocks": clocks})
        del eng
        torch.cuda.empty_cache()
    print(json.dumps(out))


def host_cores():
    """Usable host threads: the scheduler affinity mask capped by the cgroup CPU quota (os.cpu_count() alone reports
    every core of the node even inside a quota-limited container, and oversubscribed BLAS threads are slower)."""
    n = os.cpu_count() or 1
    try:
        n = min(n, len(os.sched_getaffinity(0)))
    except Exception:
        pass
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            quota, period = f.read().split()[:2]
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except Exception:
        pass
    return max(1, n)


class CpuSample:
    kind = "port"
    """The reference's decode step (oracle port of models/model_llama.py + RefAttnBackend arithmetic) on the host cores,
    on a BOUNDED sample of the workload: one timed step = ONE transformer layer of the bs/seq workload (two layers'
    weights and caches are allocated and alternated); the head is timed separately.  Full-depth step time =
    n_layers x (measured layer time) + (measured head time)."""

    def __init__(self, cfg, B, S, page=256, threads=None):
        import torch

        from oracle import chitu_oracle as O
        self.O, self.cfg, self.B, self.S = O, cfg, B, S
        self.cores = threads or host_cores()
        torch.set_num_threads(self.cores)
        self.nl = 2
        self.W = O.LlamaWeights(cfg.dim, cfg.n_layers, cfg.n_heads, cfg.n_kv_heads, cfg.ffn_dim, cfg.vocab_size,
                                n_layers_alloc=self.nl)
        pages_per = S // page + 1
        nblk = B * pages_per
        self.kc = [torch.randn(nblk, page, cfg.n_kv_heads, cfg.head_dim).bfloat16() for _ in range(self.nl)]
        self.vc = [torch.randn(nblk, page, cfg.n_kv_heads, cfg.head_dim).bfloat16() for _ in range(self.nl)]
        self.table = torch.randperm(nblk).to(torch.int32).view(B, pages_per)
        self.lens = torch.full((B,), S, dtype=torch.int32)
        self.cos, self.sin = torch.randn(B, cfg.head_dim // 2), torch.randn(B, cfg.head_dim // 2)
        self.h = torch.randn(B, cfg.dim).bfloat16()
        self.i = 0

    def layer(self):
        """one TransformerBlock of the decode step (oracle.llama_block) -> seconds"""
        i = self.i % self.nl
        self.i += 1
        cfg = self.cfg
        t0 = time.perf_counter()
        self.O.llama_block(self.W.layers[i], self.h, self.kc[i], self.vc[i], self.lens, self.table, self.cos, self.sin,
                           cfg.n_heads, cfg.n_kv_heads, cfg.norm_eps)
        return time.perf_counter() - t0

    def head(self):
        t0 = time.perf_counter()
        self.O.linear(self.O.rms_norm(self.h, self.W.norm, self.cfg.norm_eps), self.W.output)
        return time.perf_counter() - t0

    def full_step_seconds(self, t_layer, t_head):
        return t_layer * self.cfg.n_layers + t_head


class RefCodeSample:
    """The same bounded sample executed by the UNMODIFIED reference installed under baseline/_ref: its
    `TransformerBlockLlama` (models/model_llama.py:160-185) with its `RefAttnBackend` (attn_backend.py:245-501) over a
    contiguous KV cache, torch `F.linear` in bf16 as its `op_impl="torch"` path does, on the host cores (the bootstrap of
    SURVEY 8c: device name forced to "cpu", a world-size-1 gloo group, Triton in interpreter mode — no Triton kernel is on
    this path).  The head is the reference's `F.linear` over the vocab-parallel output weight.  Raises if the reference
    cannot be imported or constructed; the caller then falls back to the oracle port."""

    kind = "reference"

    def __init__(self, cfg, B, S, threads=None):
        import socket
        import types

        os.environ.setdefault("TRITON_INTERPRET", "1")
        ref = os.path.join(ROOT, "baseline", "_ref")
        if not os.path.isdir(os.path.join(ref, "chitu")):
            raise RuntimeError("baseline/_ref is not installed")
        if ref not in sys.path:
            sys.path.insert(0, ref)
        import torch
        import torch.distributed as dist
        import chitu.device_type as D
        D._device_name = "cpu"
        from chitu import global_vars
        self._own_group = not dist.is_initialized()
        if self._own_group:
            with socket.socket() as sk:
                sk.bind(("127.0.0.1", 0))
                port = sk.getsockname()[1]
            dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
        if global_vars._GLOBAL_TIMERS is None:
            global_vars._set_timers()
        from chitu.attn_backend import RefAttnBackend
        from chitu.models.model_llama import TransformerBlockLlama
        self.cfg, self.B, self.S = cfg, B, S
        self.cores = threads or host_cores()
        torch.set_num_threads(self.cores)
        self.torch = torch
        sync, torch.cuda.synchronize = torch.cuda.synchronize, (lambda *a, **k: None)     # the reference's timers call it
        self._restore_sync = sync
        margs = types.SimpleNamespace(dim=cfg.dim, n_heads=cfg.n_heads, n_kv_heads=cfg.n_kv_heads, multiple_of=cfg.multiple_of,
                                      ffn_dim_multiplier=cfg.ffn_dim_multiplier, norm_eps=cfg.norm_eps)
        outer = self

        class Cache:                                 # what Attention.decode_forward reads from KVCacheManager
            def get_cache_decode(self, layer_id):
                return outer.k[layer_id], outer.v[layer_id]

            def get_gpu_seq_lens_excl_this_decode(self):
                return outer.lens

        self.nl = 2
        torch.set_default_dtype(torch.bfloat16)       # backend.py:119: the reference runs with bf16 as the default dtype
        try:
            self.blocks = [TransformerBlockLlama(i, margs, Cache(), RefAttnBackend(), "torch") for i in range(self.nl)]
            with torch.no_grad():
                for blk in self.blocks:
                    for n, p in blk.named_parameters():
                        p.copy_(torch.randn_like(p) * (0.02 if "norm" not in n else 1.0))
            ffn = self.blocks[0].feed_forward
            got = sum(p.numel() for p in ffn.parameters())
            assert got == 3 * cfg.dim * cfg.ffn_dim, (got, cfg.ffn_dim)           # the reference derived the same hidden dim
            self.k = [torch.randn(B, S + 1, cfg.n_kv_heads, cfg.head_dim) for _ in range(self.nl)]
            self.v = [torch.randn(B, S + 1, cfg.n_kv_heads, cfg.head_dim) for _ in range(self.nl)]
            self.head_w = torch.randn(cfg.vocab_size, cfg.dim) * 0.02
            self.x = torch.randn(B, 1, cfg.dim)
        finally:
            torch.set_default_dtype(torch.float32)
        self.lens = torch.full((B,), S, dtype=torch.long)
        ang = torch.rand(B, cfg.head_dim // 2, dtype=torch.float32) * 6.28
        self.cos, self.sin = torch.cos(ang), torch.sin(ang)
        self.i = 0

    def layer(self):
        torch = self.torch
        i = self.i % self.nl
        self.i += 1
        torch.set_default_dtype(torch.bfloat16)
        try:
            t0 = time.perf_counter()
            with torch.no_grad():
                self.blocks[i](self.x.clone(), self.cos, self.sin)
            return time.perf_counter() - t0
        finally:
            torch.set_default_dtype(torch.float32)

    def head(self):
        torch = self.torch
        t0 = time.perf_counter()
        with torch.no_grad():
            torch.nn.functional.linear(self.x.view(self.B, -1), self.head_w)
        return time.perf_counter() - t0

    def full_step_seconds(self, t_layer, t_head):
        return t_layer * self.cfg.n_layers + t_head

    def close(self):
        """undo the process-wide bootstrap (tests share their process with other tests; the arm itself just exits)"""
        import torch.distributed as dist
        self.torch.cuda.synchronize = self._restore_sync
        if self._own_group and dist.is_initialized():
            dist.destroy_process_group()


def reference_sample(cfg, B, S):
    """(sample object, note): the unmodified reference from baseline/_ref when it can run here, else the oracle port."""
    try:
        smp = RefCodeSample(cfg, B, S)
        smp.layer()                                   # proves the block runs before it is timed
        return smp, "reference code from baseline/_ref (TransformerBlockLlama + RefAttnBackend, torch bf16 on the host)"
    except Exception as e:
        smp = CpuSample(cfg, B, S)
        smp.kind = "port"
        return smp, f"oracle port (reference code not runnable here: {type(e).__name__}: {str(e)[:120]})"


def cpu_baseline(B, S, layers=2, threads=None):
    """`cpu_baseline` of our arm's line: `layers` timed layers (after one untimed) + the head, bounded to ~10-30 s."""
    from chitu_b200.engine import LLAMA3_8B as cfg
    smp = CpuSample(cfg, B, S, threads=threads)
    smp.layer()                                                     # page-in
    ts = [smp.layer() for _ in range(layers)]
    t_layer = sum(ts) / len(ts)
    t_head = smp.head()
    step_s = smp.full_step_seconds(t_layer, t_head)
    return {"value": B / step_s, "unit": UNIT, "cores": smp.cores, "kind": "port",
            "sample": f"{layers} timed layers (of {cfg.n_layers}) + the head of the bs={B}, seq={S} LLaMA-3-8B decode step on "
                      f"{smp.cores} host threads ({sum(ts) + t_head:.1f} s of CPU work): {t_layer:.2f} s/layer x {cfg.n_layers} "
                      f"+ {t_head:.2f} s head = {step_s:.1f} s per full step"}


def cpu_baseline_with_reference(B, S):
    """`cpu_baseline` of our arm's line.  Preferred: the UNMODIFIED reference (baseline/_ref) on the host cores, run as
    the reference arm in its own process (`--impl reference --short`: it forces the reference's device name to
    "cpu" and must not share a process with the CUDA run); the in-process oracle port is reported next to it
    (`oracle_port`) and is the fallback when the reference cannot run on this box."""
    import subprocess
    port = cpu_baseline(B, S, layers=2)
    try:
        env = {k: v for k, v in os.environ.items() if k not in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT")}
        env["CUDA_VISIBLE_DEVICES"] = ""
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--short", "--steps", "1", "--warmup", "1",
                              "--bs", str(B), "--seq", str(S)], capture_output=True, text=True, timeout=300, env=env)
        ref = json.loads(out.stdout.strip().splitlines()[-1])["cpu_baseline"]
        if ref.get("kind") == "reference":
            ref["oracle_port"] = port
            return ref
        port["reference_note"] = ref.get("implementation", "")
    except Exception as e:
        port["reference_note"] = f"reference arm subprocess failed: {type(e).__name__}: {str(e)[:120]}"
    return port


def run_reference(args):
    """--impl reference: the reference's own implementation of the path on the host cores, all host threads: the UNMODIFIED
    reference installed under baseline/_ref (its TransformerBlockLlama + RefAttnBackend; `cpu_baseline.kind` =
    "reference"), or — when that cannot run on this box — the oracle port of its model code ("port").  The reference has no
    production CPU path (BASELINE.md §3): RefAttnBackend is its test backend and spends ~90 % of a decode layer copying /
    casting the KV cache, so the oracle port of the same arithmetic is reported beside it (`oracle_port`).  Honours --steps / --warmup: every timed step is the SAME
    bounded sample — ONE transformer layer of the bs=16 seq=4096 LLaMA-3-8B decode step (1/32 of the layer work; the
    head is timed once, outside the K steps).  `ms_per_step` is the measured time of one sample step; `value` is the
    full-depth tokens/s = bs / (32 x layer + head).  Also runs BASELINE.json configs[0] (LLaMA-2-7B bs=1 seq=128, the
    reference's CPU-runnable plumbing case, BASELINE.md §3) the same way."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    os.environ["CUDA_VISIBLE_DEVICES"] = ""          # a host-only arm: nothing here may initialise CUDA
    from chitu_b200.engine import LLAMA2_7B, LLAMA3_8B
    smp, how = reference_sample(LLAMA3_8B, args.bs, args.seq)
    port = None
    if smp.kind == "reference" and not args.short:    # the oracle port of the same arithmetic, for comparison
        try:
            port = cpu_baseline(args.bs, args.seq, layers=2)
        except Exception as e:
            port = {"error": f"{type(e).__name__}: {str(e)[:120]}"}
    t_budget = 200.0                                               # the whole run must end within a few minutes
    t0 = time.perf_counter()
    t_head = smp.head()
    for _ in range(args.warmup):
        smp.layer()
    times = []
    for _ in range(args.steps):
        times.append(smp.layer())
        if time.perf_counter() - t0 > t_budget:
            break
    t_layer = sum(times) / len(times)
    step_s = smp.full_step_seconds(t_layer, t_head)
    v = args.bs / step_s
    cb = {"value": v, "unit": UNIT, "cores": smp.cores, "kind": smp.kind, "implementation": how,
          "sample": f"one transformer layer (of {LLAMA3_8B.n_layers}) of the bs={args.bs}, seq={args.seq} LLaMA-3-8B decode step per "
                    f"timed step, {len(times)} timed steps of {t_layer:.2f} s on {smp.cores} host threads, head timed once "
                    f"({t_head:.2f} s); full-depth step = 32 x layer + head = {step_s:.1f} s"}
    if port is not None:
        cb["oracle_port"] = port
    cores = smp.cores
    del smp
    # configs[0]: LLaMA-2-7B bf16 bs=1 seq=128 decode on CPU (plumbing)
    c0, how0 = None, ""
    if not args.short:
        s0, how0 = reference_sample(LLAMA2_7B, 1, 128)
        s0.layer()
        l0 = sum(s0.layer() for _ in range(4)) / 4
        c0 = s0.full_step_seconds(l0, s0.head())
    line = {"impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus,
            "steps": len(times), "warmup": args.warmup, "ms_per_step": t_layer * 1e3,
            "ms_per_full_depth_step": step_s * 1e3, "sample_fraction_of_step": t_layer / step_s,
            "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
            "config": {"workload": f"LLaMA-3-8B bf16 paged-KV decode, bs={args.bs}, seq={args.seq}, page=256 "
                                   f"({how}; bounded sample per step: one layer)",
                       "global_batch": args.bs, "seq_len": args.seq, "parallelism": "cpu"},
            "cpu_baseline": cb,
            "config0_llama2_7b_bs1_seq128_cpu": None if c0 is None else {
                "tokens_per_s": 1.0 / c0, "ms_per_step": c0 * 1e3, "cores": cores, "implementation": how0,
                "sample": "4 timed layers of 32 + head; full step = 32 x layer + head"},
            "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--bs", type=int, default=16)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--linear-impl", type=int, default=0, help="0 auto, 1 SIMT, 2 wgmma")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-deepseek", action="store_true", help="skip the DeepSeek-R1 block of the default line")
    ap.add_argument("--no-mgpu-check", action="store_true", help="skip the multi-GPU parity preamble (N > 1)")
    ap.add_argument("--nccl-allreduce", action="store_true", help="use NCCL all-reduce instead of the fused one-shot kernel")
    ap.add_argument("--workload", default="llama3-8b", choices=["llama3-8b", "deepseek-r1", "w8a8-sweep", "mixtral", "ref-kernels"])
    ap.add_argument("--tp", type=int, default=0, help="deepseek-r1: tensor-parallel degree that shapes the shard")
    ap.add_argument("--layers", type=int, default=0, help="deepseek-r1 / sweep: layer count override")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the logits / next tokens of the last timed step of every engine to DIR/<name>.npy")
    ap.add_argument("--short", action="store_true", help="--impl reference: the bounded cpu_baseline sample only (1 warm-up, "
                    "no configs[0] run, no oracle-port leg); used by our own arm's cpu_baseline subprocess")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 1 if (args.impl == "reference" and args.short) else 3)
    if args.impl == "reference":
        run_reference(args)
    elif args.workload == "deepseek-r1":
        run_deepseek(args)
    elif args.workload == "w8a8-sweep":
        run_sweep(args)
    elif args.workload == "mixtral":
        from chitu_b200.engine_mixtral import run_bench
        run_bench(args, time_engine, ClockSampler, peaks)
    elif args.workload == "ref-kernels":
        # the unmodified reference (baseline/_ref: its Triton kernels / flash_attn calls) timed beside ours on this GPU
        from scripts.ref_gpu_compare import main as ref_compare
        print(json.dumps(ref_compare(args.bs)), flush=True)
    else:
        run_cuda(args)


if __name__ == "__main__":
    main()
