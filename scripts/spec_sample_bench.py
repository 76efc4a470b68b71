"""Cost of sampled verification of speculative drafts (chitu_b200_spec_accept_sampled) on one GPU.

1. The entry alone: bs 1 / 4 / 16, k = 1 / 3 / 7, V = 128256 bf16 logits, token-only and draft-model drafts.  Reported
   per case: us per call (median, min, max over `--windows` CUDA-event windows), beside the same rule in torch as the
   reference writes it (per row: sort, cumsum, mask, renormalise; then the acceptance and the residual draw in torch
   ops), timed alternately in the same run; and the bytes a call must read (the logits once, q once in draft-model
   mode) over the 3.35 TB/s HBM3 bound of the H100 SXM data sheet.
2. The engine: LLaMA-3-8B (32 layers) at context 4096, bf16 weights and cache, bs 1 / 4 / 16, k = 1 / 3 / 7.  One
   engine per case is built with sampled_verify=True; its sampled verify graph and a greedy verify graph of the same
   engine (argmax + greedy acceptance) are replayed alternately, with seq_lens reset before each replay.

  python scripts/spec_sample_bench.py --out DIR          writes DIR/spec_sample_bench.json

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

from paged_prefill_bench import gpu_info  # noqa: E402
from w4a16_bench import alternate  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
DEV = "cuda:0"


def torch_rule(logits, T, top_k, top_p, drafts, n, q, ua, ud):
    """The sampled acceptance as torch ops over all rows (the reference's sort / cumsum / mask sampler per row)."""
    B, k = drafts.shape
    R, V = logits.shape
    rep = lambda t: t.repeat_interleave(k + 1)[:, None]            # noqa: E731
    probs = torch.softmax(logits.float() / rep(T), dim=-1)
    ps, idx = probs.sort(dim=-1, descending=True)
    cs = ps.cumsum(-1)
    rank = torch.arange(V, device=logits.device)[None]
    tk = torch.where(rep(top_k) > 0, rep(top_k), V)
    ps = ps.masked_fill(((cs - ps) > rep(top_p)) | (rank >= tk), 0.0)
    ps = ps / ps.sum(-1, keepdim=True)
    p = torch.zeros_like(probs).scatter_(-1, idx, ps).view(B, k + 1, V)
    pd = p[:, :k].gather(-1, drafts[..., None]).squeeze(-1)
    qd = torch.ones_like(pd) if q is None else q.gather(-1, drafts[..., None]).squeeze(-1)
    ok = (ua * qd < pd) & (torch.arange(k, device=logits.device)[None] < n[:, None])
    a = ok.int().cumprod(-1).sum(-1)
    rows = torch.arange(B, device=logits.device)
    pa = p[rows, a]
    ac = a.clamp(max=k - 1)
    qa = torch.nn.functional.one_hot(drafts[rows, ac], V).float() if q is None else q[rows, ac]
    r = (pa - qa).clamp(min=0)
    r = torch.where(((a < n) & (r.sum(-1) > 0))[:, None], r, pa)
    cdf = r.cumsum(-1)
    tok = torch.searchsorted(cdf, (ud * cdf[:, -1])[:, None], right=True).clamp(max=V - 1).squeeze(-1)
    return a, tok


def entry_case(B, k, dense, args):
    from chitu_b200 import _lib
    from chitu_b200._lib import current_stream, ptr
    lib = _lib.load()
    V = 128256
    g = torch.Generator(device=DEV).manual_seed(B * 100 + k)
    logits = (torch.randn(B * (k + 1), V, generator=g, device=DEV) * 3).to(torch.bfloat16)
    T = torch.full((B,), 0.8, device=DEV)
    top_k = torch.full((B,), 50, dtype=torch.int32, device=DEV)
    top_p = torch.full((B,), 0.9, device=DEV)
    drafts = logits.float().argmax(-1).view(B, k + 1)[:, :k].contiguous()
    n = torch.full((B,), k, dtype=torch.int32, device=DEV)
    q = torch.softmax(torch.randn(B, k, V, generator=g, device=DEV), dim=-1) if dense else None
    ua = torch.rand(B, k, generator=g, device=DEV)
    ud = torch.rand(B, generator=g, device=DEV)
    seq = torch.zeros(B, dtype=torch.int32, device=DEV)
    out = torch.empty(B, k + 1, dtype=torch.int64, device=DEV)
    acc = torch.empty(B, dtype=torch.int32, device=DEV)
    nxt = torch.empty(B, dtype=torch.int64, device=DEV)
    ws = torch.empty(lib.chitu_b200_spec_accept_sampled_workspace_bytes(B, k), dtype=torch.uint8, device=DEV)

    def ours():
        lib.chitu_b200_spec_accept_sampled(ptr(logits), V, V, _lib.CB_BF16, ptr(T), ptr(top_k), ptr(top_p), ptr(drafts),
                                           ptr(n), ptr(q), 0 if q is None else V, ptr(ua), ptr(ud), ptr(seq), ptr(out),
                                           ptr(acc), ptr(nxt), B, k, ptr(ws), ws.numel(), current_stream())

    def ref():
        torch_rule(logits, T, top_k, top_p, drafts, n, q, ua, ud)

    t_ours, t_ref = alternate([ours, ref], 3, args.steps, args.windows)
    nbytes = logits.numel() * 2 + (q.numel() * 4 if dense else 0)
    us = t_ours["median"] * 1e3
    return {"bs": B, "k": k, "mode": "draft-model" if dense else "token-only", "V": V, "entry_us": t_ours,
            "torch_ms": t_ref, "speedup": t_ref["median"] / t_ours["median"], "bytes": nbytes,
            "hbm_bound_us": nbytes / HBM_BYTES_PER_S * 1e6, "share_of_hbm_bound": nbytes / HBM_BYTES_PER_S * 1e6 / us}


def engine_case(cfg, B, k, args):
    from chitu_b200.engine import LlamaDecodeEngine
    S = args.seq
    e = LlamaDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, device=DEV, page_size=256, max_draft=k,
                          sampled_verify=True)
    e.set_synthetic_context(S)
    e.n_draft.fill_(k)
    e.temperatures.fill_(0.8)
    e.top_ks.fill_(50)
    e.top_ps.fill_(0.9)
    e.capture_verify()
    sampled = e.verify_graph
    e.sampled_verify = False                 # the same engine's greedy tail: argmax + greedy acceptance
    greedy, _ = e._capture(e._verify_body)
    e.sampled_verify = True
    s0 = e.seq_lens.clone()

    def replay(graph):
        def fn():
            e.seq_lens.copy_(s0)
            graph.replay()
        return fn

    t_s, t_g = alternate([replay(sampled), replay(greedy)], 3, args.engine_steps, args.windows)
    out = {"bs": B, "k": k, "seq": S, "layers": cfg.n_layers, "sampled_ms": t_s, "greedy_ms": t_g,
           "tail_added_ms": t_s["median"] - t_g["median"], "ratio": t_s["median"] / t_g["median"]}
    del e, sampled, greedy
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=50, help="entry calls per timing window")
    ap.add_argument("--engine-steps", type=int, default=20, help="graph replays per timing window")
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--bs", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--k", type=int, nargs="+", default=[1, 3, 7])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_sample_bench.py measures on a GPU; none is visible")
    from chitu_b200.engine import LLAMA3_8B
    cfg = dataclasses.replace(LLAMA3_8B, n_layers=args.layers)
    res = {"gpu": gpu_info(), "entry": [], "engine": []}
    print(json.dumps(res["gpu"]), flush=True)
    for dense in (False, True):
        for B in args.bs:
            for k in args.k:
                c = entry_case(B, k, dense, args)
                res["entry"].append(c)
                print(f"entry {c['mode']:11s} bs={B:2d} k={k}  {c['entry_us']['median'] * 1e3:8.1f} us  torch "
                      f"{c['torch_ms']['median'] * 1e3:8.1f} us  x{c['speedup']:.1f}  {c['bytes'] / 1e6:.1f} MB  "
                      f"HBM bound {c['hbm_bound_us']:.1f} us ({c['share_of_hbm_bound']:.2f})", flush=True)
    for B in args.bs:
        for k in args.k:
            c = engine_case(cfg, B, k, args)
            res["engine"].append(c)
            print(f"engine bs={B:2d} k={k}  sampled {c['sampled_ms']['median']:7.3f} ms  greedy "
                  f"{c['greedy_ms']['median']:7.3f} ms  +{c['tail_added_ms'] * 1e3:.1f} us  ratio {c['ratio']:.4f}",
                  flush=True)
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "spec_sample_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
