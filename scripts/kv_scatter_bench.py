"""The prompt's KV write on one GPU: ops.scatter_kv_to_cache (chitu_b200_scatter_kv, one launch for the batch) against,
in the same process,
  loop        the reference's shape of finalize_cache_bylayer_prefill (cache_manager.py:93-142): a host loop over the
              requests that slices each request's rows, clamps and casts them for an e4m3 cache, and index-assigns them
              to their pages (or to a slice of the non-paged cache); the lengths are host integers, as there
  index_put   one vectorised torch index_put_ of all rows (cast first for e4m3), with the destination row of every
              source row computed once outside the timed calls (so its time is a lower bound for that approach)
Shapes, each with a bf16 cache and an e4m3 cache where that cache exists:
  LLaMA-3-8B layer (Hkv 8, D 128, 256-token pages): 16 x 2048-token prompts, 1 x 32768, 64 ragged prompts of 1-8192
  tokens (seeded);
  DeepSeek latent (576, 64-token pages): 16 x 4096;
  non-paged [16, 4096, 8, 128] cache: 16 x 4096 (bf16 only: the e4m3 cache is built for paged caches only).
Repeating a call is idempotent (the same rows land in the same slots), so the caches are not restored between calls.

For every case and path: the median, min and max ms over 5 CUDA-event windows of 20 calls each after 3 warm-up calls;
the bytes the write needs (source rows read plus cache rows written, both caches for GQA), GB/s at the median and that
rate as a share of the H100 SXM data sheet's 3.35 TB/s HBM3 bandwidth; and whether the three paths left the same bytes.

  python scripts/kv_scatter_bench.py --out DIR          writes DIR/kv_scatter_bench.json and prints a markdown table

Reads the device name, power limit and max SM clock (nvidia-smi --query-gpu, a query only); changes no device setting.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from chitu_b200 import ops  # noqa: E402
from paged_prefill_bench import gpu_info, spread, time_ms  # noqa: E402

DATASHEET_TB_S = 3.35
E4M3 = torch.float8_e4m3fn


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16}[t.element_size()])


def _stored(rows, cache_dtype):
    return rows.float().clamp(-448.0, 448.0).to(E4M3) if cache_dtype == E4M3 else rows


def ragged_lens(B, lo, hi, seed):
    return torch.randint(lo, hi + 1, (B,), generator=torch.Generator().manual_seed(seed)).tolist()


# (name, row shape, page (0: non-paged), prompt lengths, cache dtypes)
LLAMA, MLA = (8, 128), (576,)
CASES = [("llama3-8b 16 x 2048", LLAMA, 256, [2048] * 16, (torch.bfloat16, E4M3)),
         ("llama3-8b 1 x 32768", LLAMA, 256, [32768], (torch.bfloat16, E4M3)),
         ("llama3-8b 64 ragged 1-8192", LLAMA, 256, ragged_lens(64, 1, 8192, 1), (torch.bfloat16, E4M3)),
         ("deepseek latent 16 x 4096", MLA, 64, [4096] * 16, (torch.bfloat16, E4M3)),
         ("non-paged [16, 4096, 8, 128]", LLAMA, 0, [4096] * 16, (torch.bfloat16,))]


def make_case(row, page, lens, cache_dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, total, two = len(lens), sum(lens), len(row) == 2
    srcs = [torch.randn(total, *row, generator=g, device="cuda").mul_(4.0).bfloat16() for _ in range(1 + two)]
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    if page:
        per = [-(-n // page) for n in lens]
        nb = sum(per) + 1
        perm = torch.randperm(nb, generator=torch.Generator().manual_seed(seed))
        bt = torch.zeros(B, max(per), dtype=torch.int32)
        used = torch.arange(max(per))[None, :] < torch.tensor(per)[:, None]
        bt[used] = perm[:sum(per)].int()
        bt = bt.cuda()
        caches = [torch.zeros(nb, page, *row, device="cuda", dtype=torch.bfloat16).to(cache_dtype) for _ in srcs]
        pos = torch.cat([torch.arange(n) for n in lens])
        req = torch.repeat_interleave(torch.arange(B), torch.tensor(lens))
        dest = (bt.cpu().long()[req, pos // page] * page + pos % page).cuda()
    else:
        bt = None
        caches = [torch.zeros(B, max(lens), *row, device="cuda", dtype=torch.bfloat16) for _ in srcs]
        dest = torch.cat([b * max(lens) + torch.arange(n) for b, n in enumerate(lens)]).cuda()
    return srcs, caches, cu, bt, dest


def run_case(name, row, page, lens, cache_dtype, seed):
    srcs, caches, cu, bt, dest = make_case(row, page, lens, cache_dtype, seed)
    k, v = srcs[0], srcs[1] if len(srcs) > 1 else None
    kc, vc = caches[0], caches[1] if len(caches) > 1 else None
    cu_host = cu.tolist()
    bt_host_rows = None if bt is None else [bt[b] for b in range(len(lens))]

    def ours():
        ops.scatter_kv_to_cache(kc, vc, k, v, cu, bt)

    def loop():
        for cache, src in zip(caches, srcs):
            for b in range(len(lens)):
                rows = _stored(src[cu_host[b]:cu_host[b + 1]], cache_dtype)
                if bt is None:
                    cache[b, :lens[b]] = rows
                else:
                    p = torch.arange(lens[b], device="cuda")
                    _bits(cache)[bt_host_rows[b][p // page], p % page] = _bits(rows)

    def index_put():
        for cache, src in zip(caches, srcs):
            _bits(cache).view(-1, *row).index_put_((dest,), _bits(_stored(src, cache_dtype)))

    paths = {"scatter": ours, "loop": loop, "index_put": index_put}
    results = {}
    for pname, fn in paths.items():
        for c in caches:
            _bits(c).fill_(0)
        fn()
        torch.cuda.synchronize()
        results[pname] = [_bits(c).clone() for c in caches]
    same = all(torch.equal(a, b) for p in ("loop", "index_put") for a, b in zip(results["scatter"], results[p]))
    del results
    n_el = 1
    for d in row:
        n_el *= d
    nbytes = sum(lens) * n_el * (2 + torch.empty((), dtype=cache_dtype).element_size()) * len(srcs)
    out = {"case": name, "cache": str(cache_dtype).replace("torch.", ""), "rows": sum(lens), "bytes": nbytes,
           "identical": same}
    for pname, fn in paths.items():
        s = spread(time_ms(fn, 3, 20, 5))
        gbs = nbytes / (s["median"] * 1e-3) / 1e9
        out[pname] = dict(s, gb_s=gbs, datasheet_share=gbs / (DATASHEET_TB_S * 1e3))
    del srcs, caches
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_scatter_bench needs a CUDA device")
    info = gpu_info()
    rows = []
    for i, (name, row, page, lens, dtypes) in enumerate(CASES):
        for dt in dtypes:
            r = run_case(name, row, page, lens, dt, seed=10 + i)
            rows.append(r)
            print(json.dumps(r), flush=True)
    print(f"\n{info['device']}; nvidia-smi: {info['nvidia_smi']!r}\n")
    print("| case | cache | rows | MB | scatter ms | GB/s | share of 3.35 TB/s | loop ms | loop / scatter "
          "| index_put ms | index_put / scatter | same bytes |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        s, lp, ip = r["scatter"], r["loop"], r["index_put"]
        print(f"| {r['case']} | {r['cache']} | {r['rows']} | {r['bytes'] / 1e6:.0f} "
              f"| {s['median']:.3f} ({s['min']:.3f}–{s['max']:.3f}) | {s['gb_s']:.0f} | {100 * s['datasheet_share']:.0f} % "
              f"| {lp['median']:.3f} ({lp['min']:.3f}–{lp['max']:.3f}) | {lp['median'] / s['median']:.1f}x "
              f"| {ip['median']:.3f} ({ip['min']:.3f}–{ip['max']:.3f}) | {ip['median'] / s['median']:.1f}x "
              f"| {r['identical']} |")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "kv_scatter_bench.json"), "w") as f:
            json.dump({"gpu": info, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
