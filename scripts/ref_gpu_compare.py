"""GPU comparator (SURVEY §8d "bar to beat", VERDICT r1 item 9): the UNMODIFIED reference installed under baseline/_ref
(`python -m pip install --no-index --no-build-isolation --no-deps --target baseline/_ref <copy of the reference>`) — its Triton fp8 GEMM, Triton MLA decode, Triton fused experts, and flash_attn paged decode, all through the
reference's own functions / backend classes — timed on the SAME GPU beside this repository's kernels, on the same inputs,
at the DeepSeek-R1 tp=8 / LLaMA-3-8B decode shapes.  Both sides run inside CUDA graphs over rotating operand sets larger
than L2 (the reference captures its decode step the same way, models/model.py:537-622), CUDA-event timed.

    python scripts/ref_gpu_compare.py [bs]          -> one JSON line (also called by bench.py --workload ref-kernels)

Nothing here is on the product path; the reference is only ever imported from baseline/_ref (never from a source checkout)."""
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "baseline", "_ref")


def _import_reference():
    if not os.path.isdir(os.path.join(REF, "chitu")):
        return None, "baseline/_ref is not installed"
    sys.path.insert(0, REF)
    try:
        import chitu.attn_backend as rab
        import chitu.fused_moe as rfm
        import chitu.ops as rops
        return types.SimpleNamespace(ops=rops, fused_moe=rfm, attn_backend=rab), None
    except Exception as e:  # missing optional dependency of the reference on this box
        return None, f"{type(e).__name__}: {e}"


def timed(fn, nsets, reps=5):
    """us per call of fn(i), i cycling over `nsets` operand sets, inside one CUDA graph (eager loop if capture fails)."""
    import torch
    st = torch.cuda.Stream()
    mode = "graph"
    with torch.cuda.stream(st):
        for i in range(nsets):            # warm-up (Triton autotune / JIT happens here)
            fn(i)
        st.synchronize()
        g = None
        try:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                for i in range(nsets):
                    fn(i)
        except Exception:
            g, mode = None, "eager"
            torch.cuda.synchronize()

        def run():
            if g is not None:
                g.replay()
            else:
                for i in range(nsets):
                    fn(i)
        for _ in range(2):
            run()
        st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(reps):
            run()
        e1.record(st)
        st.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * nsets), mode


def make_fp8_weight(N, K, dev):
    import torch
    w = torch.randn(N, K, device=dev) * 0.02
    wb = w.view(N // 128, 128, K // 128, 128)
    s = wb.abs().amax(dim=(1, 3)).clamp_min(1e-8) / 448.0
    q = (wb / s[:, None, :, None]).clamp(-448, 448).view(N, K).to(torch.float8_e4m3fn)
    return q, s.float().contiguous()


def main(B=16, only="", side="both"):
    """only: substring filter on the op name; side: both | ref | ours (isolates a faulting side in its own process)"""
    import torch
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    ref, why = _import_reference()
    if ref is None:
        return {"label": "ref_gpu_kernels", "unavailable": why}
    from chitu_b200 import fused_moe as ofm
    from chitu_b200 import ops as oops
    from chitu_b200.attn_backend import B200AttnBackend
    rows = []

    def add(name, ref_fn, our_fn, nsets, nbytes, check=None):
        if only and only not in name:
            return
        r = {"op": name, "bytes": nbytes}
        if side in ("both", "ref"):
            try:
                r["ref_us"], r["ref_mode"] = timed(ref_fn, nsets)
                torch.cuda.synchronize()
            except Exception as e:
                r["ref_error"] = f"{type(e).__name__}: {str(e)[:200]}"
        if side in ("both", "ours"):
            r["our_us"], _ = timed(our_fn, nsets)
            torch.cuda.synchronize()
        if check is not None and "ref_us" in r and "our_us" in r:
            try:
                r["max_rel_vs_ref"] = check()
            except Exception as e:
                r["check_error"] = f"{type(e).__name__}: {str(e)[:120]}"
        if "ref_us" in r and "our_us" in r:
            r["speedup"] = r["ref_us"] / r["our_us"]
        if "our_us" in r:
            r["our_gbs"] = nbytes / r["our_us"] / 1e3
        rows.append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)

    def max_rel(a, b):
        a, b = a.float(), b.float()
        return ((a - b).abs().max() / b.abs().max().clamp_min(1e-9)).item()

    # ---- FP8 block-scaled linears of one DeepSeek-R1 layer (per-rank shapes, SURVEY 8a a8) ----
    for name, N, K in (("wqkv_a", 2112, 7168), ("wq_b", 3072, 1536), ("wo", 7168, 2048), ("dense_w13", 4608, 7168),
                       ("dense_w2", 7168, 2304)):
        nsets = max(2, int(300e6 // (N * K)) + 1)
        ws = []
        for _ in range(nsets):
            Np = (N + 127) // 128 * 128
            q, s = make_fp8_weight(Np, K, dev)
            ws.append((q[:N].contiguous(), s))
        x = torch.randn(B, K, device=dev, dtype=torch.bfloat16)
        xq, xs = oops.act_quant_deepseek_v3(x, 128)
        add(f"fp8_gemm {name} M={B} N={N} K={K}",
            lambda i: ref.ops.fp8_gemm_deepseek_v3(xq, xs, ws[i][0], ws[i][1]),
            lambda i: oops.fp8_gemm_deepseek_v3(xq, xs, ws[i][0], ws[i][1]), nsets, N * K + B * K + B * N * 2,
            check=lambda: max_rel(oops.fp8_gemm_deepseek_v3(xq, xs, ws[0][0], ws[0][1]),
                                  ref.ops.fp8_gemm_deepseek_v3(xq, xs, ws[0][0], ws[0][1])))
        del ws

    # ---- absorbed-MLA paged decode, H = 16 local heads, S = 4096, page 64 (a2 / a4) ----
    H, C, R, page, ctx = 16, 512, 64, 64, 4096
    per = (ctx + page) // page
    nsets = 4
    caches = [torch.randn(B * per, page, C + R, device=dev, dtype=torch.bfloat16) for _ in range(nsets)]
    bt = torch.randperm(B * per, device=dev, dtype=torch.int32).view(B, per).contiguous()
    excl = torch.full((B,), ctx - 1, device=dev, dtype=torch.int32)
    incl = excl + 1
    q_nope = torch.randn(B, H, C, device=dev, dtype=torch.bfloat16)
    q_pe = torch.randn(B, H, R, device=dev, dtype=torch.bfloat16)
    kv = torch.randn(B, 1, 1, C + R, device=dev, dtype=torch.bfloat16)
    scale = 0.1352
    rbe = object.__new__(ref.attn_backend.TritonAttnBackend)        # the reference class without its global-args __init__
    rbe.local_n_heads, rbe.kv_lora_rank, rbe.qk_rope_head_dim, rbe.qk_nope_head_dim = H, C, R, 128
    obe = B200AttnBackend(max_seq_len=ctx, max_reqs=B, n_local_heads=H)
    obe.prepare_metadata_for_decode(excl, incl, bt, page)
    add(f"mla_decode B={B} H=16 ctx=4096 (append + attention)",
        lambda i: rbe.mla_attn_with_kvcache(q_nope, q_pe, caches[i], kv, excl, incl, bt, softmax_scale=scale),
        lambda i: obe.mla_attn_with_kvcache(q_nope, q_pe, caches[i], kv, excl, incl, bt, softmax_scale=scale), nsets,
        B * ctx * (C + R) * 2,
        check=lambda: max_rel(obe.mla_attn_with_kvcache(q_nope, q_pe, caches[0], kv, excl, incl, bt, softmax_scale=scale),
                              rbe.mla_attn_with_kvcache(q_nope, q_pe, caches[0], kv, excl, incl, bt, softmax_scale=scale)))
    del caches

    # ---- fused experts, fp8 block-scaled, the tp=8 shard: the 256 routed experts, top-8, w13 [512,7168], w2 [7168,256] (a16);
    # the reference computes the shared expert separately (model_deepseek_v3.py:936-949), so it is left out on both sides ----
    E, N1, K1 = 256, 512, 7168
    nsets = 3
    sets = []
    for _ in range(nsets):
        # random e4m3 bit patterns; -1 = 0xFF is NaN in e4m3fn, map it to zero
        w1 = torch.randint(-60, 60, (E, N1, K1), device=dev, dtype=torch.int8)
        w2 = torch.randint(-60, 60, (E, K1, N1 // 2), device=dev, dtype=torch.int8)
        w1[w1 == -1] = 0
        w2[w2 == -1] = 0
        w1, w2 = w1.view(torch.float8_e4m3fn), w2.view(torch.float8_e4m3fn)
        sets.append((w1, w2, torch.rand(E, N1 // 128, K1 // 128, device=dev) * 0.01 + 0.001,
                     torch.rand(E, K1 // 128, N1 // 2 // 128, device=dev) * 0.01 + 0.001))
    x = torch.randn(B, K1, device=dev, dtype=torch.bfloat16)
    ids = torch.stack([torch.randperm(256, device=dev)[:8] for _ in range(B)])
    tw = torch.rand(B, 8, device=dev, dtype=torch.float32)
    nd = ids.unique().numel()
    # the reference's model calls fused_experts(..., inplace=True) (model_deepseek_v3.py:995-1009); its inplace=False branch
    # goes through torch.ops.vllm.outplace_fused_experts, which the reference never registers
    kw = dict(inplace=True, use_fp8_w8a8=True, block_shape=[128, 128])
    xr = [x.clone() for _ in range(nsets)]
    xo = [x.clone() for _ in range(nsets)]
    add(f"fused_experts fp8 T={B} topk=8 E=256 ({nd} distinct), inplace",
        lambda i: ref.fused_moe.fused_experts(xr[i], sets[i][0], sets[i][1], tw, ids, w1_scale=sets[i][2], w2_scale=sets[i][3], **kw),
        lambda i: ofm.fused_experts(xo[i], sets[i][0], sets[i][1], tw, ids, w1_scale=sets[i][2], w2_scale=sets[i][3], **kw), nsets,
        nd * (N1 * K1 + K1 * N1 // 2),
        check=lambda: max_rel(ofm.fused_experts(x.clone(), sets[0][0], sets[0][1], tw, ids, w1_scale=sets[0][2], w2_scale=sets[0][3], **kw),
                              ref.fused_moe.fused_experts(x.clone(), sets[0][0], sets[0][1], tw, ids, w1_scale=sets[0][2],
                                                          w2_scale=sets[0][3], **kw)))
    del sets

    # ---- LLaMA-3-8B GQA paged decode (a5): the reference's FlashAttnBackend = flash_attn_with_kvcache ----
    Hq, Hkv, D, page, ctx = 32, 8, 128, 256, 4096
    per = ctx // page + 1
    nsets = 3
    kcs = [torch.randn(B * per, page, Hkv, D, device=dev, dtype=torch.bfloat16) for _ in range(nsets)]
    vcs = [torch.randn(B * per, page, Hkv, D, device=dev, dtype=torch.bfloat16) for _ in range(nsets)]
    bt = torch.randperm(B * per, device=dev, dtype=torch.int32).view(B, per).contiguous()
    lens = torch.full((B,), ctx - 1, device=dev, dtype=torch.int32)
    q = torch.randn(B, 1, Hq, D, device=dev, dtype=torch.bfloat16)
    kn = torch.randn(B, 1, Hkv, D, device=dev, dtype=torch.bfloat16)
    vn = torch.randn(B, 1, Hkv, D, device=dev, dtype=torch.bfloat16)
    rfa = object.__new__(ref.attn_backend.FlashAttnBackend)
    oga = B200AttnBackend(max_seq_len=ctx + page, max_reqs=B, n_local_heads=Hq)
    add(f"gqa_paged_decode B={B} 32q/8kv D=128 ctx=4096 (flash_attn_with_kvcache)",
        lambda i: rfa.attn_with_kvcache(q, kcs[i], vcs[i], k=kn, v=vn, cache_seqlens=lens, block_table=bt, causal=True),
        lambda i: oga.attn_with_kvcache(q, kcs[i], vcs[i], k=kn, v=vn, cache_seqlens=lens, block_table=bt, causal=True), nsets,
        B * ctx * Hkv * D * 2 * 2,
        check=lambda: max_rel(oga.attn_with_kvcache(q, kcs[0], vcs[0], k=kn, v=vn, cache_seqlens=lens, block_table=bt, causal=True),
                              rfa.attn_with_kvcache(q, kcs[0], vcs[0], k=kn, v=vn, cache_seqlens=lens, block_table=bt, causal=True)))

    # ---- LLaMA-3-8B bf16 linears: F.linear (cuBLAS) is the reference's linear_op ----
    for name, N, K in (("w13", 28672, 4096), ("w2", 4096, 14336), ("wqkv", 6144, 4096), ("wo", 4096, 4096)):
        nsets = max(2, int(400e6 // (N * K * 2)) + 1)
        ws = [torch.randn(N, K, device=dev, dtype=torch.bfloat16) * 0.02 for _ in range(nsets)]
        x = torch.randn(B, K, device=dev, dtype=torch.bfloat16)
        add(f"linear bf16 {name} M={B} N={N} K={K} (F.linear)",
            lambda i: torch.nn.functional.linear(x, ws[i]), lambda i: oops.linear(x, ws[i]), nsets, N * K * 2 + B * K * 2 + B * N * 2)
        del ws
    return {"label": "ref_gpu_kernels", "bs": B, "device": torch.cuda.get_device_name(0),
            "reference": "thu-pacman/chitu installed unmodified under baseline/_ref (Triton %s, flash_attn)" % __import__("triton").__version__,
            "timing": "CUDA graph over rotating operand sets > L2, CUDA events, us per call", "ops": rows}


if __name__ == "__main__":
    out = main(int(sys.argv[1]) if len(sys.argv) > 1 else 16, sys.argv[2] if len(sys.argv) > 2 else "",
               sys.argv[3] if len(sys.argv) > 3 else "both")
    print(json.dumps(out))
