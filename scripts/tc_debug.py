"""GPU debugging aid for the wgmma GEMM: runs each case in isolation and prints the first error."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from chitu_b200 import ops, _lib
from oracle import chitu_oracle as O

dev = "cuda:0"
torch.manual_seed(0)

def report(name, y, r):
    y, r = y.float().cpu(), r.float().cpu()
    err = (y - r).abs().max().item()
    rel = err / r.abs().max().clamp(min=1e-30).item()
    bad = (~torch.isfinite(y)).sum().item()
    print(f"{name}: max_abs {err:.4e} rel {rel:.3e} nonfinite {bad} "
          f"{'OK' if rel < 8e-3 and bad == 0 else 'MISMATCH'}", flush=True)
    if rel >= 8e-3:
        d = (y - r).abs()
        idx = d.flatten().topk(5).indices
        for i in idx.tolist():
            m, n = divmod(i, y.shape[-1])
            print(f"    [{m},{n}] got {y.flatten()[i]:.5f} want {r.flatten()[i]:.5f}")

cases = [(5, 64, 512), (3, 16, 512), (5, 192, 512), (16, 128, 64), (16, 128, 128), (16, 256, 512), (1, 4096, 4096), (16, 6144, 4096), (5, 384, 1024),
         (16, 2112, 7168), (33, 512, 256), (100, 1024, 1024)]
for impl in (2,):
    ops.LINEAR_IMPL = impl
    for (M, N, K) in cases:
        x = torch.randn(M, K).bfloat16()
        w = (torch.randn(N, K) * 0.05).bfloat16()
        try:
            y = ops.linear(x.to(dev), w.to(dev))
            torch.cuda.synchronize()
            report(f"bf16 impl{impl} M{M} N{N} K{K}", y, O.linear(x, w))
        except Exception as e:
            print(f"bf16 impl{impl} M{M} N{N} K{K}: EXC {e}", flush=True)
            break

def fp8w(N, K):
    w = torch.randn(N, K) * 0.05
    nb, kb = (N + 127) // 128, (K + 127) // 128
    wp = torch.zeros(nb * 128, kb * 128); wp[:N, :K] = w
    blocks = wp.view(nb, 128, kb, 128)
    s = blocks.abs().amax(dim=(1, 3)) / 448.0
    q = (blocks / s[:, None, :, None]).reshape(nb * 128, kb * 128)[:N, :K].to(torch.float8_e4m3fn)
    return q.contiguous(), s.float().contiguous()

ops.LINEAR_IMPL = 2
for (M, N, K) in [(16, 128, 128), (16, 256, 512), (1, 2112, 7168), (16, 3072, 1536), (16, 7168, 2048), (7, 7168, 256), (40, 512, 1024)]:
    a = (torch.randn(M, K) * 2).bfloat16()
    aq, a_s = O.act_quant_deepseek_v3(a)
    bq, b_s = fp8w(N, K)
    try:
        c = ops.fp8_gemm_deepseek_v3(aq.to(dev), a_s.to(dev), bq.to(dev), b_s.to(dev))
        torch.cuda.synchronize()
        report(f"fp8 M{M} N{N} K{K}", c, O.fp8_gemm(aq, a_s, bq, b_s, out_dtype=torch.float32))
    except Exception as e:
        print(f"fp8 M{M} N{N} K{K}: EXC {e}", flush=True)
        break

from chitu_b200.quantize import w8a8gemm
w8a8gemm.IMPL = 2
for (M, N, K) in [(16, 128, 128), (2, 4096, 11008), (64, 2048, 4096)]:
    a = (torch.randn(M, K) * 4).to(torch.int8)
    b = (torch.randn(N, K) * 4).to(torch.int8)
    sa, sb = torch.rand(M) * 0.01 + 0.001, torch.rand(N) * 0.01 + 0.001
    out = torch.zeros(M, N, dtype=torch.float16, device=dev)
    try:
        w8a8gemm.mm(out, a.to(dev), b.to(dev), sa.to(dev), sb.to(dev), None)
        torch.cuda.synchronize()
        report(f"i8 M{M} N{N} K{K}", out, O.w8a8_mm(a, b, sa, sb))
    except Exception as e:
        print(f"i8 M{M} N{N} K{K}: EXC {e}", flush=True)
        break

# timing of the weight-streaming GEMM vs SIMT at the LLaMA / DeepSeek shapes
def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

try:
    for (M, N, K) in [(16, 28672, 4096), (1, 28672, 4096), (16, 6144, 4096), (16, 4096, 14336), (16, 4096, 4096)]:
        ws = [(torch.randn(N, K, device=dev) * 0.05).bfloat16() for _ in range(12)]   # > L2 in total
        x = torch.randn(M, K, device=dev).bfloat16()
        for impl in (1, 2):
            ops.LINEAR_IMPL = impl
            i = [0]
            def f():
                ops.linear(x, ws[i[0] % len(ws)]); i[0] += 1
            ms = timeit(f, 24)
            print(f"time bf16 impl{impl} M{M} N{N} K{K}: {ms*1e3:.1f} us  {N*K*2/ms/1e6:.0f} GB/s", flush=True)
        del ws
except Exception as e:
    print("timing EXC", e)
ops.LINEAR_IMPL = 0
