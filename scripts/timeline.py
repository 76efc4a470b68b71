"""dev tool: per-kernel critical-path times INSIDE the CUDA graph of a decode step (csrc/common.cuh timeline facility).

    python scripts/timeline.py deepseek 16 [layers]      # or: llama 16 / mixtral 16
prints, per launch of ONE layer in the middle of the model, the time between this kernel passing its dependency wait and the
next one passing its own (= this kernel's critical-path time incl. the next launch's latency), then totals by entry."""
import dataclasses
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
# the stamps are compiled into a separate profiling build of the library only
_TL = os.path.join(ROOT, "chitu_b200", "libchitu_b200_tl.so")
if not os.path.exists(_TL):          # `make -C chitu_b200/csrc tl`
    subprocess.run(["make", "-C", os.path.join(ROOT, "chitu_b200", "csrc"), "tl"], check=True, capture_output=True)
os.environ["CHITU_B200_LIB"] = _TL
import torch

from chitu_b200 import _lib


def main():
    what = sys.argv[1] if len(sys.argv) > 1 else "deepseek"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 16
    layers = int(sys.argv[3]) if len(sys.argv) > 3 else 0
    S = 4096
    lib = _lib.load()
    cap = 8192
    buf = torch.zeros(2 + cap, dtype=torch.int64, device="cuda")
    buf[1] = cap
    if what == "deepseek":
        from chitu_b200.engine_deepseek import DEEPSEEK_R1, DeepSeekDecodeEngine
        cfg = dataclasses.replace(DEEPSEEK_R1, n_layers=layers or 8)
        eng = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, tp_size=8)
    elif what == "mixtral":
        from chitu_b200.engine_mixtral import MixtralConfig, MixtralDecodeEngine
        eng = MixtralDecodeEngine(MixtralConfig(n_layers=layers or 6), max_reqs=B, max_seq_len=S + 512, tp_size=4)
    else:
        from chitu_b200.engine import LLAMA3_8B, LlamaDecodeEngine
        eng = LlamaDecodeEngine(dataclasses.replace(LLAMA3_8B, n_layers=layers or 8), max_reqs=B, max_seq_len=S + 512)
    eng.set_synthetic_context(S)
    eng.tokens.copy_(torch.randint(100, 1000, (B,)))
    # warm up eagerly, then capture with the name log armed
    for _ in range(2):
        eng._step_body()
    torch.cuda.synchronize()
    eng.seq_lens.fill_(S)
    _lib.check(lib.chitu_b200_debug_timeline(buf.data_ptr()), "timeline")
    eng.capture()
    names = lib.chitu_b200_debug_timeline_names().decode().split("\n")[:-1]
    n = len(names)
    for _ in range(3):
        eng.step()
    torch.cuda.synchronize()
    runs = []
    for _ in range(5):
        buf[0] = 0
        torch.cuda.synchronize()
        eng.step()
        torch.cuda.synchronize()
        cnt = int(buf[0])
        runs.append(buf[2:2 + min(cnt, cap)].cpu().clone())
    lib.chitu_b200_debug_timeline(None)
    cnt = len(runs[-1])
    print(f"{what} bs={B}: {n} launches captured, {cnt} stamps per replay")
    if cnt != n:
        print("  (stamp count != launch count: kernels without a stamp or multi-stamp kernels; mapping by order may drift)")
    import statistics
    deltas = []
    for i in range(min(cnt, n) - 1):
        deltas.append(statistics.median([(int(r[i + 1]) - int(r[i])) / 1e3 for r in runs if len(r) > i + 1]))
    total = (int(runs[-1][min(cnt, n) - 1]) - int(runs[-1][0])) / 1e3
    print(f"first stamp -> last stamp: {total:.1f} us")
    # one period of the layer pattern: find the repeat length from the names
    agg = {}
    for i, d in enumerate(deltas):
        agg.setdefault(names[i], []).append(d)
    print("---- totals by entry (us, count, mean)")
    for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
        print(f"  {sum(v):9.1f}  {len(v):4d}  {sum(v) / len(v):7.2f}  {k}")
    print("---- launch by launch (last third of the step)")
    lo = max(0, len(deltas) - max(40, len(deltas) // 3))
    for i in range(lo, len(deltas)):
        print(f"  {i:4d} {deltas[i]:7.2f} us  {names[i]}")


if __name__ == "__main__":
    main()
