"""dev tool: where the wgmma MLA decode kernel spends its time INSIDE the decode graph (profiling build of the library,
csrc/mla_tc.cu probe()): every CTA records %globaltimer at fixed points; the last layer's launch is what remains.

    python scripts/mla_probe.py [bs] [layers]
prints, over the CTAs of that launch, the median / min / max offset of every probe from the earliest CTA start."""
import dataclasses
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
_TL = os.path.join(ROOT, "chitu_b200", "libchitu_b200_tl.so")
if not os.path.exists(_TL):
    subprocess.run(["make", "-C", os.path.join(ROOT, "chitu_b200", "csrc"), "tl"], check=True, capture_output=True)
os.environ["CHITU_B200_LIB"] = _TL
import ctypes

import torch

from chitu_b200 import _lib

NAMES = {0: "cta start", 30: "first TMA issued", 1: "softmax: past griddepcontrol.wait", 2: "Q staged", 31: "MMA: q_ready seen",
         28: "last P.V done", 29: "epilogue stores issued"}
for i in range(12):
    NAMES[3 + 2 * i] = f"tile {i}: S ready"
    NAMES[4 + 2 * i] = f"tile {i}: P published"


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    layers = int(sys.argv[2]) if len(sys.argv) > 2 else 6
    S = 4096
    lib = _lib.load()
    lib.chitu_b200_debug_mla_probe.restype = ctypes.c_int
    lib.chitu_b200_debug_mla_probe.argtypes = [ctypes.c_void_p]
    from chitu_b200.engine_deepseek import DEEPSEEK_R1, DeepSeekDecodeEngine
    cfg = dataclasses.replace(DEEPSEEK_R1, n_layers=layers)
    eng = DeepSeekDecodeEngine(cfg, max_reqs=B, max_seq_len=S + 256, tp_size=8)
    eng.set_synthetic_context(S)
    eng.tokens.copy_(torch.randint(100, 1000, (B,)))
    for _ in range(2):
        eng._step_body()
    torch.cuda.synchronize()
    eng.seq_lens.fill_(S)
    eng.capture()
    for _ in range(3):
        eng.step()
    torch.cuda.synchronize()
    ncta = 4096
    buf = torch.zeros(ncta * 32, dtype=torch.int64, device="cuda")
    _lib.check(lib.chitu_b200_debug_mla_probe(buf.data_ptr()), "probe")
    eng.seq_lens.fill_(S)
    eng.step()
    torch.cuda.synchronize()
    lib.chitu_b200_debug_mla_probe(None)
    p = buf.view(ncta, 32).cpu()
    used = [i for i in range(ncta) if int(p[i, 0]) != 0]
    t0 = min(int(p[i, 0]) for i in used)
    print(f"deepseek tp8 shard bs={B} ctx={S}: {len(used)} CTAs in the MLA launch of the last layer")
    order = [0, 30, 1, 2, 31] + [3 + k for k in range(24)] + [28, 29]
    prev_med = None
    for idx in order:
        vals = [(int(p[i, idx]) - t0) / 1e3 for i in used if int(p[i, idx]) != 0]
        if not vals:
            continue
        med = statistics.median(vals)
        d = "" if prev_med is None else f"   (+{med - prev_med:5.2f})"
        print(f"  {NAMES[idx]:38s} n={len(vals):4d}  median {med:6.2f} us   min {min(vals):6.2f}   max {max(vals):6.2f}{d}")
        prev_med = med
    # per-CTA durations
    dur = [(int(p[i, 29]) - int(p[i, 0])) / 1e3 for i in used if int(p[i, 29]) != 0]
    print(f"  CTA lifetime (start -> epilogue): median {statistics.median(dur):.2f} us, min {min(dur):.2f}, max {max(dur):.2f}")
    last = max(int(p[i, 29]) for i in used)
    print(f"  first CTA start -> last CTA epilogue: {(last - t0) / 1e3:.2f} us")


if __name__ == "__main__":
    main()
