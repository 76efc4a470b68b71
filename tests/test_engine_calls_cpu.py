"""The library calls of one decode or verify step of every engine, in every mode, pinned without a GPU.

Each engine is built at toy sizes on the CPU with a recording stand-in for libchitu_b200, a fake fused all-reduce and
recording `torch.distributed` collectives, and one `_step_body()` (or LLaMA's `_verify_body()`) runs.  Every call is
recorded with its arguments; a pointer becomes (buffer number, byte offset), with buffers numbered in order of first
appearance, so the trace changes when a launch reads or writes a different buffer but not when an attribute is
renamed.  The traces are compared with
tests/golden/engine_calls.json: a change to the engines that should not alter what runs on the GPU must leave them
equal.  `python tests/test_engine_calls_cpu.py --write` regenerates the file after an intended change; its diff then
shows which launches changed."""
import argparse
import contextlib
import ctypes
import json
import os
import sys
import types
from unittest import mock

import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden", "engine_calls.json")
WS_BYTES = 1 << 16           # what every *_workspace_bytes query returns
PG = object()                # stands in for a process group


class Recorder:
    def __init__(self):
        self.calls = []
        self.storages = {}   # base pointer -> bytes, of every tensor the engine holds
        self.ids = {}        # base pointer -> buffer number
        self.on = False      # construction-time calls are not part of the step

    def watch(self, eng):
        def walk(o):
            if isinstance(o, torch.Tensor):
                s = o.untyped_storage()
                self.storages[s.data_ptr()] = s.nbytes()
            elif isinstance(o, dict):
                for v in o.values():
                    walk(v)
            elif isinstance(o, (list, tuple)):
                for v in o:
                    walk(v)
        walk(vars(eng))
        self.on = True

    def pointer(self, p):
        if p is None or p == 0:
            return p
        for base, n in self.storages.items():
            if base <= p < base + n:
                return [self.ids.setdefault(base, len(self.ids)), p - base]
        raise AssertionError(f"pointer {p:#x} is not inside any buffer the engine holds")

    def record(self, name, args):
        out = [name]
        for a in args:
            if isinstance(a, torch.Tensor):
                held = a.untyped_storage().data_ptr() in self.storages
                out.append(self.pointer(a.data_ptr()) if held else ["tmp", str(a.dtype), list(a.shape)])
            elif a is PG:
                out.append("pg")
            else:
                out.append(a)
        self.calls.append(out)


class FakeLib:
    def __init__(self, rec):
        self._rec = rec

    def __getattr__(self, name):
        from chitu_b200 import _lib
        _, argtypes = _lib.SIGNATURES[name]

        def call(*args):
            if name.endswith("_workspace_bytes"):
                return WS_BYTES
            if not self._rec.on:
                return 0
            assert len(args) == len(argtypes), f"{name}: {len(args)} arguments, the C entry takes {len(argtypes)}"
            self._rec.calls.append([name] + [self._rec.pointer(a) if t is ctypes.c_void_p else a
                                             for a, t in zip(args, argtypes)])
            return 0
        return call


class FakeComm:
    def __init__(self, rec):
        self._rec = rec

    def __call__(self, *args):
        self._rec.record("comm", args)

    def __getattr__(self, name):
        return lambda *args: self._rec.record("comm." + name, args)


@contextlib.contextmanager
def _patched(rec):
    from chitu_b200 import _lib
    lib = FakeLib(rec)

    def all_gather_into_tensor(out, inp, group=None):
        out.zero_()
        rec.record("dist.all_gather_into_tensor", (out, inp, group))

    with mock.patch.object(_lib, "load", lambda: lib), \
            mock.patch.object(torch.cuda, "current_stream", lambda *a, **k: types.SimpleNamespace(cuda_stream=0)), \
            mock.patch.object(dist, "all_reduce", lambda t, group=None: rec.record("dist.all_reduce", (t, group))), \
            mock.patch.object(dist, "all_gather_into_tensor", all_gather_into_tensor):
        yield


def _llama(head_dim=128, **kw):
    from chitu_b200.engine import LlamaConfig, LlamaDecodeEngine
    cfg = LlamaConfig(dim=512, n_layers=2, n_heads=512 // head_dim, n_kv_heads=2, vocab_size=1024, multiple_of=256,
                      ffn_dim_multiplier=None)
    return LlamaDecodeEngine(cfg, max_reqs=3, max_seq_len=512, device="cpu", **kw)


def _deepseek(**kw):
    from chitu_b200.engine_deepseek import DeepSeekConfig, DeepSeekDecodeEngine
    cfg = DeepSeekConfig(vocab_size=1024, dim=512, inter_dim=1024, moe_inter_dim=256, n_layers=2, n_dense_layers=1,
                         n_heads=4, n_routed_experts=16, n_activated_experts=4, n_expert_groups=4, n_limited_groups=2,
                         q_lora_rank=256)
    return DeepSeekDecodeEngine(cfg, max_reqs=3, max_seq_len=512, device="cpu", **kw)


def _mixtral(**kw):
    from chitu_b200.engine_mixtral import MixtralConfig, MixtralDecodeEngine
    cfg = MixtralConfig(dim=512, n_layers=2, n_heads=4, n_kv_heads=2, vocab_size=1024, intermediate_dim=512,
                        num_local_experts=4, num_experts_per_tok=2)
    return MixtralDecodeEngine(cfg, max_reqs=3, max_seq_len=512, device="cpu", **kw)


_TP = dict(tp_size=2, process_group=PG, use_fused_allreduce=False)
_E4M3 = dict(kv_dtype=torch.float8_e4m3fn)
_VERIFY = dict(max_draft=3)
_SAMPLED = dict(max_draft=3, sampled_verify=True)
STEP, VERIFY = "_step_body", "_verify_body"

# mode -> (engine factory, reduce mode under tensor parallelism: "push" / "pull" (fake comm) / "nccl" (no comm),
#          the engine method that runs the step: the decode step or the speculative verify step)
MODES = {
    "llama_single_rope": (lambda: _llama(128), None, STEP),
    "llama_single_unfused_rope": (lambda: _llama(64), None, STEP),
    "llama_linear_impl1": (lambda: _llama(128, linear_impl=1), None, STEP),
    "llama_tp_push": (lambda: _llama(128, **_TP), "push", STEP),
    "llama_tp_pull": (lambda: _llama(128, **_TP), "pull", STEP),
    "llama_tp_nccl": (lambda: _llama(128, **_TP), "nccl", STEP),
    "deepseek_single": (lambda: _deepseek(tp_size=1), None, STEP),
    "deepseek_shard": (lambda: _deepseek(tp_size=2), None, STEP),
    "deepseek_tp_push": (lambda: _deepseek(**_TP), "push", STEP),
    "deepseek_tp_pull": (lambda: _deepseek(**_TP), "pull", STEP),
    "deepseek_tp_nccl": (lambda: _deepseek(**_TP), "nccl", STEP),
    "deepseek_e4m3_kv": (lambda: _deepseek(tp_size=1, **_E4M3), None, STEP),
    "mixtral_shard": (lambda: _mixtral(tp_size=2), None, STEP),
    "mixtral_tp_push": (lambda: _mixtral(**_TP), "push", STEP),
    "mixtral_tp_pull": (lambda: _mixtral(**_TP), "pull", STEP),
    "mixtral_tp_nccl": (lambda: _mixtral(**_TP), "nccl", STEP),
    "llama_w4a16": (lambda: _llama(128, weight_format="w4a16"), None, STEP),
    "llama_w4a16_shard": (lambda: _llama(128, tp_size=2, weight_format="w4a16"), None, STEP),
    "llama_fp8": (lambda: _llama(128, weight_format="fp8"), None, STEP),
    "llama_e4m3_kv": (lambda: _llama(128, **_E4M3), None, STEP),
    "llama_fp8_e4m3_kv": (lambda: _llama(128, weight_format="fp8", **_E4M3), None, STEP),
    "mixtral_w4a16": (lambda: _mixtral(tp_size=1, weight_format="w4a16"), None, STEP),
    "mixtral_w4a16_shard": (lambda: _mixtral(tp_size=2, weight_format="w4a16"), None, STEP),
    "llama_verify": (lambda: _llama(128, **_VERIFY), None, VERIFY),
    "llama_verify_tp_push": (lambda: _llama(128, **_VERIFY, **_TP), "push", VERIFY),
    "llama_verify_w4a16": (lambda: _llama(128, **_VERIFY, weight_format="w4a16"), None, VERIFY),
    "llama_verify_fp8_e4m3_kv": (lambda: _llama(128, **_VERIFY, weight_format="fp8", **_E4M3), None, VERIFY),
    "llama_verify_sampled_fp8_draft_probs": (lambda: _llama(128, **_SAMPLED, weight_format="fp8", draft_probs=True),
                                             None, VERIFY),
    "llama_verify_sampled": (lambda: _llama(128, **_SAMPLED), None, VERIFY),
}


def trace(mode):
    make, reduce, body = MODES[mode]
    rec = Recorder()
    with _patched(rec):
        eng = make()
        if reduce is not None:
            eng.comm = None if reduce == "nccl" else FakeComm(rec)
            eng.ar_push = reduce == "push"
        rec.watch(eng)
        getattr(eng, body)()
    return json.loads(json.dumps(rec.calls))


@pytest.mark.parametrize("mode", list(MODES))
def test_engine_launch_sequence(mode):
    with open(GOLDEN) as f:
        want = json.load(f)[mode]
    got = trace(mode)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{mode}: call {i} differs"
    assert len(got) == len(want), f"{mode}: {len(got)} calls, golden has {len(want)}"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--write", action="store_true", help=f"write every mode's trace to {os.path.relpath(GOLDEN, ROOT)}")
    args = ap.parse_args()
    traces = {m: trace(m) for m in MODES}
    if not args.write:
        for m, calls in traces.items():
            print(f"{m}: {len(calls)} calls")
        return
    lines = []
    for m, calls in traces.items():
        body = ",\n".join("  " + json.dumps(c) for c in calls)
        lines.append(f"{json.dumps(m)}: [\n{body}\n]")
    with open(GOLDEN, "w") as f:
        f.write("{\n" + ",\n".join(lines) + "\n}\n")


if __name__ == "__main__":
    main()
