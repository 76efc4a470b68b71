"""CPU-side checks: the C-ABI library loads and exports every symbol include/chitu_b200.h
declares, argument validation returns status codes (never exits), the host shims refuse CPU
tensors (no fallback), the roofline byte model matches BASELINE.md, and the tensor-parallel
host logic (world_size 2, gloo) equals the unsharded result."""
import ctypes
import os
import re
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from chitu_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "chitu_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(chitu_b200_\w+)\s*\(", hdr))
    assert len(declared) >= 25
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    assert lib.chitu_b200_version() >= 100


def test_bad_arguments_return_status_not_abort():
    from chitu_b200 import _lib
    lib = _lib.load()
    rc = lib.chitu_b200_append_paged_kv(None, None, None, None, 1, 1, 64, 64, 1152, None)
    assert rc < 0 and b"append_paged_kv" in lib.chitu_b200_last_error()
    rc = lib.chitu_b200_moe_align_block_size(None, _lib.CB_F32, 0, 8, 16, None, None, None, None, None)
    assert rc < 0
    rc = lib.chitu_b200_mla_decode(None, None, None, None, None, None, 1, 1, 16, 512, 64, 64, 4, 0, 1.0, None, None, 0, None)
    assert rc < 0
    with pytest.raises(RuntimeError):
        _lib.check(rc, "mla_decode")
    # the MLA kernel stages whole 64-token pages: any other page size is refused before anything is dereferenced
    dummy = 16
    rc = lib.chitu_b200_mla_decode(dummy, dummy, dummy, None, dummy, dummy, 1, 1, 16, 512, 64, 32, 4, 0, 1.0, None, None, 0, None)
    assert rc < 0 and b"page" in lib.chitu_b200_last_error()
    assert lib.chitu_b200_attn_workspace_bytes(16, 16, 512, 8) > 16 * 16 * 8 * 512 * 4
    # out = NULL leaves the partials in the workspace, which must hold one split; any workspace must hold the split plan
    for out, ws, ws_bytes in ((None, None, 0), (None, dummy, 100), (dummy, dummy, 100)):
        rc = lib.chitu_b200_mla_decode(dummy, dummy, dummy, None, dummy, dummy, 1, 1, 16, 512, 64, 64, 4, 0, 1.0, out, ws,
                                       ws_bytes, None)
        assert rc < 0 and b"workspace" in lib.chitu_b200_last_error()
    # the merging absorb-o reads the partials of the split count it recomputes: one split here, one byte missing
    one_split = lib.chitu_b200_attn_workspace_bytes(1, 16, 512, 1)
    rc = lib.chitu_b200_mla_absorb_o_merge_quant(dummy, one_split - 1, 4096, dummy, None, dummy, None, None, 1, 16, 128,
                                                 128, 512, None)
    assert rc < 0 and b"workspace" in lib.chitu_b200_last_error()


# chitu_b200_mla_num_splits(B, H, hint, workspace_bytes): {(B, H): one row per hint in _HINTS, one column per size in _WS}
_HINTS, _WS = (200, 4096, 65536), (0, 100, 1 << 18, 1 << 22, 256 << 20)
_MLA_SPLITS = {
    (1, 16): [[1, 1, 2, 2, 2], [1, 1, 7, 32, 32], [1, 1, 7, 127, 128]],
    (1, 40): [[1, 1, 2, 2, 2], [1, 1, 3, 32, 32], [1, 1, 3, 44, 44]],
    (1, 128): [[1, 1, 1, 2, 2], [1, 1, 1, 15, 16], [1, 1, 1, 15, 16]],
    (3, 16): [[1, 1, 2, 2, 2], [1, 1, 2, 32, 32], [1, 1, 2, 42, 44]],
    (3, 40): [[1, 1, 1, 2, 2], [1, 1, 1, 14, 14], [1, 1, 1, 14, 14]],
    (3, 128): [[1, 1, 1, 2, 2], [1, 1, 1, 5, 5], [1, 1, 1, 5, 5]],
    (8, 16): [[1, 1, 1, 2, 2], [1, 1, 1, 15, 16], [1, 1, 1, 15, 16]],
    (8, 40): [[1, 1, 1, 2, 2], [1, 1, 1, 5, 5], [1, 1, 1, 5, 5]],
    (8, 128): [[1, 1, 1, 1, 2], [1, 1, 1, 1, 2], [1, 1, 1, 1, 2]],
}


def test_split_counts_and_workspace_sizes_are_pinned():
    """The host arithmetic of the split-KV workspace: the MLA split count, the workspace size of a split count and the
    capped size the Python side allocates."""
    from chitu_b200 import _lib, workspace
    lib = _lib.load()
    got = {bh: [[lib.chitu_b200_mla_num_splits(*bh, hint, n) for n in _WS] for hint in _HINTS] for bh in _MLA_SPLITS}
    assert got == _MLA_SPLITS
    for args, want in (((1, 1, 64, 1), 516), ((16, 16, 512, 8), 4202752), ((16, 128, 512, 128), 537919744),
                       ((256, 32, 128, 64), 270532864), ((3, 40, 128, 5), 309856)):
        assert lib.chitu_b200_attn_workspace_bytes(*args) == want, args
    for args, want in (((1, 128, 512), 33620224), ((64, 128, 512), 134480128), ((256, 32, 128), 135266560),
                       ((4096, 128, 512), 1075839232)):
        assert workspace.attn_bytes(*args) == want, args


def test_round2_entries_validate_arguments():
    """The entries added in round 2 return status codes on bad arguments like the rest of the ABI (no GPU needed)."""
    from chitu_b200 import _lib
    lib = _lib.load()
    # push-mode reduce: no communicator
    assert lib.chitu_b200_allreduce_consume(None, None, None, None, None, None, None, 1, 4096, 1e-6, None) < 0
    assert lib.chitu_b200_linear_bf16_ar(None, None, 1, 4096, 4096, None, None, 0, None) < 0
    assert lib.chitu_b200_fp8_gemm_ar(None, None, None, None, 1, 4096, 4096, None, None, 0, None) < 0
    assert lib.chitu_b200_comm_status(None) < 0
    area, nbytes, calls = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_void_p()
    assert lib.chitu_b200_debug_comm_push_area(None, ctypes.byref(area), ctypes.byref(nbytes), ctypes.byref(calls)) < 0
    assert b"debug_comm_push_area" in lib.chitu_b200_last_error()
    # device-side step preparation / plan / sampling
    assert lib.chitu_b200_decode_prepare(None, None, None, 1, None, None, None, 1, 64, 1, None) < 0
    assert lib.chitu_b200_sample_top_k_top_p(None, 128, 1, 128, _lib.CB_BF16, None, None, None, None, None, None, None, None) < 0
    assert lib.chitu_b200_linear_bf16_silu_pairs(None, None, None, 1, 7, 64, None, 0, None) < 0      # odd N
    assert lib.chitu_b200_moe_gate_workspace_bytes(16, 256) >= 16 * 256 * 2 + 256


def test_product_code_never_reads_the_reference_install():
    """baseline/_ref (the unmodified reference) is a bench / script comparator only."""
    pkg = os.path.join(ROOT, "chitu_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                # (docstrings cite reference file:line; what must not exist is code that loads it)
                assert "baseline/_ref" not in src and not re.search(r"sys\.path[^\n]*reference", src), os.path.join(dirpath, f)


def test_no_cpu_fallback():
    from chitu_b200 import fused_moe, ops
    from chitu_b200.attn_backend import B200AttnBackend
    x = torch.randn(2, 256).bfloat16()
    with pytest.raises(RuntimeError):
        ops.act_quant_deepseek_v3(x)
    with pytest.raises(RuntimeError):
        ops.linear(x, torch.randn(8, 256).bfloat16())
    with pytest.raises(RuntimeError):
        fused_moe.moe_align_block_size(torch.zeros(4, dtype=torch.int32), 16, 8)
    be = B200AttnBackend()
    with pytest.raises(RuntimeError):
        be.mla_attn_with_kvcache(torch.zeros(1, 16, 512).bfloat16(), torch.zeros(1, 16, 64).bfloat16(),
                                 torch.zeros(2, 64, 576).bfloat16(), None, torch.zeros(1, dtype=torch.int32),
                                 torch.zeros(1, dtype=torch.int32), torch.zeros(1, 2, dtype=torch.int32))


def test_product_code_never_imports_the_oracle():
    """Prompt (3): only tests/, smoke() and bench.py's cpu_baseline leg may touch oracle/."""
    pat = re.compile(r"^\s*(from\s+oracle|import\s+oracle|from\s+\.+\s*oracle)|oracle/|chitu_oracle", re.M)
    pkg = os.path.join(ROOT, "chitu_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not pat.search(src), os.path.join(dirpath, f)


def test_roofline_byte_model_matches_baseline_md():
    sys.path.insert(0, ROOT)
    import bench
    from chitu_b200.engine import LLAMA3_8B
    b1 = bench.bytes_per_step(LLAMA3_8B, 1, 4096, 1)[0]
    b16 = bench.bytes_per_step(LLAMA3_8B, 16, 4096, 1)[0]
    # BASELINE.md §2 quotes 16.6 GB / 24.65 GB including the 1.05 GB embedding table; a decode step
    # only gathers B rows of it, so the algorithmic model here excludes it.
    emb = 128256 * 4096 * 2 / 1e9
    assert abs(b1 / 1e9 - (16.6 - emb)) < 0.15
    assert abs(b16 / 1e9 - (24.65 - emb)) < 0.15
    assert LLAMA3_8B.ffn_dim == 14336


def _tp_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from chitu_b200 import tensor_parallel as tp
    tp.init_tp()
    torch.manual_seed(0)
    x = torch.randn(4, 64)
    w1, b1 = torch.randn(96, 64), torch.randn(96)
    w2, b2 = torch.randn(64, 96), torch.randn(64)
    op = lambda a, w, b=None: torch.nn.functional.linear(a, w, b)    # test double for the CUDA linear_op
    col = tp.ColumnParallelLinear.from_full(w1, b1, gather_output=False, linear_op=op)
    row = tp.RowParallelLinear.from_full(w2, b2, input_is_parallel=True, linear_op=op)
    y = row(torch.relu(col(x)))
    ref = torch.nn.functional.linear(torch.relu(torch.nn.functional.linear(x, w1, b1)), w2, b2)
    colg = tp.ColumnParallelLinear.from_full(w1, b1, gather_output=True, linear_op=op)
    # reference constructor / attributes (tensor_parallel.py:42-169): parameters, in/out_features, default input slicing
    rowd = tp.RowParallelLinear(96, 64, has_bias=True, dtype=torch.float32, linear_op=op)
    rowd.weight.data, rowd.bias.data = tp.shard_cols(w2, rank, world), b2.clone()
    assert rowd.in_features == 96 and rowd.out_features == 64 and 'weight' in dict(rowd.named_parameters())
    full_act = torch.relu(torch.nn.functional.linear(x, w1, b1))
    assert torch.allclose(rowd(full_act), ref, atol=1e-4)          # input_is_parallel=False slices the full activation
    ok = torch.allclose(y, ref, atol=1e-4) and torch.allclose(colg(x), torch.nn.functional.linear(x, w1, b1), atol=1e-5)
    # vocab-parallel greedy sampling: (max, index) all-gather == argmax of the all-gathered logits, ties -> lowest index
    g = torch.Generator().manual_seed(7)
    full = torch.randn(5, 40, generator=g).bfloat16()
    full[1, 3] = full[1, 25] = 9.0          # tie across the two shards -> index 3
    full[2, 30] = full[2, 38] = 9.0         # tie inside the upper shard -> index 30
    local = full[:, rank * 20:(rank + 1) * 20].contiguous()
    gathered = torch.empty(world, 5, 2)
    tok = tp.global_argmax(local, local.float().argmax(dim=1), rank, 20, None, gathered)
    ok = ok and torch.equal(tok, full.float().argmax(dim=1)) and int(tok[1]) == 3 and int(tok[2]) == 30
    # vocab-parallel embedding: masked local lookup (test double of the CUDA op) + all_reduce == full lookup
    table = torch.randn(40, 16, generator=g)

    def emb_double(ids, local, start):
        inside = (ids >= start) & (ids < start + local.shape[0])
        out = torch.nn.functional.embedding((ids - start).clamp(0, local.shape[0] - 1), local)
        return out * inside[..., None]
    ids = torch.tensor([0, 19, 20, 39, 7, 33])
    emb = tp.VocabParallelEmbedding.from_full(table, embedding_op=emb_double)
    ok = ok and torch.equal(emb(ids), torch.nn.functional.embedding(ids, table))
    ret[rank] = bool(ok)
    dist.destroy_process_group()


def test_tensor_parallel_world2_gloo():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, port, ret)) for r in range(2)]
    [p.start() for p in procs]
    [p.join(120) for p in procs]
    assert ret.get(0) and ret.get(1)


def test_clock_sampler_windows_samples(tmp_path, monkeypatch):
    """bench.ClockSampler keeps only the samples that arrive between mark_begin() and mark_end() and reports throttle
    reasons (fake nvidia-smi on PATH; the real one is sampled during the timed region on the GPU box)."""
    import importlib.util
    import stat
    import time

    fake = tmp_path / "nvidia-smi"
    fake.write_text("#!/bin/sh\nwhile true; do echo '0, 1965, 1965, 700.0, 0x0, Not Active, Not Active, Not Active, Active'; sleep 0.05; done\n")
    fake.chmod(fake.stat().st_mode | stat.S_IEXEC)
    monkeypatch.setenv("PATH", f"{tmp_path}:{os.environ['PATH']}")
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    s = bench.ClockSampler(0)
    s.start()
    time.sleep(0.3)
    n_before = len(s.samples)
    s.mark_begin()
    time.sleep(0.4)
    s.mark_end()
    time.sleep(0.2)
    out = s.stop()
    assert n_before >= 2                                  # sampling started before the window ...
    assert 3 <= out["samples"] <= 12                      # ... but only the window is reported
    assert out["sm_mhz"] == 1965.0 and out["sm_max_mhz"] == 1965.0
    assert out["reasons"] == ["sw_power_cap"]
    assert bench.host_cores() >= 1


def test_w8a8_linear_dispatch_and_buffers(monkeypatch):
    """W8A8Linear host logic with CPU doubles for the three CUDA entry points: buffer names / dtypes of the reference
    checkpoints (quantize/w8a8.py:53-78), mv for [bs <= 4, seq, K], mm otherwise, bias added once, from_float."""
    from chitu_b200.quantize import w8a8 as M
    calls = []

    def quant_act_double(x):
        r = x.reshape(-1, x.shape[-1]).float()
        s = r.abs().amax(dim=-1).clamp(min=1e-5) / 127.0
        return torch.round(r / s[:, None]).to(torch.int8), s

    def mm_double(out, a, b, a_s, b_s, bias=None):
        calls.append("mm")
        out.copy_(((a.float() @ b.float().T) * a_s[:, None] * b_s[None, :]).half())

    def mv_double(a, b, a_s, b_s):
        calls.append("mv")
        bs, seq, K = a.shape
        return ((a.reshape(-1, K).float() @ b.float().T) * a_s[:, None] * b_s[None, :]).half().view(bs, seq, -1)

    monkeypatch.setattr(M, "quant_act", quant_act_double)
    monkeypatch.setattr(M.w8a8gemm, "mm", mm_double)
    monkeypatch.setattr(M.w8a8gemv, "mv", mv_double)
    torch.manual_seed(0)
    lin = torch.nn.Linear(64, 24, bias=True).half()
    q = M.W8A8Linear.from_float(lin)
    q.act_quant = quant_act_double                      # the constructor captured the CUDA function
    sd = q.state_dict()
    assert set(sd) == {"weight", "scale_channel", "bias"}       # from_float re-binds `bias` to the source Parameter
    assert list(M.W8A8Linear(64, 24).state_dict()) == ["weight", "scale_channel", "bias"]
    assert sd["weight"].dtype == torch.int8 and sd["weight"].shape == (24, 64)
    assert sd["scale_channel"].dtype == torch.float32 and sd["bias"].dtype == torch.float16
    wq, ws = M.quant_weight(lin.weight.data)
    assert torch.equal(wq, sd["weight"]) and torch.equal(ws, sd["scale_channel"])
    # quant_weight == the reference formula (scales.clamp_(1e-5).div_(127); w.div(scales).round_())
    sc = lin.weight.data.abs().max(dim=-1, keepdim=True)[0].to(torch.float)
    sc.clamp_(min=1e-5).div_(127.0)
    assert torch.equal(wq, lin.weight.data.div(sc).round_().to(torch.int8)) and torch.equal(ws, sc.view(-1))
    for shape, want in (((5, 64), "mm"), ((2, 3, 64), "mv"), ((4, 1, 64), "mv"), ((6, 3, 64), "mm")):
        calls.clear()
        x = torch.randn(*shape).half()
        y = q(x)
        qa, sa = quant_act_double(x)
        ref = ((qa.float() @ wq.float().T) * sa[:, None] * ws[None, :]).half().view(*shape[:-1], 24) + lin.bias.data
        assert calls == [want] and y.shape == (*shape[:-1], 24) and y.dtype == torch.float16
        assert torch.allclose(y.float(), ref.float(), atol=2e-3)
    nb = M.W8A8Linear(8, 4, bias=False)
    assert nb.bias is None and "bias" not in nb.state_dict()
    arch = M.W8A8Linear.from_float(lin, model_arch_only=True)
    assert int(arch.weight.abs().sum()) == 0 and "W8A8Linear(64, 24, bias=True)" in repr(arch)


def test_linear_deepseek_v3_dispatch(monkeypatch):
    """ops.linear_deepseek_v3 (model_deepseek_v3.py:53-106): three-way dispatch on the weight's element size and the
    soft-fp8 switch, leading dims kept, bias added once — with CPU doubles for the CUDA operators."""
    from chitu_b200 import ops
    calls = []
    monkeypatch.setattr(ops, "linear", lambda x, w, b=None: (calls.append("linear"), torch.nn.functional.linear(x, w, b))[1])
    monkeypatch.setattr(ops, "soft_fp8_gemm_deepseek_v3",
                        lambda a, b, s: (calls.append("soft"), torch.zeros(a.shape[0], b.shape[0], dtype=a.dtype))[1])
    monkeypatch.setattr(ops, "act_quant_deepseek_v3", lambda x, bs=128: (calls.append("quant"), (x, torch.ones(x.shape[0], 1)))[1])
    monkeypatch.setattr(ops, "fp8_gemm_deepseek_v3",
                        lambda a, a_s, b, b_s: (calls.append("fp8"), torch.ones(a.shape[0], b.shape[0], dtype=a.dtype))[1])
    x = torch.randn(2, 3, 256).bfloat16()
    w16 = torch.randn(8, 256).bfloat16()
    w8 = torch.zeros(8, 256, dtype=torch.float8_e4m3fn)
    sc = torch.ones(1, 2)
    bias = torch.full((8,), 2.0).bfloat16()
    assert ops.linear_deepseek_v3(x, w16).shape == (2, 3, 8) and calls == ["linear"]
    y = ops.linear_deepseek_v3(x, w8, sc, bias)
    assert calls[1:] == ["quant", "fp8"] and y.shape == (2, 3, 8) and torch.all(y == 3.0)
    y = ops.linear_deepseek_v3(x, w8, sc, soft_fp8=True)
    assert calls[3:] == ["soft"] and y.shape == (2, 3, 8)
    monkeypatch.setattr(ops, "SOFT_FP8", True)
    ops.linear_deepseek_v3(x, w8, sc)
    assert calls[-1] == "soft"
    with pytest.raises(AssertionError):
        ops.linear_deepseek_v3(x, w8)                  # one-byte weights need their scales


def test_reference_arm_samples_run_on_the_host():
    """bench.py --impl reference: the bounded sample runs through the UNMODIFIED reference (baseline/_ref) when it is installed,
    and falls back to the oracle port — saying why — when it is not."""
    sys.path.insert(0, ROOT)
    import bench
    from chitu_b200.engine import LlamaConfig
    cfg = LlamaConfig(dim=256, n_layers=2, n_heads=8, n_kv_heads=2, vocab_size=512, multiple_of=64, ffn_dim_multiplier=None)
    smp, how = bench.reference_sample(cfg, 2, 40)
    try:
        assert smp.layer() > 0 and smp.head() > 0 and smp.full_step_seconds(1.0, 0.5) == 2.5
        if os.path.isdir(os.path.join(ROOT, "baseline", "_ref", "chitu")):
            assert smp.kind == "reference" and "baseline/_ref" in how
        else:
            assert smp.kind == "port" and "not runnable" in how
    finally:
        if hasattr(smp, "close"):
            smp.close()
    port = bench.CpuSample(cfg, 2, 40, page=16)
    assert port.kind == "port" and port.layer() > 0

