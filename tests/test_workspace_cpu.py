"""The persistent workspaces of the plugin path (chitu_b200/workspace.py), on the host: for the decode shapes of the
models the reference serves, `reserve_decode(max_reqs)` with its default arguments (what `plugin.install(max_reqs)`
passes) leaves every tag at least as large as each plugin function asks at every batch size B <= max_reqs, so the
per-batch-size CUDA graphs never make a tag grow.

A request is computed the way the plugin function computes it: `ops._linear_ws`, `fused_moe._chunks` and
`B200AttnBackend._ws` are run with `workspace.get` recording the (tag, bytes) they ask for; `moe_gate` and the
quantised linear modules are restated from their one-line byte requests.  The buffer a reservation leaves is the
request rounded up to a power of two, as `workspace.get` allocates it.  Needs only the built library."""
import sys

import pytest
import torch

from chitu_b200 import _lib, fused_moe, ops, plugin, workspace
from chitu_b200.attn_backend import B200AttnBackend

MAX_REQS = (16, 64, 256)
VERIFY_K = (1, 2, 3, 4, 7)              # drafts per request of a speculative verify step: B * (k + 1) rows
DECODE_TAGS = ("attn", "linear", "moe", "moe_gate")


class Recorder:
    def __init__(self):
        self.asked = []

    def get(self, tag, nbytes, device):
        self.asked.append((tag, int(nbytes)))
        return torch.empty(0, dtype=torch.uint8)


@pytest.fixture
def recorder(monkeypatch):
    r = Recorder()
    monkeypatch.setattr(workspace, "get", r.get)
    return r


def reserved(max_reqs, **shapes):
    """{tag: bytes of the buffer reserve_decode(max_reqs, **shapes) leaves}."""
    left = {}
    orig = workspace.reserve
    try:
        workspace.reserve = lambda tag, nbytes, device: left.__setitem__(tag, workspace._round_up_pow2(nbytes))
        workspace.reserve_decode("cpu", max_reqs, **shapes)
    finally:
        workspace.reserve = orig
    return left


# ------------------------------------------------------------------------------------------- model tables
def llama3_8b(tp):
    return dict(name=f"llama3-8b-tp{tp}", dim=4096, Hq=32 // tp, D=128,
                linears=[(6144 // tp, 4096), (4096, 4096 // tp), (2 * 14336 // tp, 4096), (4096, 14336 // tp),
                         (128256 // tp, 4096)],
                verify=True)


def mixtral_8x7b(tp):
    return dict(name=f"mixtral-8x7b-tp{tp}", dim=4096, Hq=32 // tp, D=128,
                linears=[(6144 // tp, 4096), (4096, 4096 // tp), (32000 // tp, 4096)],
                gate=(8, 4096), experts=(2, 8, 2 * 14336 // tp, 4096))


def deepseek_r1(tp):
    H = 128 // tp
    return dict(name=f"deepseek-r1-tp{tp}", dim=7168, H=H,
                linears=[(1536 + 512 + 64, 7168), (H * 192, 1536), (7168, H * 128), (2 * 18432 // tp, 7168),
                         (7168, 18432 // tp), (129280 // tp, 7168)],
                gate=(256, 7168), experts=(9, 257, 2 * 2048 // tp, 7168))


def quantised_linears():
    """The LLaMA-3-8B linears through W4A16Linear and Fp8Linear (their forward asks linear_workspace_bytes(max(M, 1),
    N), W8A8's w8a8gemm.mm linear_workspace_bytes(M, N))."""
    return dict(name="w4a16-fp8-w8a8-llama3-8b", linears=llama3_8b(1)["linears"], modules=True)


MODELS = ([llama3_8b(tp) for tp in (1, 2, 4, 8)] + [mixtral_8x7b(tp) for tp in (1, 2, 4)]
          + [deepseek_r1(tp) for tp in (8, 16)] + [quantised_linears()])


def requests(model, B, rec):
    """Every (tag, bytes) the model's plugin calls ask of the workspaces at decode batch B."""
    lib = _lib.load()
    rec.asked.clear()
    rows = [B] + ([B * (k + 1) for k in VERIFY_K] if model.get("verify") else [])
    for M in rows:
        for N, _K in model["linears"]:
            ops._linear_ws(M, N, "cpu")
            if model.get("modules"):
                rec.asked.append(("linear", lib.chitu_b200_linear_workspace_bytes(max(M, 1), N)))
    be = B200AttnBackend(n_local_heads=model.get("H", 128))
    if "Hq" in model:                                  # GQA decode and verify: one workspace call per batch
        be._ws(B, model["Hq"], model["D"], "cpu")
    if "H" in model:                                   # absorbed MLA: latent rows of 512
        be._ws(B, model["H"], 512, "cpu")
    if "gate" in model:
        E, _dim = model["gate"]
        rec.asked.append(("moe_gate", lib.chitu_b200_moe_gate_workspace_bytes(B, E)))
    if "experts" in model:
        topk, E, N1, K1 = model["experts"]
        for _ in fused_moe._chunks(lib, B, topk, E, N1, K1, "cpu"):
            pass
    return list(rec.asked)


@pytest.mark.parametrize("max_reqs", MAX_REQS)
def test_default_reservation_covers_every_model_at_every_batch(max_reqs, recorder):
    """reserve_decode(max_reqs) with no shapes: every request of every model table, at every B <= max_reqs, fits the
    buffer left for its tag, and nothing asks for a tag reserve_decode does not reserve."""
    left = reserved(max_reqs)
    assert set(left) == set(DECODE_TAGS), left
    short = []
    for model in MODELS:
        for B in range(1, max_reqs + 1):
            for tag, nbytes in requests(model, B, recorder):
                if nbytes > left.get(tag, 0):
                    short.append(f"{model['name']} B={B}: '{tag}' asks {nbytes} > {left.get(tag, 0)}")
    assert not short, "\n".join(short[:20])


def test_linear_workspace_stops_growing_at_the_widest_token_tile():
    """The reservation of "linear" relies on it: no M asks more than M = LINEAR_MAX_TILE_ROWS does."""
    lib = _lib.load()
    top = lib.chitu_b200_linear_workspace_bytes(workspace.LINEAR_MAX_TILE_ROWS, 4096)
    assert lib.chitu_b200_linear_workspace_bytes(workspace.LINEAR_MAX_TILE_ROWS // 2, 4096) < top
    for M in (1, 16, 17, 64, 65, 127, 200, 1024, 8192, 65536):
        assert lib.chitu_b200_linear_workspace_bytes(M, 4096) <= top


def test_each_tag_is_reserved_once_for_the_largest_batch():
    """Reservations are monotone in max_reqs, and a reservation at max_reqs covers every smaller one."""
    prev = None
    for max_reqs in (1, 3, 8, 16, 32, 64, 256):
        left = reserved(max_reqs)
        if prev is not None:
            assert all(left[t] >= prev[t] for t in DECODE_TAGS), (max_reqs, left, prev)
        prev = left


def test_install_reserves_with_default_shapes(monkeypatch):
    """plugin.install(max_reqs) calls reserve_decode(device, max_reqs) and passes no shapes: the defaults are what the
    table above is checked against; install() without max_reqs reserves nothing."""
    calls = []
    monkeypatch.setattr(workspace, "reserve_decode", lambda *a, **kw: calls.append((a, kw)))
    for name in ("chitu_backend", "w8a8gemm", "w8a8gemv"):
        monkeypatch.delitem(sys.modules, name, raising=False)
    plugin.install(max_reqs=32, device="cpu")
    assert calls == [(("cpu", 32), {})]
    plugin.install(device="cpu")
    assert len(calls) == 1


def test_grouped_gemm_workspace_is_left_unreserved():
    """"moe_gg" (invoke_fused_moe_kernel, the reference's per-GEMM entry) is not a decode tag: at DeepSeek-R1 tp8
    shapes it would ask hundreds of MB (moe_align_block_size pads every expert to a block), so reserve_decode leaves it
    alone.  That is safe because fused_experts never calls it (the GPU test pins that, and that its first use inside a
    capture raises)."""
    lib = _lib.load()
    topk, E, N1, K1 = 9, 257, 2 * 2048 // 8, 7168
    for max_reqs in MAX_REQS:
        em = max_reqs * topk + E * (128 - 1)                # moe_align_block_size's padded length at BLOCK_SIZE_M 128
        gg = lib.chitu_b200_moe_grouped_gemm_workspace_bytes(em, N1, K1)
        assert gg > 256 << 20, gg
        assert "moe_gg" not in reserved(max_reqs)
