"""Persistent per-device workspaces (SURVEY.md §8b "Ownership": the C ABI never allocates; the
Python shim owns outputs and a persistent workspace so that decode steps are CUDA-graph safe).

CUDA-graph safety (the reference captures one graph per batch size in whatever order requests arrive,
models/model.py:537-622): a buffer that a captured kernel was given must never go back to the caching
allocator while that graph can still be replayed.  Therefore
  * a superseded buffer is RETIRED, not freed: it stays referenced here for the life of the process (sizes
    grow geometrically, so the retired buffers together are smaller than the live one);
  * `reserve_decode()` sizes every tag once for the largest decode batch, so that in steady state nothing
    grows at all (B200AttnBackend / plugin.install call it);
  * growing while the current stream is being captured raises: the zero-fill of the new buffer would be
    recorded into the graph and the ticket counters of the wgmma GEMM would be shared with eager calls.
"""
from __future__ import annotations

import torch

_ws = {}
_retired = []


def _round_up_pow2(n: int) -> int:
    n = max(int(n), 256)
    return 1 << (n - 1).bit_length()


def get(tag: str, nbytes: int, device) -> torch.Tensor:
    """Return a zero-initialised uint8 CUDA buffer of at least `nbytes` for (tag, device); grows, never shrinks,
    never frees what it handed out before."""
    dev = torch.device(device)
    key = (tag, dev.index if dev.index is not None else torch.cuda.current_device())
    buf = _ws.get(key)
    if buf is None or buf.numel() < nbytes:
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError(
                f"chitu_b200 workspace '{tag}' would have to grow to {nbytes} bytes during CUDA-graph capture; "
                "call chitu_b200.workspace.reserve_decode(max_reqs, ...) (or run one eager step at the largest "
                "batch size) before capturing")
        if buf is not None:
            _retired.append(buf)          # a captured graph may still point at it
        # zero-filled: the split-K ticket counters of the wgmma GEMM must start at 0 (they self-reset)
        buf = torch.zeros(_round_up_pow2(nbytes), dtype=torch.uint8, device=dev)
        _ws[key] = buf
    return buf


def reserve(tag: str, nbytes: int, device) -> None:
    get(tag, nbytes, device)


def reserve_decode(device, max_reqs: int, *, heads: int = 128, head_dim_v: int = 512, max_splits: int = 128,
                   max_out_features: int = 1 << 18, topk: int = 9, num_experts: int = 257, expert_n1: int = 4096,
                   expert_k: int = 7168, attn_cap_bytes: int = 256 << 20) -> None:
    """Size every workspace tag the plugin path uses for a decode batch of up to `max_reqs` requests, so that
    graphs captured at any smaller batch size, in any order, share buffers that never move."""
    from . import _lib

    lib = _lib.load()
    B = max(int(max_reqs), 1)
    splits = max_splits
    while splits > 1 and lib.chitu_b200_attn_workspace_bytes(B, heads, head_dim_v, splits) > attn_cap_bytes:
        splits //= 2
    reserve("attn", lib.chitu_b200_attn_workspace_bytes(B, heads, head_dim_v, splits), device)
    reserve("linear", lib.chitu_b200_linear_workspace_bytes(B, max_out_features), device)
    reserve("moe", lib.chitu_b200_moe_workspace_bytes(B, topk, num_experts, expert_n1, expert_k), device)
    reserve("moe_gate", lib.chitu_b200_moe_gate_workspace_bytes(B, max(num_experts, 8)), device)


def retired_bytes() -> int:
    return sum(b.numel() for b in _retired)


def clear() -> None:
    """Drop every buffer (tests only: never while a captured graph is alive)."""
    _ws.clear()
    _retired.clear()
