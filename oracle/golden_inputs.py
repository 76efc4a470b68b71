"""Large seeded inputs of the golden files, regenerated instead of stored.

The generators (oracle/gen_golden.py, oracle/gen_golden_models.py) draw their inputs from seeded CPU torch generators.
Where those inputs are hundreds of kilobytes of random weights or caches, the .npz keeps only the reference's outputs
plus a SHA-256 of every input left out (key `<name>__sha256`); tests/conftest.py rebuilds the input with the same draws
and refuses to use it unless the digest matches.  An output that differs from an input in a few places (a cache after
an append) is stored as that input plus the changed elements (`<name>__delta_base`, `__delta_idx`, `__delta_val`).
"""
import hashlib

import numpy as np
import torch

BF = torch.bfloat16


def bits(t: torch.Tensor) -> np.ndarray:
    """The storage format of the golden files: bf16 as uint16 bits, everything else as is."""
    if t.dtype == BF:
        return t.contiguous().view(torch.int16).numpy().view(np.uint16)
    return t.contiguous().numpy()


def _append_kv():
    g = torch.Generator().manual_seed(12)                                  # gen_golden.gen_append
    return {"cache_before": torch.randn(20, 64, 576, generator=g).bfloat16()}


def _ref_attn_gqa():
    g = torch.Generator().manual_seed(20)                                  # gen_golden.gen_ref_attn
    k = torch.randn(3, 300, 2, 128, generator=g).bfloat16()
    v = torch.randn(3, 300, 2, 128, generator=g).bfloat16()
    return {"k_cache": k, "v_cache": v}


def _gate_sigmoid_f32bias():
    g = torch.Generator().manual_seed(18)                                  # gen_golden.gen_gate
    return {"weight": (torch.randn(256, 7168, generator=g) * 0.02).bfloat16()}


def _fused_experts():
    g = torch.Generator().manual_seed(17)                                  # gen_golden.gen_fused_experts
    torch.randn(3, 256, generator=g)                                       # x (stored)
    w1 = (torch.randn(8, 256, 256, generator=g) * 0.05).bfloat16()
    w2 = (torch.randn(8, 256, 128, generator=g) * 0.05).bfloat16()
    return {"w1": w1, "w2": w2}


def _block_llama():
    # gen_golden_models.gen_llama_block: global seed 21, default dtype bf16, the block's parameters in registration order
    g = torch.Generator().manual_seed(21)
    out = {"k_cache": torch.randn(3, 48, 2, 32, generator=g, dtype=BF), "v_cache": torch.randn(3, 48, 2, 32, generator=g, dtype=BF)}
    params = [("attention__wq__weight", (256, 256)), ("attention__wk__weight", (64, 256)), ("attention__wv__weight", (64, 256)),
              ("attention__wo__weight", (256, 256)), ("feed_forward__w1__weight", (704, 256)),
              ("feed_forward__w2__weight", (256, 704)), ("feed_forward__w3__weight", (704, 256)),
              ("attention_norm__weight", (256,)), ("ffn_norm__weight", (256,))]
    for name, shape in params:
        r = torch.randn(*shape, generator=g, dtype=BF)
        out[name] = 1.0 + 0.1 * r if "norm" in name else r * 0.05
    return out


def _block_mixtral_moe():
    # gen_golden_models.gen_mixtral_moe: global seed 41, default dtype bf16, gate then (gate_up, down) per expert
    g = torch.Generator().manual_seed(41)
    torch.randn(8, 256, generator=g, dtype=BF)                             # gate.weight (stored)
    w1, w2 = [], []
    for _ in range(8):
        w1.append(torch.randn(768, 256, generator=g, dtype=BF) * 0.06)
        w2.append(torch.randn(256, 384, generator=g, dtype=BF) * 0.06)
    return {"w1": torch.stack(w1), "w2": torch.stack(w2)}


RECIPES = {"append_kv": _append_kv, "ref_attn_gqa": _ref_attn_gqa, "gate_sigmoid_f32bias": _gate_sigmoid_f32bias,
           "fused_experts": _fused_experts, "block_llama": _block_llama, "block_mixtral_moe": _block_mixtral_moe}


def regenerate(name: str) -> dict:
    """{key: numpy array in storage format} of the inputs of golden file `name` that are not stored in it."""
    fn = RECIPES.get(name)
    return {} if fn is None else {k: bits(v) for k, v in fn().items()}


# outputs stored as a delta against one of the file's inputs: {file: {output key: base key}}
DELTAS = {"append_kv": {"cache_after": "cache_before"}, "ref_attn_gqa": {"k_cache_after": "k_cache", "v_cache_after": "v_cache"},
          "block_llama": {"k_after": "k_cache", "v_after": "v_cache"}}


def _sha256(a: np.ndarray) -> np.ndarray:
    return np.array(hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest())


def compact(name: str, arrays: dict) -> dict:
    """The stored form of golden file `name` from its full {key: numpy array} (storage format): regenerable inputs are
    replaced by their SHA-256, DELTAS outputs by base key + changed flat indices + values (+ SHA-256)."""
    regen = regenerate(name)
    out = {}
    for k, v in arrays.items():
        if k in regen:
            assert np.array_equal(regen[k], v), f"{name}: {k} is not what oracle/golden_inputs.py regenerates"
            out[k + "__sha256"] = _sha256(v)
        elif k in DELTAS.get(name, {}):
            base = arrays[DELTAS[name][k]]
            idx = np.flatnonzero(base.reshape(-1) != v.reshape(-1)).astype(np.int64)
            out[k + "__delta_base"] = np.array(DELTAS[name][k])
            out[k + "__delta_idx"] = idx
            out[k + "__delta_val"] = v.reshape(-1)[idx]
            out[k + "__sha256"] = _sha256(v)
        else:
            out[k] = v
    return out
