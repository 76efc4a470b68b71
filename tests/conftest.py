import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


class Golden:
    """npz fixture written by oracle/gen_golden.py (bf16 stored as uint16 bits, fp8 as uint8).  Large seeded inputs are
    regenerated (oracle/golden_inputs.py) and near-copies rebuilt from their deltas; both must match the stored SHA-256."""

    def __init__(self, name):
        import hashlib

        from oracle.golden_inputs import regenerate

        raw = np.load(os.path.join(GOLDEN, name + ".npz"))
        z = {k: raw[k] for k in raw.files if "__" not in k or not k.rsplit("__", 1)[1] in ("sha256", "delta_base", "delta_idx", "delta_val")}
        z.update(regenerate(name))
        for k in raw.files:
            if k.endswith("__delta_base"):
                key = k[: -len("__delta_base")]
                a = z[str(raw[k])].copy()
                a.reshape(-1)[raw[key + "__delta_idx"]] = raw[key + "__delta_val"]
                z[key] = a
        for k in raw.files:
            if k.endswith("__sha256"):
                key = k[: -len("__sha256")]
                assert hashlib.sha256(np.ascontiguousarray(z[key]).tobytes()).hexdigest() == str(raw[k]), \
                    f"{name}.npz: rebuilt {key} differs from the recorded input"
        self.z = z

    def np(self, key):
        return self.z[key]

    def t(self, key, dtype=None):
        a = self.z[key]
        if dtype == torch.bfloat16:
            return torch.from_numpy(a.view(np.int16).copy()).view(torch.bfloat16)
        if dtype == torch.float8_e4m3fn:
            return torch.from_numpy(a.copy()).view(torch.float8_e4m3fn)
        t = torch.from_numpy(np.array(a))
        return t if dtype is None else t.to(dtype)


@pytest.fixture
def golden():
    return Golden


def cos_diff(a: torch.Tensor, b: torch.Tensor) -> float:
    """FlashMLA's criterion (third_party/FlashMLA/tests/test_flash_mla.py:31-37)."""
    a, b = a.double().flatten(), b.double().flatten()
    denom = (a * a + b * b).sum().item()
    if denom == 0:
        return 0.0
    return 1.0 - 2.0 * (a * b).sum().item() / denom


def max_rel(a: torch.Tensor, b: torch.Tensor) -> float:
    """max |a-b| / max|b| (relative to the reference's dynamic range)."""
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-30)).item()
