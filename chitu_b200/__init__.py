"""chitu_b200 — H100-native (sm_90a) decode operators behind Chitu's plugin surfaces.

Host side mirrors the reference's operator interfaces (same names / argument meaning):
  chitu_b200.ops            <-> chitu.ops
  chitu_b200.attn_backend   <-> chitu.attn_backend
  chitu_b200.fused_moe      <-> chitu.fused_moe
  chitu_b200.chitu_backend  <-> chitu_backend (pybind module, csrc/binding.cpp)
  chitu_b200.quantize       <-> chitu.quantize.w8a8 (+ closed w8a8gemm / w8a8gemv)
All of them call libchitu_b200.so through the C ABI in include/chitu_b200.h.
`chitu_b200.install()` patches them into an importable `chitu` package (INTEGRATION.md).
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401


def install():
    from .plugin import install as _install

    return _install()
