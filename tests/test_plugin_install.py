"""`chitu_b200.install()` against the REAL reference package (a thu-pacman/chitu checkout named by $CHITU_REFERENCE;
skipped without one): every operator name the reference's model files hold is rebound to this library's
implementation, and each replacement accepts the reference's parameters (drop-in signature check)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("CHITU_REFERENCE", "")

SCRIPT = r"""
import inspect, json, os, sys, types
sys.path.insert(0, %(ref)r); sys.path.insert(0, %(root)r)
import torch
sys.modules['chitu_backend'] = types.ModuleType('chitu_backend')           # fused_moe.py:20 imports it at import time
for n in ('w8a8gemm', 'w8a8gemv'):
    sys.modules[n] = types.ModuleType(n)
import chitu.device_type as D
D._device_name = 'cpu'
import chitu.ops, chitu.fused_moe, chitu.attn_backend
import chitu.models.model, chitu.models.model_deepseek_v3                   # hold the operators BY NAME
import chitu_b200
from chitu_b200 import plugin, ops, fused_moe, attn_backend, chitu_backend

names = plugin._OPS + plugin._MOE
orig = {n: getattr(chitu.ops if n in plugin._OPS else chitu.fused_moe, n) for n in names}
def params(f):
    f = getattr(f, '__wrapped__', f)
    names = [p.name for p in inspect.signature(f).parameters.values()]
    if names == ['args', 'kwargs'] and getattr(f, '__closure__', None):     # @auto_retry_triton_compilation wrapper
        for cell in f.__closure__:
            if inspect.isfunction(cell.cell_contents):
                return params(cell.cell_contents)
    return names
ref_params = {n: params(orig[n]) for n in names}
patched = plugin.install()
ours = {n: getattr(ops if n in plugin._OPS else fused_moe, n) for n in names}
res = {'patched': len(patched), 'rebound': {}, 'holders': {}, 'sig': {}}
for n in names:
    res['rebound'][n] = getattr(chitu.ops if n in plugin._OPS else chitu.fused_moe, n) is ours[n]
    res['sig'][n] = {'ref': ref_params[n], 'ours': params(ours[n])}
for mod in (chitu.models.model, chitu.models.model_deepseek_v3, chitu.attn_backend):
    for n in names:
        if hasattr(mod, n):
            res['holders'][mod.__name__ + '.' + n] = getattr(mod, n) is ours[n]
res['backend_module'] = sys.modules['chitu_backend'] is chitu_backend
res['has_cuda_moe_align'] = hasattr(sys.modules['chitu_backend'], 'cuda_moe_align_block_size')
res['attn'] = chitu.attn_backend.B200AttnBackend is attn_backend.B200AttnBackend
res['attn_methods'] = {m: params(getattr(attn_backend.B200AttnBackend, m)) == params(getattr(chitu.attn_backend.AttnBackend, m))
                       for m in ('attn_varlen_func', 'attn_with_kvcache')}
# the abstract prepare_metadata_for_decode is (*args, **kwargs): compare with the concrete paged-MLA backend
res['attn_methods']['prepare_metadata_for_decode'] = (
    params(attn_backend.B200AttnBackend.prepare_metadata_for_decode) ==
    params(chitu.attn_backend.TritonAttnBackend.prepare_metadata_for_decode))
res['mla_params_ref'] = params(chitu.attn_backend.TritonAttnBackend.mla_attn_with_kvcache)
res['mla_params_ours'] = params(attn_backend.B200AttnBackend.mla_attn_with_kvcache)
print('RESULT' + json.dumps(res))
"""


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "chitu")), reason="needs a reference checkout ($CHITU_REFERENCE)")
def test_install_rebinds_every_holder_and_signatures_are_drop_in():
    env = dict(os.environ, TRITON_INTERPRET="1")
    out = subprocess.run([sys.executable, "-c", SCRIPT % {"ref": REF, "root": ROOT}], capture_output=True, text=True,
                         env=env, timeout=300)
    line = [l for l in out.stdout.splitlines() if l.startswith("RESULT")]
    assert line, out.stderr[-2000:]
    res = json.loads(line[0][len("RESULT"):])
    assert res["patched"] >= len(res["rebound"])
    assert all(res["rebound"].values()), res["rebound"]
    assert res["holders"] and all(res["holders"].values()), res["holders"]       # modules that imported by name
    assert res["backend_module"] and res["has_cuda_moe_align"] and res["attn"]
    for name, sig in res["sig"].items():
        # drop-in: the reference's positional parameters, in order, under the same names (ours may add trailing
        # keyword parameters with defaults)
        assert sig["ours"][:len(sig["ref"])] == sig["ref"], (name, sig)
    assert all(res["attn_methods"].values()), res["attn_methods"]
    assert res["mla_params_ours"][:len(res["mla_params_ref"])] == res["mla_params_ref"]
