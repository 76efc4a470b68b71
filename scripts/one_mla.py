"""dev tool: a few wgmma MLA decode launches at the bench shape (B=16, S=4096, H=16) for `ncu --set full`"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from chitu_b200.attn_backend import B200AttnBackend

B, ctx, H, C, R, page = int(sys.argv[1]) if len(sys.argv) > 1 else 16, 4096, 16, 512, 64, 64
per = (ctx + page) // page
caches = [torch.randn(B * per, page, C + R, device="cuda", dtype=torch.bfloat16) for _ in range(4)]
bt = torch.randperm(B * per, device="cuda", dtype=torch.int32).view(B, per).contiguous()
excl = torch.full((B,), ctx - 1, device="cuda", dtype=torch.int32)
q_nope = torch.randn(B, H, C, device="cuda", dtype=torch.bfloat16)
q_pe = torch.randn(B, H, R, device="cuda", dtype=torch.bfloat16)
kv = torch.randn(B, 1, 1, C + R, device="cuda", dtype=torch.bfloat16)
be = B200AttnBackend(max_seq_len=ctx, max_reqs=B, n_local_heads=H)
for i in range(4):
    o = be.mla_attn_with_kvcache(q_nope, q_pe, caches[i], kv, excl, excl + 1, bt, softmax_scale=0.1352)
torch.cuda.synchronize()
print(float(o.float().abs().mean()))
