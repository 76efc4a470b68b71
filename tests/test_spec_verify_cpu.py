"""The speculative verify step without a GPU: the refusals of the greedy acceptance entry, its Python wrapper and the
LLaMA engine's verify step, and the verify step's library calls recorded with test_engine_calls_cpu's stand-ins."""
import json

import pytest
import torch

import test_engine_calls_cpu as EC

K = 3                     # drafts per request in the traced engines; EC._llama has 3 requests
ATTN = ("chitu_b200_gqa_paged_decode_rope", "chitu_b200_gqa_paged_attn_fp8kv")


def _lib():
    from chitu_b200 import _lib as L
    return L.load()


def test_c_entry_refuses_bad_arguments_and_launches_nothing():
    from chitu_b200._lib import launch_count
    lib = _lib()
    A = 1 << 20                              # stand-ins: every case is refused before a dereference
    ptrs = dict(target=A, drafts=2 * A, n_draft=3 * A, seq_lens=4 * A, out=5 * A, accepted=6 * A, nxt=7 * A)

    def call(**kw):
        v = dict(ptrs, B=4, k=3)
        v.update(kw)
        return lib.chitu_b200_spec_accept_greedy(v["target"], v["drafts"], v["n_draft"], v["seq_lens"], v["out"],
                                                 v["accepted"], v["nxt"], v["B"], v["k"], None)

    before = launch_count()
    for kw in [{name: None} for name in ptrs] + [dict(B=-1), dict(k=0), dict(k=-2)]:
        assert call(**kw) < 0, kw
        assert "chitu_b200_spec_accept_greedy" in lib.chitu_b200_last_error().decode(), kw
    assert call(B=0) == 0                    # nothing to do
    assert launch_count() == before


def test_wrapper_refusals():
    from chitu_b200._lib import launch_count
    from chitu_b200.ops import accept_draft_tokens_greedy as acc
    _lib()
    i64, i32 = torch.int64, torch.int32
    B, k = 4, 3
    ok = dict(target=torch.zeros(B, k + 1, dtype=i64), drafts=torch.zeros(B, k, dtype=i64),
              n_draft=torch.zeros(B, dtype=i32), seq_lens=torch.zeros(B, dtype=i32))
    before = launch_count()
    bad = [dict(target=None),
           dict(target=torch.zeros(B, k + 1, dtype=i32)), dict(drafts=torch.zeros(B, k, dtype=i32)),
           dict(n_draft=torch.zeros(B, dtype=i64)), dict(seq_lens=torch.zeros(B, dtype=i64)),
           dict(target=torch.zeros(B, 1, dtype=i64)), dict(target=torch.zeros(B * (k + 1), dtype=i64)),
           dict(drafts=torch.zeros(B, k + 1, dtype=i64)), dict(n_draft=torch.zeros(B + 1, dtype=i32)),
           dict(seq_lens=torch.zeros(B, 1, dtype=i32)),
           dict(drafts=torch.zeros(k, B, dtype=i64).t())]
    for kw in bad + [{}]:                    # {}: CPU tensors are refused too
        args = dict(ok, **kw)
        with pytest.raises(ValueError):
            acc(args["target"], args["drafts"], args["n_draft"], args["seq_lens"])
    assert launch_count() == before


def test_engine_refusals():
    with pytest.raises(ValueError, match="max_draft"):
        EC._llama(128, max_draft=-1)
    with pytest.raises(ValueError, match="linear_impl"):
        EC._llama(128, max_draft=2, linear_impl=1)
    with pytest.raises(ValueError, match="head dim"):
        EC._llama(64, max_draft=2)
    with pytest.raises(ValueError, match="multiple of 64"):
        EC._llama(128, max_draft=2, page_size=32)
    with pytest.raises(ValueError, match="256 rows"):
        EC._llama(128, max_draft=85)                 # 3 * 86 rows
    EC._llama(128, max_draft=84)                     # 3 * 85 = 255 rows
    eng = EC._llama(128)
    for call in (lambda: eng.verify(torch.zeros(3, dtype=torch.int64), torch.zeros(3, 1, dtype=torch.int64),
                                    torch.zeros(3, dtype=torch.int32)), eng.capture_verify, eng.verify_step):
        with pytest.raises(ValueError, match="max_draft"):
            call()
    eng = EC._llama(128, max_draft=K)
    tok, nd = torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int32)
    for drafts, n in ((torch.zeros(3, K + 1, dtype=torch.int64), nd),          # wider than max_draft
                      (torch.zeros(2, K, dtype=torch.int64), nd),
                      (torch.zeros(3, K, dtype=torch.int64), torch.zeros(2, dtype=torch.int32)),
                      (torch.zeros(3, K, dtype=torch.int64), torch.full((3,), K + 1, dtype=torch.int32)),
                      (torch.zeros(3, 1, dtype=torch.int64), torch.full((3,), 2, dtype=torch.int32)),
                      (torch.zeros(3, K, dtype=torch.int64), torch.full((3,), -1, dtype=torch.int32))):
        with pytest.raises(ValueError):
            eng.verify(tok, drafts, n)
    with pytest.raises(ValueError, match="tokens"):
        eng.verify(torch.zeros(2, dtype=torch.int64), torch.zeros(3, K, dtype=torch.int64), nd)


# ------------------------------------------------------------------------------------------------------ call lists
VERIFY_MODES = {
    "single": (dict(), None),
    "single_e4m3_kv": (dict(kv_dtype=torch.float8_e4m3fn), None),
    "single_w4a16": (dict(weight_format="w4a16"), None),
    "single_fp8": (dict(weight_format="fp8"), None),
    "shard": (dict(tp_size=2), None),
    "tp_push": (EC._TP, "push"),
    "tp_pull": (EC._TP, "pull"),
    "tp_nccl": (EC._TP, "nccl"),
}


def _trace(kw, reduce, body):
    rec = EC.Recorder()
    with EC._patched(rec):
        eng = EC._llama(128, **kw)
        if reduce is not None:
            eng.comm = None if reduce == "nccl" else EC.FakeComm(rec)
            eng.ar_push = reduce == "push"
        rec.watch(eng)
        getattr(eng, body)()
    return eng, rec


@pytest.mark.parametrize("mode", list(VERIFY_MODES))
def test_verify_step_calls(mode):
    """The verify step is the decode step's calls over B * (k + 1) rows, with the attention call replaced by the rotary
    over those rows and the multi-token attention at sq = k + 1, and the acceptance kernel last."""
    kw, reduce = VERIFY_MODES[mode]
    _, dec = _trace(kw, reduce, "_step_body")                       # the decode step of an engine without drafts
    eng, rec = _trace(dict(kw, max_draft=K), reduce, "_verify_body")
    B, R, sq = eng.B, eng.B * (K + 1), K + 1
    D, Hq, Hkv = eng.D, eng.Hq, eng.Hkv
    qkv_w = (Hq + 2 * Hkv) * D
    p = lambda t: rec.pointer(t.data_ptr())                         # noqa: E731
    for t in (eng.h, eng.h2, eng.xn, eng.qkv, eng.attn_out, eng.act, eng.logits, eng.q_rot, eng.k_rot, eng.verify_cos):
        assert t.shape[0] == R
    if eng.weight_format == "fp8":
        assert eng.xq.shape[0] == R and eng.xs.shape[0] == R

    # names: the decode step's, each attention call -> rotary + multi-token attention, then the acceptance
    attn = "chitu_b200_gqa_paged_attn_fp8kv" if eng.kv_fp8 else "chitu_b200_gqa_paged_prefill"
    want = []
    for c in dec.calls:
        want += ["chitu_b200_rotary_interleaved", attn] if c[0] in ATTN else [c[0]]
    names = [c[0] for c in rec.calls]
    assert names == want + ["chitu_b200_spec_accept_greedy"]

    # every row count is B * (k + 1)
    rows_at = {"chitu_b200_embedding": 4, "chitu_b200_rmsnorm": 4, "chitu_b200_linear_bf16": 6,
               "chitu_b200_linear_bf16_silu_pairs": 4, "chitu_b200_argmax": 3, "chitu_b200_rotary_interleaved": 7,
               "chitu_b200_add": 4, "chitu_b200_w4a16_gemm": 7, "chitu_b200_w4a16_gemm_silu_pairs": 6,
               "chitu_b200_fp8_rowwise_gemm": 8, "chitu_b200_fp8_rowwise_gemm_silu_pairs": 6,
               "chitu_b200_quant_fp8_rowwise": 4, "chitu_b200_rmsnorm_quant_fp8_rowwise": 6,
               "comm.linear_push": 3, "comm.consume": 7, "comm": 8}
    for c in rec.calls:
        if c[0] in rows_at:
            want_rows = R * eng.cfg.dim if c[0] == "chitu_b200_add" else R
            assert c[rows_at[c[0]]] == want_rows, c
    emb = rec.calls[0]
    assert emb[1] == p(eng.verify_tokens)

    # attention: q and k rotated into q_rot / k_rot, v from the qkv output, sq = k + 1 over B requests, causal
    for li in range(len(eng.layers)):
        rot = [c for c in rec.calls if c[0] == "chitu_b200_rotary_interleaved"][li]
        at = [c for c in rec.calls if c[0] == attn][li]
        assert rot[1:7] == [p(eng.qkv), [p(eng.qkv)[0], Hq * D * 2], p(eng.q_rot), p(eng.k_rot), p(eng.verify_cos),
                            p(eng.verify_sin)]
        assert rot[8:15] == [Hq, Hkv, D, qkv_w, D, qkv_w, D]
        v_ptr = [p(eng.qkv)[0], (Hq + Hkv) * D * 2]
        strides = [sq * Hkv * D, Hkv * D, sq * qkv_w, qkv_w]
        if eng.kv_fp8:
            assert at[1:11] == [p(eng.q_rot), sq * Hq * D, p(eng.k_cache[li]), p(eng.v_cache[li]), p(eng.k_rot),
                                v_ptr] + strides
            assert at[11:13] == [None, None]                       # no fused rotary
            rest = at[13:]
        else:
            assert at[1:10] == [p(eng.q_rot), p(eng.k_cache[li]), p(eng.v_cache[li]), p(eng.k_rot), v_ptr] + strides
            rest = at[10:]
        assert rest[:12] == [p(eng.seq_lens), p(eng.block_table), eng.max_blocks, B, sq, Hq, Hkv, D, eng.page,
                             eng.k_cache.shape[1], eng.max_seq_len, 1]
        assert rest[13:16] == [p(eng.attn_out), p(eng.verify_attn_ws), eng.verify_attn_ws.numel()]

    # the head's argmax into target, then (tensor parallel) the global argmax over B * (k + 1) rows
    am = [c for c in rec.calls if c[0] == "chitu_b200_argmax"]
    assert len(am) == 1 and am[0][1:5] == [p(eng.logits), p(eng.target), R, eng.head.shape[0]]
    if eng.tp_on:
        g = [c for c in rec.calls if c[0] == "dist.all_gather_into_tensor"]
        assert len(g) == 1 and g[0][1] == p(eng.verify_gather) and tuple(eng.verify_gather.shape) == (2, R, 2)
    acc = rec.calls[-1]
    assert acc[1:] == [p(eng.target), p(eng.draft_tokens), p(eng.n_draft), p(eng.seq_lens), p(eng.out_tokens),
                       p(eng.accepted), p(eng.next_tokens), B, K, 0]


@pytest.mark.parametrize("mode", ["llama_single_rope", "llama_tp_push", "llama_tp_pull", "llama_tp_nccl"])
def test_decode_step_unchanged_with_drafts(mode):
    """An engine built for drafts runs exactly the golden decode step."""
    with open(EC.GOLDEN) as f:
        want = json.load(f)[mode]
    kw, reduce = {"llama_single_rope": (dict(), None), "llama_tp_push": (EC._TP, "push"),
                  "llama_tp_pull": (EC._TP, "pull"), "llama_tp_nccl": (EC._TP, "nccl")}[mode]
    _, rec = _trace(dict(kw, max_draft=K), reduce, "_step_body")
    assert json.loads(json.dumps(rec.calls)) == want
