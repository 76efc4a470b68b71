"""ops.scatter_kv_to_cache (chitu_b200_scatter_kv): a batch of prompts' k / v or latent rows written into the KV cache in
one launch.  Every case is compared byte for byte with the reference's per-request torch loop over whole caches
pre-filled with NaN bytes, so the slots the scatter must not touch are checked as well: paged GQA caches in bf16 / fp16
/ e4m3 over page sizes 16 / 64 / 256, ragged lengths with empty and one-row requests that cross page boundaries from
mid-page starting positions, k / v as strided views of a fused qkv output (16-byte and narrow copies), the MLA latent
cache, non-paged caches with rows past capacity, the e4m3 clamp rule on its edge values, more than 65535 rows and
requests, CUDA-graph replay with new lengths, and a prompt written by the scatter then decoded, against the same prompt
appended by the seqlen_q > 1 attention paths."""
import pytest
import torch

from chitu_b200 import _lib, ops

DEV = "cuda:0"
BF, F16, E4M3 = torch.bfloat16, torch.float16, torch.float8_e4m3fn
LENS = [0, 1, 37, 0, 300, 2]            # ragged: empty and one-row requests, runs across page boundaries
STARTS = [5, 0, 15, 9, 250, 63]         # tokens already cached: mid-page prefixes (chunked prefill)
# e4m3 edge values: the clamp bound, the first values plain .to() turns into NaN, huge values, NaN, subnormals, ties
SPECIALS = [448.0, -448.0, 464.0, -464.0, 1e9, -1e9, float("nan"), 2.0 ** -9, -(2.0 ** -9), 3 * 2.0 ** -10,
            2.0 ** -10, 2.0 ** -7, 0.0, -0.0, 449.0, 500.0, 240.0, 17.0, 0.0625 + 2.0 ** -8, -1.125]


def _bits(t):
    """The tensor's bits as an integer tensor of the same shape (NaN payloads compare equal)."""
    return t.view({1: torch.uint8, 2: torch.int16}[t.element_size()])


def nan_tensor(shape, dtype):
    """A tensor of `shape` whose every byte is 0xFF (NaN in bf16, fp16 and e4m3fn)."""
    esize = torch.empty((), dtype=dtype).element_size()
    return torch.full((*shape[:-1], shape[-1] * esize), 0xFF, dtype=torch.uint8, device=DEV).view(dtype)


def stored(rows, cache_dtype):
    """What a cache of `cache_dtype` holds for `rows`: their bits, or the reference's clamp and cast."""
    return rows.float().clamp(-448.0, 448.0).to(E4M3) if cache_dtype == E4M3 else rows


def reference_scatter(k_cache, v_cache, k, v, cu_seqlens, block_table=None, cache_seqlens=None):
    """The caches' bits after the reference's per-request loop (cache_manager.py:93-142): for each request, slice its
    rows in their stored form and index-assign them to positions cache_seqlens[b] + t: page block_table[b, p // page]
    slot p % page, or row p of cache entry b while p < S.  Runs on CPU copies; the stored form is taken on the device
    (an elementwise cast, the same for the whole source as for a slice)."""
    cu = cu_seqlens.tolist()
    B = len(cu) - 1
    start = cache_seqlens.tolist() if cache_seqlens is not None else [0] * B
    bt = None if block_table is None else block_table.cpu().long()
    out = []
    for cache, src in ((k_cache, k), (v_cache, v)):
        if cache is None:
            continue
        want, rows = _bits(cache).cpu(), _bits(stored(src, cache.dtype)).cpu()
        for b in range(B):
            n = cu[b + 1] - cu[b]
            if n == 0:
                continue
            pos, r = torch.arange(start[b], start[b] + n), rows[cu[b]:cu[b + 1]]
            if bt is not None:
                page = cache.shape[1]
                want[bt[b, pos // page], pos % page] = r
            else:
                keep = pos < cache.shape[1]
                want[b, pos[keep]] = r[keep]
        out.append(want)
    return out


def check_scatter(k_cache, v_cache, k, v, cu_seqlens, block_table=None, cache_seqlens=None):
    """One scatter call: one launch, and both caches equal the reference's bytes everywhere."""
    want = reference_scatter(k_cache, v_cache, k, v, cu_seqlens, block_table, cache_seqlens)
    before = _lib.launch_count()
    ops.scatter_kv_to_cache(k_cache, v_cache, k, v, cu_seqlens, block_table, cache_seqlens)
    assert _lib.launch_count() - before == 1
    torch.cuda.synchronize()
    got = [c for c in (k_cache, v_cache) if c is not None]
    for g, w in zip(got, want):
        assert torch.equal(_bits(g).cpu(), w)


def cu_of(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)


def paged_table(lens, starts, page, seed):
    """A block table over shuffled pages; every column a request does not need points at a trap page no request owns
    (the whole-cache comparison then sees a write through it).  Returns (block_table, num_blocks)."""
    need = (torch.tensor(starts) + torch.tensor(lens) + page - 1) // page
    num_blocks = int(need.sum()) + 2
    trap = num_blocks - 1
    perm = torch.randperm(num_blocks - 1, generator=torch.Generator().manual_seed(seed)).to(torch.int32)
    bt = torch.full((len(lens), int(need.max()) + 2), trap, dtype=torch.int32)
    used = torch.arange(bt.shape[1])[None, :] < need[:, None]
    bt[used] = perm[:int(need.sum())]
    return bt.to(DEV), num_blocks


def fused_qkv(total, Hq, Hkv, D, dtype, narrow, specials, seed):
    """k / v [total, Hkv, D] as views of one fused qkv output row [q | k | v] (plus one pad element when `narrow`, so
    rows are 2-byte aligned and the copy cannot use 16-byte accesses)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    width = (Hq + 2 * Hkv) * D + (1 if narrow else 0)
    qkv = torch.randn(total, width, generator=g, device=DEV).mul_(4.0).to(dtype)
    k = qkv[:, Hq * D:(Hq + Hkv) * D].unflatten(1, (Hkv, D))
    v = qkv[:, (Hq + Hkv) * D:(Hq + 2 * Hkv) * D].unflatten(1, (Hkv, D))
    if specials:
        sp = torch.tensor(SPECIALS, device=DEV).to(dtype)
        k[:, 0, :len(SPECIALS)] = sp
        v[:, -1, D - len(SPECIALS):] = sp.flip(0)
    return k, v


@pytest.mark.gpu
@pytest.mark.parametrize("page", [16, 64, 256])
@pytest.mark.parametrize("Hkv,D", [(1, 64), (2, 128), (8, 128), (8, 64)])
@pytest.mark.parametrize("src_dtype,cache_dtype", [(BF, BF), (F16, F16), (BF, E4M3), (F16, E4M3)])
def test_paged_gqa_scatter_matches_the_per_request_loop(src_dtype, cache_dtype, Hkv, D, page):
    bt, num_blocks = paged_table(LENS, STARTS, page, seed=page + Hkv)
    k, v = fused_qkv(sum(LENS), 2 * Hkv, Hkv, D, src_dtype, False, cache_dtype == E4M3, seed=D + Hkv)
    k_cache, v_cache = nan_tensor((num_blocks, page, Hkv, D), cache_dtype), nan_tensor((num_blocks, page, Hkv, D),
                                                                                         cache_dtype)
    starts = torch.tensor(STARTS, dtype=torch.int32, device=DEV)
    check_scatter(k_cache, v_cache, k, v, cu_of(LENS), bt, starts)


@pytest.mark.gpu
@pytest.mark.parametrize("page", [16, 256])
@pytest.mark.parametrize("dtype", [BF, F16])
def test_paged_gqa_scatter_narrow_copies_and_no_prefix(dtype, page):
    """Rows at odd element strides take the narrow copy; without cache_seqlens every request starts at position 0."""
    zero = [0] * len(LENS)
    bt, num_blocks = paged_table(LENS, zero, page, seed=7)
    k, v = fused_qkv(sum(LENS), 4, 2, 64, dtype, True, False, seed=8)
    assert k.stride(0) % 8 != 0
    k_cache, v_cache = nan_tensor((num_blocks, page, 2, 64), dtype), nan_tensor((num_blocks, page, 2, 64), dtype)
    check_scatter(k_cache, v_cache, k, v, cu_of(LENS), bt, None)


@pytest.mark.gpu
@pytest.mark.parametrize("cache_dtype", [BF, E4M3])
def test_mla_latent_scatter_matches_the_per_request_loop(cache_dtype):
    """DeepSeek's latent rows [total, 576] (a view of a wider projection output) into [num_blocks, 64, 576]."""
    bt, num_blocks = paged_table(LENS, STARTS, 64, seed=11)
    g = torch.Generator(device=DEV).manual_seed(12)
    wide = torch.randn(sum(LENS), 640, generator=g, device=DEV).mul_(8.0).to(BF)
    kv = wide[:, :576]
    if cache_dtype == E4M3:
        kv[:, 100:100 + len(SPECIALS)] = torch.tensor(SPECIALS, device=DEV).to(BF)
    kv_cache = nan_tensor((num_blocks, 64, 576), cache_dtype)
    check_scatter(kv_cache, None, kv, None, cu_of(LENS), bt, torch.tensor(STARTS, dtype=torch.int32, device=DEV))


@pytest.mark.gpu
@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("dtype", [BF, F16])
def test_nonpaged_scatter_matches_the_per_request_loop_and_stops_at_capacity(dtype, narrow):
    """[Bc, S, Hkv, D] caches as a [:, :S] view of a larger buffer (batch stride (S + 8) rows), Bc > B; the request
    that starts at 250 with 300 rows runs past S = 320, and its rows from position 320 on are not written."""
    B, S, Hkv, D = len(LENS), 320, 2, 128
    k, v = fused_qkv(sum(LENS), 8, Hkv, D, dtype, narrow, False, seed=13)
    k_cache = nan_tensor((B + 1, S + 8, Hkv, D), dtype)[:, :S]
    v_cache = nan_tensor((B + 1, S + 8, Hkv, D), dtype)[:, :S]
    check_scatter(k_cache, v_cache, k, v, cu_of(LENS), None, torch.tensor(STARTS, dtype=torch.int32, device=DEV))


@pytest.mark.gpu
def test_e4m3_store_bytes_follow_the_clamp_rule():
    """The stored bytes of the edge values, stated independently of torch's cast: saturation to +-448 (0x7E / 0xFE)
    from 449 up, NaN kept (0x7F / 0xFF), subnormals and ties rounded to nearest even."""
    want = [0x7E, 0xFE, 0x7E, 0xFE, 0x7E, 0xFE, 0x7F, 0x01, 0x81, 0x02, 0x00, 0x04, 0x00, 0x80, 0x7E, 0x7E, 0x77, 0x58,
            0x18, 0xB9]                                    # SPECIALS in order
    vals = torch.tensor(SPECIALS + [0.0] * (32 - len(SPECIALS)), device=DEV)
    for dtype in (BF, F16):
        src = vals.to(dtype).view(1, 32)
        cache = nan_tensor((1, 16, 32), E4M3)
        ops.scatter_kv_to_cache(cache, None, src, None, cu_of([1]), torch.zeros(1, 1, dtype=torch.int32, device=DEV),
                                torch.tensor([3], dtype=torch.int32, device=DEV))
        rows = _bits(cache)[0].cpu()
        assert rows[3, :len(want)].tolist() == want, (dtype, [hex(b) for b in rows[3].tolist()])
        assert (rows[3, len(want):] == 0).all()
        assert (rows[[0, 1, 2, 4, 15]] == 0xFF).all()


@pytest.mark.gpu
@pytest.mark.parametrize("cache_dtype", [BF, E4M3])
def test_scatter_more_than_65535_rows(cache_dtype):
    lens, starts = [70000, 0, 5], [100, 3, 0]
    bt, num_blocks = paged_table(lens, starts, 256, seed=21)
    k, v = fused_qkv(sum(lens), 2, 1, 64, BF, False, False, seed=22)
    k_cache, v_cache = nan_tensor((num_blocks, 256, 1, 64), cache_dtype), nan_tensor((num_blocks, 256, 1, 64),
                                                                                     cache_dtype)
    check_scatter(k_cache, v_cache, k, v, cu_of(lens), bt, torch.tensor(starts, dtype=torch.int32, device=DEV))


@pytest.mark.gpu
def test_scatter_more_than_65535_requests():
    B = 70001
    lens = [(b * 7) % 3 for b in range(B)]                 # 0, 1 and 2 rows
    starts = [(b * 5) % 16 for b in range(B)]
    bt, num_blocks = paged_table(lens, starts, 16, seed=23)
    k, v = fused_qkv(sum(lens), 1, 1, 64, F16, False, False, seed=24)
    k_cache, v_cache = nan_tensor((num_blocks, 16, 1, 64), F16), nan_tensor((num_blocks, 16, 1, 64), F16)
    check_scatter(k_cache, v_cache, k, v, cu_of(lens), bt, torch.tensor(starts, dtype=torch.int32, device=DEV))


@pytest.mark.gpu
@pytest.mark.parametrize("cache_dtype", [BF, E4M3])
def test_scatter_cuda_graph_replays_new_lengths_positions_and_contents(cache_dtype):
    """A graph captured once for total_rows rows replays with other lengths (an empty request included), other
    starting positions and new rows, and writes what an eager call writes."""
    lens_a, starts_a = [100, 200, 0, 60], [0, 30, 7, 250]
    lens_b, starts_b = [0, 1, 300, 59], [64, 255, 16, 0]
    assert sum(lens_a) == sum(lens_b)
    bt, num_blocks = paged_table(lens_a + lens_b, starts_a + starts_b, 256, seed=31)
    bt_a, bt_b = bt[:4].contiguous(), bt[4:].contiguous()
    k, v = fused_qkv(sum(lens_a), 8, 8, 128, BF, False, False, seed=32)
    k2, v2 = fused_qkv(sum(lens_a), 8, 8, 128, BF, False, False, seed=33)
    cu, starts, table = cu_of(lens_a), torch.tensor(starts_a, dtype=torch.int32, device=DEV), bt_a.clone()
    k_cache, v_cache = nan_tensor((num_blocks, 256, 8, 128), cache_dtype), nan_tensor((num_blocks, 256, 8, 128),
                                                                                      cache_dtype)
    blank_k, blank_v = k_cache.clone(), v_cache.clone()
    ops.scatter_kv_to_cache(k_cache, v_cache, k, v, cu, table, starts)          # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.scatter_kv_to_cache(k_cache, v_cache, k, v, cu, table, starts)
    k_cache.copy_(blank_k)
    v_cache.copy_(blank_v)
    cu.copy_(cu_of(lens_b))
    starts.copy_(torch.tensor(starts_b, dtype=torch.int32))
    table.copy_(bt_b)
    k.copy_(k2)
    v.copy_(v2)
    g.replay()
    torch.cuda.synchronize()
    replay_k, replay_v = k_cache.clone(), v_cache.clone()
    k_cache.copy_(blank_k)
    v_cache.copy_(blank_v)
    check_scatter(k_cache, v_cache, k, v, cu, table, starts)
    assert torch.equal(_bits(replay_k), _bits(k_cache)) and torch.equal(_bits(replay_v), _bits(v_cache))


# ------------------------------------------------------------------------- composition with the attention paths
def _randn(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def _filled_cache(shape, dtype, seed):
    """A cache of finite values (the prefix the prompt is written after)."""
    return _randn(shape, BF, seed, 2.0).to(dtype) if dtype == E4M3 else _randn(shape, dtype, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["paged", "paged_e4m3", "nonpaged"])
def test_gqa_prompt_written_by_the_scatter_decodes_like_the_multi_token_append(layout):
    """A prompt of sq rows per request on a cached prefix, written (a) by the scatter and (b) by attn_with_kvcache
    with seqlen_q = sq, then three decode steps through attn_with_kvcache on each: caches and outputs bit-identical."""
    from chitu_b200.attn_backend import B200AttnBackend
    be = B200AttnBackend()
    B, sq, Hq, Hkv, D, page = 3, 300, 8, 2, 128, 256
    starts = torch.tensor([0, 17, 261], dtype=torch.int32, device=DEV)
    cache_dtype = E4M3 if layout == "paged_e4m3" else BF
    if layout == "nonpaged":
        shape, bt = (B, 1024, Hkv, D), None
    else:
        bt, num_blocks = paged_table([sq + 3] * B, starts.tolist(), page, seed=41)
        shape = (num_blocks, page, Hkv, D)
    caches = [[_filled_cache(shape, cache_dtype, 42 + i) for i in range(2)]]
    caches.append([c.clone() for c in caches[0]])
    k, v = _randn((B * sq, Hkv, D), BF, 43), _randn((B * sq, Hkv, D), BF, 44)
    ops.scatter_kv_to_cache(*caches[0], k, v, cu_of([sq] * B), bt, starts)
    be.attn_with_kvcache(_randn((B, sq, Hq, D), BF, 45), *caches[1], k.view(B, sq, Hkv, D), v.view(B, sq, Hkv, D),
                         starts, block_table=bt, causal=True)
    torch.cuda.synchronize()
    for a, b in zip(*caches):
        assert torch.equal(_bits(a), _bits(b))
    for step in range(3):
        q1 = _randn((B, 1, Hq, D), BF, 50 + step)
        k1, v1 = _randn((B, 1, Hkv, D), BF, 60 + step), _randn((B, 1, Hkv, D), BF, 70 + step)
        lens = starts + sq + step
        outs = [be.attn_with_kvcache(q1, *c, k1, v1, lens, block_table=bt, causal=True) for c in caches]
        torch.cuda.synchronize()
        assert torch.equal(_bits(outs[0]), _bits(outs[1])), step
        assert torch.isfinite(outs[0].float()).all()
    for a, b in zip(*caches):
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.gpu
@pytest.mark.parametrize("cache_dtype", [BF, E4M3])
def test_mla_prompt_written_by_the_scatter_decodes_like_the_multi_token_append(cache_dtype):
    """The same for the latent cache: the scatter against mla_attn_with_kvcache with seqlen_q = sq, then three decode
    steps through mla_attn_with_kvcache."""
    from chitu_b200.attn_backend import B200AttnBackend
    be = B200AttnBackend(max_seq_len=1024, n_local_heads=16)
    B, sq, H, C, R = 3, 130, 16, 512, 64
    starts = torch.tensor([0, 17, 69], dtype=torch.int32, device=DEV)
    bt, num_blocks = paged_table([sq + 3] * B, starts.tolist(), 64, seed=81)
    caches = [_filled_cache((num_blocks, 64, C + R), cache_dtype, 82)]
    caches.append(caches[0].clone())
    kv = _randn((B * sq, C + R), BF, 83, 4.0)
    ops.scatter_kv_to_cache(caches[0], None, kv, None, cu_of([sq] * B), bt, starts)
    be.mla_attn_with_kvcache(_randn((B, sq, H, C), BF, 84), _randn((B, sq, H, R), BF, 85), caches[1],
                             kv.view(B, sq, C + R), starts, starts + sq, bt, causal=True)
    torch.cuda.synchronize()
    assert torch.equal(_bits(caches[0]), _bits(caches[1]))
    for step in range(3):
        qn, qp = _randn((B, H, C), BF, 90 + step), _randn((B, H, R), BF, 95 + step)
        kv1 = _randn((B, C + R), BF, 99 + step)
        excl = starts + sq + step
        outs = [be.mla_attn_with_kvcache(qn, qp, c, kv1, excl, excl + 1, bt) for c in caches]
        torch.cuda.synchronize()
        assert torch.equal(_bits(outs[0]), _bits(outs[1])), step
        assert torch.isfinite(outs[0].float()).all()
    assert torch.equal(_bits(caches[0]), _bits(caches[1]))
