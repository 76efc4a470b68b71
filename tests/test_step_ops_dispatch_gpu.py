"""The small kernels of a decode step against fp64 references or bit-exact restatements, through their C entries, on
every launch path the host code can pick: rotary (both layouts, the 16-byte and the scalar interleaved kernel), RMSNorm
(plain, strided and fused with the fp8 quantiser), SiLU * mul (plain and fused with the quantiser), the fp8 group and
int8 per-token quantisers, fp8 weight dequant (normal and soft), embedding, add, argmax, `mla_prep`,
`mla_absorb_o_quant` and top-k / top-p sampling.

Every output lives in a buffer with sentinel bytes before and after it (and in the gaps between rows when the row stride
is larger than the row); every input is NaN-poisoned where the kernel must not read: rows past the batch, columns between
the row and its stride, the W_UV half of `wkv_b` for the absorb-q role and the W_UK half for absorb-o.

Bounds.  u = 2^-24 is the fp32 unit roundoff and u_out the output's (bf16 2^-8, fp16 2^-11, fp32 2^-24); eta is half the
smallest fp16 subnormal (2^-25) for fp16 outputs and 0 otherwise.  The fp32 error of `rsqrtf` (2 ulp) and `expf` (2 ulp)
is from the single-precision table of the CUDA C++ Programming Guide (Mathematical Functions appendix), that of `__expf`
(2 + floor(|1.173 x|) ulp) from its intrinsic-functions table; an ulp is at most 2^-23 of the value.  Each bound is
    |y - ref| <= u_out |ref| + (1 + u_out) * ACC + eta
with ACC the fp32 error before the output rounding:
  - rotary (interleaved; the k_pe / q_pe part of `mla_prep`): ACC = 2^-23 (|x0 c| + |x1 s|) — one rounded product and
    one rounded fma (or two products and a sum) per output.
  - RMSNorm (and the kv_norm of `mla_prep`, and the y of `rmsnorm_quant_fp8`): ACC = ((n + 3) / 2 + 7) u |ref|.  The sum
    of squares is n levels of positive fp32 additions (n = per-thread terms + 5 butterfly levels + 8 warp partials:
    ceil(dim / 256) + 13 for the plain kernel, 4 ceil(dim / 1024) + 13 for the fused one), plus the square, the division
    by dim and the + eps: (n + 3) u relative on the argument of rsqrtf, half of it on the result; rsqrtf adds 4 u, the
    two products 2 u, and one u covers the second-order terms.
  - SiLU * mul: ACC = ((1 + u_out) (u_out + 6 u) + u) |ref| + eta |x_up|: expf (4 u) and the sum (u) in the
    denominator, the division (u), the rounding of silu to the io dtype (u_out, plus eta when it lands on an fp16
    subnormal), the product (u).
  - absorb-q (`mla_prep`): ACC = (dn / 8 + 9) u sum_d |q_d W_dc|: each warp runs a chain of dn / 8 fmas, the 8 partials
    are summed in sequence.
  - absorb-o (`mla_absorb_o_quant`): ACC = (8 ceil(C / 256) + 6) u sum_c |x_c W_dc|: each lane runs a chain of
    8 ceil(C / 256) fmas, then 5 butterfly levels.
Bit-exact checks (one IEEE operation or one rounding): `rotary_half` against `O.rotary_half` on the CPU, the fp8 and
int8 quantisers, weight dequant, embedding, add (an fp32 add rounded once), argmax (the first maximal index), the fp8
payload and scales of the fused quantisers against `O.act_quant_deepseek_v3` of the kernel's own bf16 values, and the
16-byte rotary kernel against the scalar one.  `test_bound_rejects_injected_errors` shows, on the host, that these
bounds admit the correctly rounded fp64 result and reject eps dropped, the mean over dim - 1 (fp32 output), a sin sign
flipped, cos and sin swapped on one pair, one absorb-q warp partial dropped, a W_UV row off by one and the kv_norm
weight shifted by one element.

Sampling.  The rule is restated in fp64: p = softmax(logit * fl32(1 / T)); entry i is kept when the fp64 mass of the
strictly larger entries is <= top_p, fewer than top_k entries are strictly larger, and p_i > 0.  The kernel's p_i carries
a relative error rho_i = u (|l_i / T| + |max| + |d_i|) + (2 + 1.173 |d_i|) 2^-23 (d_i = the exponent argument:
its two roundings and __expf) plus (V / 1024 + 40) u + max_j rho_j from the fp32 sum and the reciprocal.  Two entries
within 2 rho of each other may swap order (or tie), entries whose exclusive mass is within
delta = (V + 6144) u + 2 rho of top_p may fall either way (the threshold walk adds up to V atomics and 3 x 2048 bins in
fp32), and an entry whose fp64 p is below 2^-100 may come out 0 (__expf flushes below 2^-126).  The kept count and mass
must lie between those of the sure and the possible sets.  The drawn token must be possibly kept, and its vocabulary-order
CDF interval must come within delta_d = (V / 1024 + 1024 + 64) u + 2 rho (of the kept mass) of u * z: the per-thread
sums, the 1024-term scan and the block reduction."""
import math

import pytest
import torch

from oracle import chitu_oracle as O

BF, F16, F32, F8 = torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn
DEV = "cuda:0"
U = 2.0 ** -24
U_OUT = {BF: 2.0 ** -8, F16: 2.0 ** -11, F32: 2.0 ** -24}
ETA = {BF: 0.0, F16: 2.0 ** -25, F32: 0.0}
EPS = 1e-6


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------- references and bounds
def bound(ref, acc, dtype):
    return U_OUT[dtype] * ref.abs() + (1 + U_OUT[dtype]) * acc + ETA[dtype]


def ratio(y, ref, bnd):
    """max over elements of |y - ref| / bound; inf when y is not finite or differs where the bound is 0."""
    y = y.to(ref.device).double()
    if not bool(torch.isfinite(y).all()):
        return math.inf
    err = (y - ref).abs()
    r = torch.where(bnd > 0, err / bnd.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def rms_ref(x, w, eps, n_acc, mean_div=None):
    """fp64 RMSNorm of rows x [.., dim] with weight w; returns (ref, ACC)."""
    dim = x.shape[-1]
    ms = (x * x).sum(-1, keepdim=True) / (mean_div or dim)
    ref = x / torch.sqrt(ms + eps) * w
    return ref, ((n_acc + 3) / 2 + 7) * U * ref.abs()


def rms_terms(dim, fused=False):
    return (4 * _cdiv(dim, 1024) if fused else _cdiv(dim, 256)) + 13


def rotary_ref(x, c, s):
    """interleaved pairs of x [.., rot] (fp64) rotated by c / s [.., rot / 2]; returns (ref, ACC)."""
    x0, x1 = x[..., 0::2], x[..., 1::2]
    ref = torch.stack([x0 * c - x1 * s, x1 * c + x0 * s], -1).flatten(-2)
    acc = torch.stack([(x0 * c).abs() + (x1 * s).abs(), (x1 * c).abs() + (x0 * s).abs()], -1).flatten(-2)
    return ref, 2.0 ** -23 * acc


def absorb_q_ref(q_nope, w_uk):
    """q_nope [B, H, dn], W_UK [H, dn, C] (fp64) -> (q_abs [B, H, C], ACC)."""
    dn = q_nope.shape[-1]
    ref = torch.einsum("bhd,hdc->bhc", q_nope, w_uk)
    return ref, (dn // 8 + 9) * U * torch.einsum("bhd,hdc->bhc", q_nope.abs(), w_uk.abs())


def absorb_o_ref(x, w_uv):
    """x [B, H, C], W_UV [H, dv, C] (fp64) -> (out [B, H, dv], ACC)."""
    C = x.shape[-1]
    ref = torch.einsum("bhc,hdc->bhd", x, w_uv)
    return ref, (8 * _cdiv(C, 256) + 6) * U * torch.einsum("bhc,hdc->bhd", x.abs(), w_uv.abs())


def silu_mul_ref(g, u_, dtype):
    ref = g / (1 + torch.exp(-g)) * u_
    return ref, ((1 + U_OUT[dtype]) * (U_OUT[dtype] + 6 * U) + U) * ref.abs() + ETA[dtype] * u_.abs()


# ------------------------------------------------------------------------- injected-error self-test of the bounds
def test_bound_rejects_injected_errors():
    """The bounds admit the correctly rounded fp64 result and reject each injected error."""
    g = torch.Generator().manual_seed(0)
    names = set()

    def check(name, good, wrong, ref, bnd):
        assert ratio(good, ref, bnd) <= 1.0, name
        assert ratio(wrong, ref, bnd) > 1.0, name
        names.add(name)

    for dim in (64, 100, 512, 1536, 4096, 7168, 8192):
        for fused in (False, True):
            x = torch.randn(4, dim, generator=g, dtype=torch.float64) * 1e-3      # mean(x^2) ~ eps: eps matters
            x[1] *= 1000
            w = torch.rand(dim, generator=g, dtype=torch.float64) + 0.5
            ref, acc = rms_ref(x, w, EPS, rms_terms(dim, fused))
            bnd = bound(ref, acc, F32)
            good = ref.float()
            check("eps dropped", good, (x / torch.sqrt((x * x).mean(-1, keepdim=True)) * w).float(), ref, bnd)
            wrong, _ = rms_ref(x, w, EPS, 0, mean_div=dim - 1)
            check("mean over dim - 1", good, wrong.float(), ref, bnd)
            assert ratio(ref.to(BF), ref, bound(ref, acc, BF)) <= 1.0
    # rotary: bf16 data, fp32 cos / sin of random angles
    for rot in (64, 128):
        x = torch.randn(8, 4, rot, generator=g).to(BF).double()
        ang = torch.rand(8, 1, rot // 2, generator=g, dtype=torch.float64) * 100
        c, s = torch.cos(ang).float().double(), torch.sin(ang).float().double()
        ref, acc = rotary_ref(x, c, s)
        bnd = bound(ref, acc, BF)
        s2 = s.clone()
        s2[3, 0, 5] = -s2[3, 0, 5]
        check("sin sign flipped", ref.to(BF), rotary_ref(x, c, s2)[0].to(BF), ref, bnd)
        c2, s2 = c.clone(), s.clone()
        c2[5, 0, 7], s2[5, 0, 7] = s[5, 0, 7], c[5, 0, 7]
        check("cos and sin swapped on one pair", ref.to(BF), rotary_ref(x, c2, s2)[0].to(BF), ref, bnd)
    # absorb-q: one of the 8 warp partials dropped
    B, H, dn, dv, C = 3, 2, 128, 128, 512
    q = torch.randn(B, H, dn, generator=g).to(BF).double()
    wkv = (torch.randn(H, dn + dv, C, generator=g) * 0.05).to(BF).double()
    ref, acc = absorb_q_ref(q, wkv[:, :dn])
    part = torch.einsum("bhd,hdc->bhc", q[..., 48:64], wkv[:, 48:64])               # warp 3's 16 rows
    check("absorb-q warp partial dropped", ref.to(BF), (ref - part).to(BF), ref, bound(ref, acc, BF))
    # absorb-o: a W_UV row off by one
    x = torch.randn(B, H, C, generator=g).to(BF).double()
    ref, acc = absorb_o_ref(x, wkv[:, dn:])
    wrong, _ = absorb_o_ref(x, torch.roll(wkv[:, dn:], -1, dims=1))
    check("W_UV row off by one", ref.to(BF), wrong.to(BF), ref, bound(ref, acc, BF))
    # kv_norm weight shifted by one element
    kv = torch.randn(B, C, generator=g).to(BF).double()
    w = (torch.rand(C, generator=g) + 0.5).to(BF).double()
    ref, acc = rms_ref(kv, w, EPS, rms_terms(C))
    wrong, _ = rms_ref(kv, torch.roll(w, 1), EPS, rms_terms(C))
    check("kv_norm weight shifted", ref.to(BF), wrong.to(BF), ref, bound(ref, acc, BF))
    assert names == {"eps dropped", "mean over dim - 1", "sin sign flipped", "cos and sin swapped on one pair",
                     "absorb-q warp partial dropped", "W_UV row off by one", "kv_norm weight shifted"}


# ------------------------------------------------------------------------------------------------ refusals (host)
def _L():
    from chitu_b200 import _lib as L
    return L


def _lib():
    return _L().load()


def _last_error():
    return _lib().chitu_b200_last_error().decode(errors="replace")


def test_step_entries_refuse_what_the_kernels_cannot_load():
    """Operands that the kernels read or write with 4-, 8- or 16-byte vector accesses are refused, before anything is
    launched, when their base is not aligned to that width."""
    L, lib = _L(), _lib()
    A = 4096

    def rmsq(x=A, w=A, y=A, q=A):
        return lib.chitu_b200_rmsnorm_quant_fp8(x, w, y, q, A, 4, 1536, 2112, 1536, 1e-6, None)

    def silq(x=A, q=A):
        return lib.chitu_b200_silu_mul_quant_fp8(x, q, A, 4, 256, None)

    def emb(table=A, out=A):
        return lib.chitu_b200_embedding(A, table, out, 4, 64, 0, 100, L.CB_BF16, None)

    def abso(x=A, w=A, out=A, q=A):
        return lib.chitu_b200_mla_absorb_o_quant(x, w, out, q, A, 3, 16, 128, 128, 512, None)

    def merge(ws=A, w=A, x_out=A, out=A, q=A):
        return lib.chitu_b200_mla_absorb_o_merge_quant(ws, 1 << 30, 4096, w, x_out, out, q, A, 3, 16, 128, 128, 512,
                                                       None)

    def prep(w=A):
        return lib.chitu_b200_mla_prep(A, A, 2112, A, A, A, w, A, A, A, 3, 16, 128, 128, 512, 64, 1e-6, None)

    bad = [(rmsq, "rmsnorm_quant_fp8", dict(x=A + 4)), (rmsq, "rmsnorm_quant_fp8", dict(w=A + 4)),
           (rmsq, "rmsnorm_quant_fp8", dict(y=A + 4)), (rmsq, "rmsnorm_quant_fp8", dict(q=A + 2)),
           (silq, "silu_mul_quant_fp8", dict(x=A + 4)), (silq, "silu_mul_quant_fp8", dict(q=A + 2)),
           (emb, "embedding", dict(table=A + 8)), (emb, "embedding", dict(out=A + 8)),
           (abso, "mla_absorb_o_quant", dict(x=A + 8)), (abso, "mla_absorb_o_quant", dict(w=A + 8)),
           (abso, "mla_absorb_o_quant", dict(out=A + 4)), (abso, "mla_absorb_o_quant", dict(q=A + 2)),
           (merge, "mla_absorb_o_merge_quant", dict(ws=A + 8)), (merge, "mla_absorb_o_merge_quant", dict(w=A + 8)),
           (merge, "mla_absorb_o_merge_quant", dict(x_out=A + 4)), (merge, "mla_absorb_o_merge_quant", dict(out=A + 4)),
           (merge, "mla_absorb_o_merge_quant", dict(q=A + 2)), (prep, "mla_prep", dict(w=A + 2))]
    before = L.launch_count()
    for fn, entry, kw in bad:
        assert fn(**kw) < 0, (entry, kw)
        assert entry in _last_error(), (entry, kw, _last_error())
    assert L.launch_count() == before


# ---------------------------------------------------------------------------------------------------- GPU calls
PAD = 256          # bytes of pad before and after every operand view (keeps the views 16-byte aligned)
NAN_BYTE = 0xFF    # NaN in bf16, fp16, fp8 e4m3 and fp32
SENTINEL = 0xA5


class Padded:
    """A contiguous view in the middle of a larger byte buffer; the pads hold `pad` bytes."""

    def __init__(self, t=None, pad=NAN_BYTE, fill=None, shape=None, dtype=None):
        shape, dtype = (t.shape, t.dtype) if t is not None else (shape, dtype)
        nbytes = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        self.buf = torch.full((2 * PAD + nbytes,), pad, dtype=torch.uint8, device=DEV)
        self.pad, self.nbytes = pad, nbytes
        self.bytes = self.buf[PAD:PAD + nbytes]
        self.view = self.bytes.view(dtype).view(shape)
        if t is not None:
            self.view.copy_(t)
        elif fill is not None:
            self.bytes.fill_(fill)

    def pads_intact(self):
        return bool((self.buf[:PAD] == self.pad).all()) and bool((self.buf[PAD + self.nbytes:] == self.pad).all())


def out_buf(shape, dtype):
    return Padded(pad=SENTINEL, fill=SENTINEL, shape=shape, dtype=dtype)


def gaps_intact(P, row):
    """the bytes past `row` elements of every row of P.view [rows, stride] still hold the sentinel"""
    es = P.view.element_size()
    return bool((P.bytes.view(P.view.shape[0], -1)[:, row * es:] == SENTINEL).all())


def nan_full(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def ptr(t):
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def ok(rc, what):
    assert rc == 0, (what, rc, _last_error())


def bits(t):
    return t.contiguous().view(torch.uint8)


def dcode(dtype):
    return _L().dtype_code(dtype)


def rand(shape, g, dtype, scale=1.0):
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _dn(dtype):
    return {BF: "bf16", F16: "fp16", F32: "fp32"}[dtype]


def assert_bound(y, ref, acc, dtype, what):
    r = ratio(y, ref, bound(ref, acc, dtype))
    assert r <= 1.0, (what, r)


# ------------------------------------------------------------------------------------------------ rotary (interleaved)
ROT_VIEWS = ("dense", "q_pe", "odd_sh", "cos_off4", "hq0", "hk0")
ROT_CASES = [(v, d, bs) for v in ROT_VIEWS for d in (BF, F16, F32) for bs in (1, 16, 256)]


def _rot_geometry(view):
    """(hq, hk, rot, head width of q, q head stride, k head stride, offset of the rotated part in a head,
    k row width, cos offset in floats)"""
    if view == "q_pe":                # DeepSeek: q_pe = the last 64 of a 192-wide head, k_pe = the last 64 of a 576 row
        return dict(hq=16, hk=1, rot=64, q_sh=192, q_off=128, k_sh=64, k_sb=576, k_off=512, cos_off=0)
    if view == "odd_sh":              # head strides that are not multiples of 8 elements
        return dict(hq=4, hk=2, rot=64, q_sh=68, q_off=2, k_sh=76, k_sb=152, k_off=6, cos_off=0)
    hq, hk = {"hq0": (0, 2), "hk0": (8, 0)}.get(view, (8, 2))
    return dict(hq=hq, hk=hk, rot=128, q_sh=128, q_off=0, k_sh=128, k_sb=hk * 128, k_off=0,
                cos_off=1 if view == "cos_off4" else 0)


def _rot_vec(dtype, geo, q_ptr, k_ptr, cos_ptr):
    """the host condition of chitu_b200_rotary_interleaved that picks the 16-byte kernel"""
    q_sb = geo["hq"] * geo["q_sh"]
    strides = (q_sb, geo["q_sh"], geo["k_sb"], geo["k_sh"], geo["hq"] * geo["rot"], geo["hk"] * geo["rot"])
    return (dtype in (BF, F16) and geo["rot"] % 8 == 0 and all(s % 8 == 0 for s in strides)
            and all(p % 16 == 0 for p in (q_ptr, k_ptr, cos_ptr)))


def _run_rotary(dtype, bs, geo, q_in, k_in, cos, sin):
    hq, hk, rot = geo["hq"], geo["hk"], geo["rot"]
    oq, ok_ = out_buf((bs, hq, rot), dtype), out_buf((bs, hk, rot), dtype)
    vptr = lambda P: P.buf.data_ptr() + PAD                        # an empty view (hq or hk 0) has no data_ptr
    q_ptr = q_in.data_ptr() + geo["q_off"] * q_in.element_size()
    k_ptr = k_in.data_ptr() + geo["k_off"] * k_in.element_size()
    ok(_lib().chitu_b200_rotary_interleaved(q_ptr, k_ptr, vptr(oq), vptr(ok_), cos, sin, bs, hq, hk, rot,
                                            hq * geo["q_sh"], geo["q_sh"], geo["k_sb"], geo["k_sh"], dcode(dtype),
                                            stream()), "rotary_interleaved")
    return oq, ok_, _rot_vec(dtype, geo, q_ptr, k_ptr, cos)


@pytest.mark.gpu
@pytest.mark.parametrize("view,dtype,bs", ROT_CASES, ids=[f"rotary_interleaved-{v}-{_dn(d)}-bs{b}" for v, d, b in ROT_CASES])
def test_rotary_interleaved(view, dtype, bs):
    g = _gen(bs * 7 + ROT_VIEWS.index(view))
    geo = _rot_geometry(view)
    hq, hk, rot = geo["hq"], geo["hk"], geo["rot"]
    half = rot // 2
    # inputs: q rows of hq heads of q_sh elements, the rotated part at q_off; NaN everywhere else and on row bs
    qb = nan_full((bs + 1, max(hq, 1) * geo["q_sh"]), dtype)
    kb = nan_full((bs + 1, geo["k_sb"] if hk else 8), dtype)
    q = rand((bs, hq, rot), g, dtype)
    k = rand((bs, hk, rot), g, dtype)
    for h in range(hq):
        qb[:bs, h * geo["q_sh"] + geo["q_off"]:h * geo["q_sh"] + geo["q_off"] + rot] = q[:, h]
    for h in range(hk):
        kb[:bs, h * geo["k_sh"] + geo["k_off"]:h * geo["k_sh"] + geo["k_off"] + rot] = k[:, h]
    ang = torch.rand(bs, half, generator=g, device=DEV, dtype=torch.float64) * 1000
    cs = torch.cat([torch.cos(ang), torch.sin(ang)], 1).float()
    cb = nan_full((2, (bs + 1) * half + 4), F32)                    # one float past 16-byte alignment for "cos_off4"
    off = geo["cos_off"]
    cb[0, off:off + bs * half] = cs[:, :half].flatten()
    cb[1, :bs * half] = cs[:, half:].flatten()
    Q, K = Padded(qb), Padded(kb)
    oq, ok_, vec = _run_rotary(dtype, bs, geo, Q.view, K.view, cb[0, off:].data_ptr(), cb[1].data_ptr())
    torch.cuda.synchronize()
    assert vec == (dtype != F32 and view in ("dense", "q_pe", "hq0", "hk0")), (view, vec)
    c, s = cs[:, None, :half].double(), cs[:, None, half:].double()
    for x, o, name in ((q, oq, "q"), (k, ok_, "k")):
        ref, acc = rotary_ref(x.double(), c, s)
        assert_bound(o.view, ref, acc, dtype, (view, name))
        assert o.pads_intact(), (view, name)
    if view == "cos_off4" and dtype != F32:
        # the 16-byte kernel on the same values (cos aligned) gives the same bytes as the scalar kernel
        ca = cs[:, :half].contiguous()
        oq2, ok2, vec2 = _run_rotary(dtype, bs, geo, Q.view, K.view, ca.data_ptr(), cb[1].data_ptr())
        torch.cuda.synchronize()
        assert vec2 and not vec
        assert torch.equal(bits(oq2.view), bits(oq.view)) and torch.equal(bits(ok2.view), bits(ok_.view))


# ------------------------------------------------------------------------------------------------- rotary (halves)
ROTH_CASES = [(d, heads, D, strided) for d in (BF, F16, F32) for heads, D, strided in
              ((1, 128, False), (8, 64, False), (48, 128, False), (32, 128, True), (48, 128, True))]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,heads,D,strided", ROTH_CASES,
                         ids=[f"rotary_half{'_strided' if s else ''}-{_dn(d)}-h{h}-d{D}" for d, h, D, s in ROTH_CASES])
def test_rotary_half(dtype, heads, D, strided):
    """bit exact against O.rotary_half; the strided case is Mixtral's qkv view (q heads, then 2 x Hkv heads of k / v)"""
    g = _gen(heads * 3 + D)
    bs, hkv = 37, 8
    x_sb = (heads + 2 * hkv) * D if strided else heads * D
    xb = nan_full((bs + 1, x_sb), dtype)
    x = rand((bs, heads, D), g, dtype)
    xb[:bs, :heads * D] = x.flatten(1)
    ang = torch.rand(bs, D // 2, generator=g, device=DEV) * 100
    cos, sin = Padded(torch.cos(ang).to(dtype)), Padded(torch.sin(ang).to(dtype))
    X = Padded(xb)
    out = out_buf((bs, heads, D), dtype)
    lib = _lib()
    if strided:
        ok(lib.chitu_b200_rotary_half_strided(ptr(X.view), x_sb, ptr(out.view), ptr(cos.view), ptr(sin.view), bs, heads,
                                              D, dcode(dtype), stream()), "rotary_half_strided")
    else:
        ok(lib.chitu_b200_rotary_half(ptr(X.view), ptr(out.view), ptr(cos.view), ptr(sin.view), bs, heads, D,
                                      dcode(dtype), stream()), "rotary_half")
    ref, _ = O.rotary_half(x.cpu(), x.cpu(), cos.view.cpu(), sin.view.cpu())
    assert torch.equal(bits(out.view.cpu()), bits(ref))
    assert out.pads_intact()


# ---------------------------------------------------------------------------------------------------------- RMSNorm
RMS_DIMS = (64, 100, 512, 1536, 4096, 7168, 8192)
RMS_CASES = [(d, dim, rows, xs, ys) for d in (BF, F16, F32) for dim in RMS_DIMS
             for rows, xs, ys in ((1, 0, 0), (37, 3, 5), (256, 64, 0))]


def _rows_in(rows, dim, stride, dtype, g, scales=(1e-3, 1.0, 30.0)):
    """x [rows, dim] with rows of three magnitudes (the smallest makes eps matter) in a NaN-poisoned [rows + 1, stride]
    buffer"""
    x = rand((rows, dim), g, dtype) * torch.tensor(scales, device=DEV).repeat(_cdiv(rows, 3))[:rows, None].to(dtype)
    xb = nan_full((rows + 1, stride), dtype)
    xb[:rows, :dim] = x
    return x, Padded(xb)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,dim,rows,xs,ys", RMS_CASES,
                         ids=[f"rmsnorm{'_strided' if xs or ys else ''}-{_dn(d)}-dim{dim}-rows{r}-xs+{xs}-ys+{ys}"
                              for d, dim, r, xs, ys in RMS_CASES])
def test_rmsnorm(dtype, dim, rows, xs, ys):
    g = _gen(dim + rows)
    x, X = _rows_in(rows, dim, dim + xs, dtype, g)
    w = Padded((torch.rand(dim, generator=g, device=DEV) + 0.5).to(dtype))
    Y = out_buf((rows, dim + ys), dtype)
    lib = _lib()
    if xs or ys:
        ok(lib.chitu_b200_rmsnorm_strided(ptr(X.view), ptr(w.view), ptr(Y.view), rows, dim, dim + xs, dim + ys, EPS,
                                          dcode(dtype), stream()), "rmsnorm_strided")
    else:
        ok(lib.chitu_b200_rmsnorm(ptr(X.view), ptr(w.view), ptr(Y.view), rows, dim, EPS, dcode(dtype), stream()),
           "rmsnorm")
    ref, acc = rms_ref(x.double(), w.view.double(), EPS, rms_terms(dim))
    assert_bound(Y.view[:, :dim], ref, acc, dtype, "y")
    assert Y.pads_intact() and gaps_intact(Y, dim)


RMSQ_CASES = [(dim, rows, dim, dim + 64) for dim in (128, 1536, 2176, 3200, 4224, 5248, 7168, 8192) for rows in (1, 256)]
RMSQ_CASES += [(1536, 33, 2112, 1536), (512, 17, 2112, 516)]       # the engine's q_a / kv views of the wqkv_a output


@pytest.mark.gpu
@pytest.mark.parametrize("dim,rows,xs,ys", RMSQ_CASES,
                         ids=[f"rmsnorm_quant_fp8-bf16-dim{d}-nit{_cdiv(d, 1024)}-rows{r}-xs{x}-ys{y}"
                              for d, r, x, y in RMSQ_CASES])
def test_rmsnorm_quant_fp8(dim, rows, xs, ys):
    """y only, q only and both: y within the RMSNorm bound, q / scales bit exact against act_quant of the kernel's own y,
    and the q-only run writes the same bytes as the run that writes both"""
    g = _gen(dim * 3 + rows)
    x, X = _rows_in(rows, dim, xs, BF, g)
    w = Padded((torch.rand(dim, generator=g, device=DEV) + 0.5).to(BF))
    lib = _lib()
    res = {}
    for mode in ("y", "q", "both"):
        Y = out_buf((rows, ys), BF) if mode != "q" else None
        Q = out_buf((rows, dim), torch.uint8) if mode != "y" else None
        S = out_buf((rows, dim // 128), F32) if mode != "y" else None
        ok(lib.chitu_b200_rmsnorm_quant_fp8(ptr(X.view), ptr(w.view), Y and ptr(Y.view), Q and ptr(Q.view),
                                            S and ptr(S.view), rows, dim, xs, ys, EPS, stream()), "rmsnorm_quant_fp8")
        for P in (Y, Q, S):
            assert P is None or P.pads_intact(), mode
        if Y is not None:
            assert gaps_intact(Y, dim), mode
        res[mode] = (Y, Q, S)
    ref, acc = rms_ref(x.double(), w.view.double(), EPS, rms_terms(dim, fused=True))
    for mode in ("y", "both"):
        assert_bound(res[mode][0].view[:, :dim], ref, acc, BF, mode)
    y = res["both"][0].view[:, :dim].cpu()
    assert torch.equal(bits(y), bits(res["y"][0].view[:, :dim].cpu()))
    qo, so = O.act_quant_deepseek_v3(y)
    assert torch.equal(res["both"][2].view.cpu(), so)
    assert torch.equal(res["both"][1].view.cpu(), bits(qo).view(rows, dim))
    assert torch.equal(res["q"][1].view, res["both"][1].view) and torch.equal(res["q"][2].view, res["both"][2].view)


# ------------------------------------------------------------------------------------------------------ SiLU * mul
SILU_CASES = [(d, rows, n) for d in (BF, F16, F32) for rows, n in ((1, 128), (5, 1001), (300, 1001), (64, 18432))]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,rows,d", SILU_CASES,
                         ids=[f"silu_and_mul-{_dn(t)}-rows{r}-d{d}{'-gridloop' if r * d > 132 * 8 * 256 else ''}"
                              for t, r, d in SILU_CASES])
def test_silu_and_mul(dtype, rows, d):
    g = _gen(rows + d)
    x = rand((rows, 2 * d), g, dtype, 2.0)
    xb = nan_full((rows + 1, 2 * d), dtype)
    xb[:rows] = x
    X, Y = Padded(xb), out_buf((rows, d), dtype)
    ok(_lib().chitu_b200_silu_and_mul(ptr(X.view), ptr(Y.view), rows, d, dcode(dtype), stream()), "silu_and_mul")
    xd = x.double()
    ref, acc = silu_mul_ref(xd[:, :d], xd[:, d:], dtype)
    assert_bound(Y.view, ref, acc, dtype, "out")
    assert Y.pads_intact()


SILQ_CASES = [(1, 128), (256, 128), (3, 18432), (64, 18432)]


@pytest.mark.gpu
@pytest.mark.parametrize("rows,F", SILQ_CASES, ids=[f"silu_mul_quant_fp8-bf16-rows{r}-F{f}" for r, f in SILQ_CASES])
def test_silu_mul_quant_fp8(rows, F):
    g = _gen(rows * 5 + F)
    x = rand((rows, 2 * F), g, BF, 2.0)
    xb = nan_full((rows + 1, 2 * F), BF)
    xb[:rows] = x
    X, Q, S = Padded(xb), out_buf((rows, F), torch.uint8), out_buf((rows, F // 128), F32)
    ok(_lib().chitu_b200_silu_mul_quant_fp8(ptr(X.view), ptr(Q.view), ptr(S.view), rows, F, stream()),
       "silu_mul_quant_fp8")
    qo, so = O.act_quant_deepseek_v3(O.silu_and_mul(x.cpu()))
    assert torch.equal(S.view.cpu(), so) and torch.equal(Q.view.cpu(), bits(qo).view(rows, F))
    assert Q.pads_intact() and S.pads_intact()


# ------------------------------------------------------------------------------------------------ fp8 group quantiser
AQ_CASES = [(d, gs, mode) for d in (BF, F16, F32) for gs in (128, 64, 32) for mode in (0, 1)]


def _saturating_amax(dtype, g):
    """a value v of the dtype for which fl32(v / fl32(v / 448)) > 448: its group's largest element quantises above 448"""
    for _ in range(100):
        v = (torch.rand(4096, generator=g, device=DEV) * 1000 + 1).to(dtype).float().cpu()
        hit = (v / (v / torch.tensor(448.0))) > 448.0                    # IEEE fp32 divisions, as the kernel's
        if bool(hit.any()):
            return float(v[hit][0])
    raise AssertionError("no saturating value found")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,group,mode", AQ_CASES,
                         ids=[f"act_quant_fp8-mode{m}-{_dn(d)}-g{gs}" for d, gs, m in AQ_CASES])
def test_act_quant_fp8(dtype, group, mode):
    """bit exact against act_quant_deepseek_v3 (mode 0) / per_token_group_quant_fp8 (mode 1); an all-zero group gives
    scale 0 and a NaN payload in mode 0 (as the reference) and takes the eps path in mode 1"""
    g = _gen(group + mode + dtype.itemsize)
    rows, K = 7, 512
    x = rand((rows, K), g, dtype, 3.0)
    x[0, :group] *= 40
    amax = _saturating_amax(dtype, g)
    x[0, group:2 * group] = (x[0, group:2 * group].float().clamp(-0.9, 0.9) * amax).to(dtype)
    x[0, group + 3] = amax
    x[1, group:2 * group] = 0
    x[2, 2 * group:3 * group] = rand((group,), g, dtype, 1e-6 if dtype != F16 else 1e-4)
    X = Padded(x)
    Y, S = out_buf((rows, K), torch.uint8), out_buf((rows, K // group), F32)
    ok(_lib().chitu_b200_act_quant_fp8(ptr(X.view), ptr(Y.view), ptr(S.view), rows, K, group, mode, 1e-10, dcode(dtype),
                                       stream()), "act_quant_fp8")
    xc = x.cpu()
    yo, so = O.act_quant_deepseek_v3(xc, group) if mode == 0 else O.per_token_group_quant_fp8(xc, group, 1e-10)
    assert torch.equal(S.view.cpu(), so)
    y = Y.view.cpu().view(F8)
    nan_ref = torch.isnan(yo.float())
    assert torch.equal(torch.isnan(y.float()), nan_ref)
    assert bool(nan_ref.any()) == (mode == 0)
    assert torch.equal(bits(y)[~nan_ref], bits(yo)[~nan_ref])
    assert bool((xc[0, group:2 * group].float() / so[0, 1] > 448).any())      # the planted group saturates
    assert Y.pads_intact() and S.pads_intact()


# ------------------------------------------------------------------------------------------------ int8 quantiser
QI_CASES = [(d, K) for d in (BF, F16, F32) for K in (256, 1024, 1000, 4104)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,K", QI_CASES, ids=[f"quant_act_int8-{_dn(d)}-K{k}" for d, k in QI_CASES])
def test_quant_act_int8(dtype, K):
    """bit exact against quant_act (quantize/w8a8.py:18-26): scale = clamp(max|x| as fp32, 1e-5) / 127,
    q = round-half-even(x / scale) (torch promotes the division to fp32)"""
    g = _gen(K + dtype.itemsize)
    rows = 5
    x = rand((rows, K), g, dtype, 2.0)
    halves = (torch.arange(K, device=DEV) % 253 - 126).float() + 0.5                 # x / 1.0 = k + 0.5
    x[0] = halves.to(dtype)
    x[0, 7] = 127.0                                                                  # max 127: scale exactly 1
    x[1] = (torch.rand(K, generator=g, device=DEV) * 9e-6).to(dtype)                 # max < 1e-5: the clamp
    assert bool((x[0].float() == halves).sum() > K // 2)
    X = Padded(x)
    Q, S = out_buf((rows, K), torch.int8), out_buf((rows,), F32)
    ok(_lib().chitu_b200_quant_act_int8(ptr(X.view), ptr(Q.view), ptr(S.view), rows, K, dcode(dtype), stream()),
       "quant_act_int8")
    xf = x.cpu().float()
    s = xf.abs().amax(dim=-1, keepdim=True).clamp(min=1e-5) / 127.0
    q = torch.round(xf / s).to(torch.int8)
    assert float(s[0]) == 1.0
    assert torch.equal(S.view.cpu(), s.view(-1)) and torch.equal(Q.view.cpu(), q)
    assert Q.pads_intact() and S.pads_intact()


# ---------------------------------------------------------------------------------------------------- weight dequant
WD_CASES = [(B, M, N, soft) for B, M, N in ((1, 129, 300), (3, 200, 16500)) for soft in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,M,N,soft", WD_CASES,
                         ids=[f"weight_dequant_fp8-{'soft' if s else 'normal'}-B{b}-M{m}-N{n}" for b, m, n, s in WD_CASES])
def test_weight_dequant_fp8(B, M, N, soft):
    """every e4m3 byte (subnormals, +-0, the NaNs 0x7f / 0xff) at M and N that are not multiples of 128; N > 64 x 256
    makes the 64-block grid loop.  Bit exact (NaN compared as NaN in the normal mode)"""
    g = _gen(M + N + soft)
    x = torch.randint(0, 256, (B, M, N), generator=g, device=DEV, dtype=torch.uint8)
    x.view(-1)[:256] = torch.arange(256, device=DEV, dtype=torch.uint8)
    s = torch.rand(B, _cdiv(M, 128), _cdiv(N, 128), generator=g, device=DEV) * 0.01 + 1e-4
    X, Sc, Y = Padded(x), Padded(s), out_buf((B, M, N), BF)
    ok(_lib().chitu_b200_weight_dequant_fp8(ptr(X.view), ptr(Sc.view), ptr(Y.view), B, M, N, 128, soft, stream()),
       "weight_dequant_fp8")
    xc, sc = x.cpu().view(F8), s.cpu()
    ref = O.weight_dequant_soft_fp8(xc, sc) if soft else O.weight_dequant(xc, sc)
    y = Y.view.cpu()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(y), nan) and bool(nan.any()) == (not soft)
    assert torch.equal(bits(y).view(B, M, N, 2)[~nan], bits(ref).view(B, M, N, 2)[~nan])
    assert Y.pads_intact()


# ------------------------------------------------------------------------------------------------------- embedding
EMB_CASES = [(d, T, dim, shard) for d in (BF, F16) for T in (1, 256) for dim in (8, 4096, 7168) for shard in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,T,dim,shard", EMB_CASES,
                         ids=[f"embedding-{_dn(d)}-T{t}-dim{m}-{'shard' if s else 'full'}" for d, t, m, s in EMB_CASES])
def test_embedding(dtype, T, dim, shard):
    """bit exact; in a vocab shard [start, start + rows) the ids below and past it give zero rows"""
    g = _gen(T + dim + shard)
    rows, start = (500, 1000) if shard else (700, 0)
    tbits = torch.randint(-(1 << 15), 1 << 15, (rows, dim), generator=g, device=DEV, dtype=torch.int16)
    ids = torch.randint(0, 2000 if shard else rows, (T,), generator=g, device=DEV)
    if shard:
        ids[:3] = torch.tensor([999, 1000, 1500], device=DEV)[:T]
    Tb, Ids, Y = Padded(tbits.view(dtype)), Padded(ids), out_buf((T, dim), dtype)
    ok(_lib().chitu_b200_embedding(ptr(Ids.view), ptr(Tb.view), ptr(Y.view), T, dim, start, rows, dcode(dtype),
                                   stream()), "embedding")
    local = ids - start
    inside = (local >= 0) & (local < rows)
    want = torch.where(inside[:, None], tbits[local.clamp(0, rows - 1)], 0)
    assert torch.equal(bits(Y.view), bits(want))
    assert Y.pads_intact()


# ------------------------------------------------------------------------------------------------------------- add
ADD_CASES = [(d, n) for d in (BF, F16) for n in (1, 999, 1000001)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,n", ADD_CASES,
                         ids=[f"add-{_dn(d)}-n{n}{'-gridloop' if n > 132 * 8 * 256 else ''}" for d, n in ADD_CASES])
def test_add(dtype, n):
    g = _gen(n)
    a, b = rand((n,), g, dtype, 3.0), rand((n,), g, dtype, 3.0)
    A, Bp, Y = Padded(a), Padded(b), out_buf((n,), dtype)
    ok(_lib().chitu_b200_add(ptr(A.view), ptr(Bp.view), ptr(Y.view), n, dcode(dtype), stream()), "add")
    assert torch.equal(bits(Y.view), bits((a.float() + b.float()).to(dtype)))
    assert Y.pads_intact()


# ---------------------------------------------------------------------------------------------------------- argmax
AM_CASES = [(d, V) for d in (BF, F32) for V in (1, 1000, 1024, 1025, 32000, 129280)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,V", AM_CASES, ids=[f"argmax-{_dn(d)}-V{v}" for d, v in AM_CASES])
def test_argmax(dtype, V):
    """the first maximal index (torch.argmax's documented tie rule): ties planted within one thread's stride (i and
    i + 1024) and across threads, an all -inf row, and random rows"""
    g = _gen(V)
    T = 6
    x = rand((T, V), g, dtype, 3.0)
    big = torch.tensor(100.0, dtype=dtype, device=DEV)
    if V > 1030:
        x[0, 5], x[0, 5 + 1024] = big, big                   # same thread
    if V > 700:
        x[1, 700], x[1, 3] = big, big                        # different threads, the later index first in thread order
    x[2] = -math.inf
    x[3, 0], x[3, V - 1] = big, big
    X, Y = Padded(x), out_buf((T,), torch.int64)
    ok(_lib().chitu_b200_argmax(ptr(X.view), ptr(Y.view), T, V, dcode(dtype), stream()), "argmax")
    want = torch.argmax(x.cpu().float(), dim=-1)
    assert torch.equal(Y.view.cpu(), want)
    assert int(want[2]) == 0 and Y.pads_intact()


# -------------------------------------------------------------------------------------------------------- mla_prep
PREP_CASES = [(B, H, 2112 if (i + j) % 2 == 0 else 576, 128, 128, 512, 64)
              for i, B in enumerate((1, 2, 15, 16, 17, 33, 129, 256)) for j, H in enumerate((8, 16, 32, 128))]
PREP_CASES += [(17, 4, 400, 64, 64, 256, 32)]                                      # generic dn / dv / C / R


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,kv_sb,dn,dv,C,R", PREP_CASES,
                         ids=[f"mla_prep-bf16-B{b}-H{h}-kvsb{s}" + ("" if c == 512 else f"-dn{dn}-dv{dv}-C{c}-R{r}")
                              for b, h, s, dn, dv, c, r in PREP_CASES])
def test_mla_prep(B, H, kv_sb, dn, dv, C, R):
    """q_abs within the absorb-q bound, kv_norm within the RMSNorm bound, q_pe and k_pe within the rotary bound; the
    W_UV half of wkv_b, the q_nope columns the rotary must not touch and every row past B are NaN"""
    g = _gen(B * 131 + H)
    qk = dn + R
    q = rand((B, H, qk), g, BF)
    qb = nan_full((B + 1, H, qk), BF)
    qb[:B] = q
    kv = rand((B, C + R), g, BF, 2.0)
    kvb = nan_full((B + 1, kv_sb), BF)
    kvb[:B, kv_sb - C - R:] = kv
    w = nan_full((H, dn + dv, C), BF)
    w[:, :dn] = rand((H, dn, C), g, BF, 0.05)
    nw = (torch.rand(C, generator=g, device=DEV) + 0.5).to(BF)
    ang = torch.rand(B, R // 2, generator=g, device=DEV, dtype=torch.float64) * 1000
    cos, sin = nan_full((B + 1, R // 2), F32), nan_full((B + 1, R // 2), F32)
    cos[:B], sin[:B] = torch.cos(ang).float(), torch.sin(ang).float()
    Qb, KV, W, NW, Cs, Sn = Padded(qb), Padded(kvb), Padded(w), Padded(nw), Padded(cos), Padded(sin)
    q_abs, q_pe, new_kv = out_buf((B, H, C), BF), out_buf((B, H, R), BF), out_buf((B, C + R), BF)
    kv_ptr = KV.view.data_ptr() + (kv_sb - C - R) * 2
    ok(_lib().chitu_b200_mla_prep(ptr(Qb.view), kv_ptr, kv_sb, ptr(NW.view), ptr(Cs.view), ptr(Sn.view), ptr(W.view),
                                  ptr(q_abs.view), ptr(q_pe.view), ptr(new_kv.view), B, H, dn, dv, C, R, EPS, stream()),
       "mla_prep")
    qd, kvd = q.double(), kv.double()
    ref, acc = absorb_q_ref(qd[..., :dn], w[:, :dn].double())
    assert_bound(q_abs.view, ref, acc, BF, "q_abs")
    ref, acc = rms_ref(kvd[:, :C], nw.double(), EPS, rms_terms(C))
    assert_bound(new_kv.view[:, :C], ref, acc, BF, "kv_norm")
    c, s = cos[:B].double(), sin[:B].double()
    ref, acc = rotary_ref(qd[..., dn:], c[:, None], s[:, None])
    assert_bound(q_pe.view, ref, acc, BF, "q_pe")
    ref, acc = rotary_ref(kvd[:, C:], c, s)
    assert_bound(new_kv.view[:, C:], ref, acc, BF, "k_pe")
    for P in (q_abs, q_pe, new_kv):
        assert P.pads_intact()


# ------------------------------------------------------------------------------------------------- mla_absorb_o_quant
ABS_CASES = [(B, H, 128, 512) for B in (1, 3, 17) for H in (8, 16, 128)] + [(5, 4, 64, 320)]   # + the C != 512 loop


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,dn,C", ABS_CASES,
                         ids=[f"mla_absorb_o_quant-bf16-B{b}-H{h}" + ("" if c == 512 else f"-dn{dn}-C{c}")
                              for b, h, dn, c in ABS_CASES])
def test_mla_absorb_o_quant(B, H, dn, C):
    """out only, q only and both: out within the absorb-o bound, q / scales bit exact against act_quant of the kernel's
    own out, the q-only bytes equal to those of the run that writes both; W_UK and the rows past B are NaN"""
    g = _gen(B * 17 + H + C)
    dv = 128
    x = rand((B, H, C), g, BF)
    xb = nan_full((B + 1, H, C), BF)
    xb[:B] = x
    w = nan_full((H, dn + dv, C), BF)
    w[:, dn:] = rand((H, dv, C), g, BF, 0.05)
    X, W = Padded(xb), Padded(w)
    res = {}
    for mode in ("out", "q", "both"):
        Y = out_buf((B, H, dv), BF) if mode != "q" else None
        Q = out_buf((B, H * dv), torch.uint8) if mode != "out" else None
        S = out_buf((B, H), F32) if mode != "out" else None
        ok(_lib().chitu_b200_mla_absorb_o_quant(ptr(X.view), ptr(W.view), Y and ptr(Y.view), Q and ptr(Q.view),
                                                S and ptr(S.view), B, H, dn, dv, C, stream()), "mla_absorb_o_quant")
        for P in (Y, Q, S):
            assert P is None or P.pads_intact(), mode
        res[mode] = (Y, Q, S)
    ref, acc = absorb_o_ref(x.double(), w[:, dn:].double())
    for mode in ("out", "both"):
        assert_bound(res[mode][0].view, ref, acc, BF, mode)
    out = res["both"][0].view.cpu()
    assert torch.equal(bits(out), bits(res["out"][0].view.cpu()))
    qo, so = O.act_quant_deepseek_v3(out.reshape(B, H * dv))
    assert torch.equal(res["both"][2].view.cpu(), so) and torch.equal(res["both"][1].view.cpu(), bits(qo).view(B, -1))
    assert torch.equal(res["q"][1].view, res["both"][1].view) and torch.equal(res["q"][2].view, res["both"][2].view)


# ---------------------------------------------------------------------------------------------------------- sampling
THREADS = 1024


def sample_rule(l, T, top_k, top_p, V):
    """The fp64 rule and its slack for one row of logits l [V] (fp64, as stored).  Returns p, the sure and the possible
    kept masks, delta and delta_d (see the module docstring)."""
    inv_t = float(torch.tensor(1.0, dtype=F32) / torch.tensor(T, dtype=F32))
    a = l * inv_t
    mx = float(a.max())
    d = a - mx
    e = torch.exp(d)
    p = e / e.sum()
    fin = torch.isfinite(d)
    rho_i = torch.where(fin, U * (a.abs() + abs(mx) + d.abs()) + (2 + 1.173 * d.abs()) * 2.0 ** -23, 0.0)
    rho = float(rho_i[p >= 2.0 ** -100].max()) * 2 + (_cdiv(V, THREADS) + 40) * U
    ps, _ = p.sort(descending=True)
    asc = ps.flip(0)
    cs = torch.cumsum(ps, 0)

    def n_greater(th):
        return V - torch.searchsorted(asc, th, right=True)

    def mass_top(n):
        return torch.where(n > 0, cs[(n - 1).clamp(min=0)], torch.zeros((), dtype=cs.dtype, device=cs.device))

    eq = torch.searchsorted(asc, p, right=True) - torch.searchsorted(asc, p, right=False)
    n_sure = n_greater(p * (1 + 2 * rho))
    n_all = n_greater(p * (1 - 2 * rho))
    m_sure, m_maybe = mass_top(n_sure), mass_top(n_all) - eq * p
    n_maybe = n_all - eq
    delta = (V + 6144) * U + 2 * rho
    must = (p >= 2.0 ** -100) & (m_maybe <= top_p - delta) & (n_maybe < top_k)
    may = (p > 0) & (m_sure <= top_p + delta) & (n_sure < top_k)
    delta_d = (_cdiv(V, THREADS) + THREADS + 64) * U + 2 * rho
    return p, must, may, delta, delta_d


def check_draw(p, must, may, tok, u, delta_d):
    """the drawn token is possibly kept and its CDF interval (vocabulary order, over any kept set between `must` and
    `may`) comes within delta_d of u times the kept mass"""
    assert bool(may[tok]), ("token not keepable", tok, float(p[tok]))
    lo, hi = torch.where(must, p, 0.0), torch.where(may, p, 0.0)
    z_lo, z_hi = float(lo.sum()), float(hi.sum())
    before_lo, before_hi = float(lo[:tok].sum()), float(hi[:tok].sum())
    slack = delta_d * z_hi
    assert before_lo <= u * z_hi + slack, ("token past the target", tok, before_lo, u * z_hi)
    assert before_hi + float(p[tok]) >= u * z_lo - slack, ("token before the target", tok, before_hi + float(p[tok]),
                                                          u * z_lo)


U_TOP = 0.99999994                  # the largest float below 1


def _sample_rows(V, g, dtype):
    """(logits [B, V], T, top_k, top_p, u) rows covering the cases of the module docstring"""
    top = lambda k: k if k <= V else V
    spec = [  # (T, top_k, top_p, u, -inf fraction)
        (1.0, 0, 1.0, 0.5, 0.0), (1.0, 1, 1.0, 0.3, 0.0), (1.0, V, 0.3, 0.0, 0.0), (0.05, 0, 0.3, U_TOP, 0.0),
        (0.05, 0, 1.0, 0.7, 0.0), (1.0, 0, 1.0, U_TOP, 0.3), (0.7, top(50), 0.9, 0.0, 0.3), (1.0, 0, 1.0, U_TOP, 0.0),
        (1.0, -3, 1.0, 0.25, 0.5), (0.05, top(7), 1.0, U_TOP, 0.5)]
    B = len(spec)
    logits = torch.randn(B, V, generator=g, device=DEV) * 3
    for b, (_, _, _, _, frac) in enumerate(spec):
        if frac:
            m = torch.rand(V, generator=g, device=DEV) < frac
            m[int(torch.argmax(logits[b]))] = False
            logits[b][m] = -math.inf
    T = torch.tensor([s[0] for s in spec], device=DEV)
    K = torch.tensor([s[1] for s in spec], device=DEV, dtype=torch.int32)
    P = torch.tensor([s[2] for s in spec], device=DEV)
    Uu = torch.tensor([s[3] for s in spec], device=DEV)
    return logits.to(dtype), T, K, P, Uu


def _fallback_rows(g, B=64, V=4096):
    """top_p = 1 and u just below 1 on rows whose only finite logits sit in the last 16 threads' ranges (4 entries each,
    the last of every four -inf): the draw lands on the last kept entry, where the per-thread and the block sums round
    differently (the target can pass the end of the scan, or a picked thread can miss it in its own sum), and the sum
    of the positive probabilities is <= 1 on about half the rows"""
    logits = torch.full((B, V), -math.inf, device=DEV)
    logits[:, V - 64:] = torch.randn(B, 64, generator=g, device=DEV) * 0.3
    logits[:, V - 64 + 3::4] = -math.inf
    ones = torch.ones(B, device=DEV)
    return logits, ones, torch.zeros(B, device=DEV, dtype=torch.int32), ones, ones * U_TOP


def _run_sample(logits, T, K, P, Uu, dtype, pad=3):
    B, V = logits.shape
    lb = nan_full((B + 1, V + pad), dtype)
    lb[:B, :V] = logits.to(dtype)
    Lg = Padded(lb)
    tok, kept, mass = out_buf((B,), torch.int64), out_buf((B,), torch.int32), out_buf((B,), F32)
    ok(_lib().chitu_b200_sample_top_k_top_p(ptr(Lg.view), V + pad, B, V, dcode(dtype), ptr(T), ptr(K), ptr(P), ptr(Uu),
                                            ptr(tok.view), ptr(kept.view), ptr(mass.view), stream()), "sample_top_k_top_p")
    for X in (tok, kept, mass):
        assert X.pads_intact()
    return tok.view.cpu(), kept.view.cpu(), mass.view.cpu()


def _check_rows(logits, T, K, P, Uu, tok, kept, mass, what):
    B, V = logits.shape
    for b in range(B):
        top_k = int(K[b]) if int(K[b]) > 0 else V
        p, must, may, delta, delta_d = sample_rule(logits[b].double(), float(T[b]), top_k, float(P[b]), V)
        n_must, n_may = int(must.sum()), int(may.sum())
        ctx = (what, b, float(T[b]), top_k, float(P[b]), float(Uu[b]))
        assert n_must <= int(kept[b]) <= n_may, ctx + ("kept", int(kept[b]), n_must, n_may)
        z = float(mass[b])
        assert float(p[must].sum()) - delta <= z <= float(p[may].sum()) + delta, ctx + ("mass", z)
        check_draw(p, must, may, int(tok[b]), float(Uu[b]), delta_d)


SAMPLE_CASES = [(d, V) for d in (BF, F16, F32) for V in (1, 7, 1000, 1024, 1025, 129280)]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype,V", SAMPLE_CASES, ids=[f"sample_top_k_top_p-{_dn(d)}-V{v}" for d, v in SAMPLE_CASES])
def test_sample_top_k_top_p(dtype, V):
    """kept count and mass between those of the sure and the possible fp64 kept sets; the drawn token's CDF interval at
    u * z.  A padded row stride with a NaN pad, -inf logits, T = 0.05, top_k <= 0 / 1 / V, top_p 1 and 0.3, u 0 and
    the largest float below 1"""
    g = _gen(V + dtype.itemsize)
    logits, T, K, P, Uu = _sample_rows(V, g, dtype)
    tok, kept, mass = _run_sample(logits, T, K, P, Uu, dtype)
    _check_rows(logits, T, K, P, Uu, tok, kept, mass, "rows")
    if V > 1:
        assert int(tok[1]) == int(logits[1].float().argmax())                    # top_k = 1 is greedy


@pytest.mark.gpu
def test_sample_draw_at_the_end_of_the_kept_set():
    """the last-kept-entry fallback of the draw never returns an entry of probability 0, and returns the last kept
    entry, not the first of its thread"""
    g = _gen(4096)
    logits, T, K, P, Uu = _fallback_rows(g)
    tok, kept, mass = _run_sample(logits, T, K, P, Uu, F32)
    _check_rows(logits, T, K, P, Uu, tok, kept, mass, "fallback")
    last = logits.shape[1] - 2                                                    # the last finite logit of every row
    assert bool((tok == last).all()), tok.tolist()
