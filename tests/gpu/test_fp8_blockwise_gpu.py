"""Blockwise FP8 on the GPU: the single-pass cast bit for bit against the torch reference, the blockwise wgmma GEMM
bit for bit on exact data with a different scale in every block, the two autograd nodes against their reference path,
and training (ZeRO-3, convergence on a bigram stream beside bf16 and the tensorwise recipe)."""
import math

import pytest
import torch

from tests.common import run_distributed
from tests.numerics import U, assert_bits_equal, assert_within, dswiglu_reference, swiglu_reference, ulp

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
NAN8 = 0x7F  # a NaN byte in both formats
B = 128
FMT_IDS = dict(argvalues=[E4M3, E5M2], ids=["e4m3", "e5m2"])


def _F8():
    from deepspeed_b200.ops import fp8
    return fp8


def _K():
    from deepspeed_b200.ops.kernels import gemm_sm100
    return gemm_sm100


def _ops():
    from deepspeed_b200.ops.kernels import fp8_ops
    return fp8_ops


def _NE():
    from deepspeed_b200.ops.native import NativeOpError
    return NativeOpError


def u8(t):
    return t.view(torch.uint8)


def assert_bytes_equal(out, ref, what):
    assert out.dtype == ref.dtype and out.shape == ref.shape, (what, out.dtype, ref.dtype, out.shape, ref.shape)
    bad = u8(out.contiguous()) != u8(ref.contiguous())
    if bool(bad.any()):
        k = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} bytes differ; first at flat {k}: "
                             f"got {int(u8(out.contiguous()).reshape(-1)[k])}, want {int(u8(ref.contiguous()).reshape(-1)[k])}")


def guarded(rows, cols, dtype, fill, top=2, left=16, extra=32):
    """A ``[rows, cols]`` view (16-byte aligned rows and start) into a buffer of ``fill``: returns (buffer, view)."""
    ld = -(-(left + cols + extra) // 16) * 16
    buf = torch.full((rows + top + 3, ld), fill, dtype=torch.uint8 if dtype in (E4M3, E5M2) else dtype, device="cuda")
    buf = buf.view(dtype) if buf.dtype != dtype else buf
    return buf, buf[top:top + rows, left:left + cols]


def guard_intact(buf, view):
    """Nothing outside ``view`` was written (the fill was a NaN, or NaN bytes)."""
    mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    off = (view.data_ptr() - buf.data_ptr()) // buf.element_size()
    r0, c0 = off // buf.stride(0), off % buf.stride(0)
    mask[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = False
    out = u8(buf)[mask] == NAN8 if buf.element_size() == 1 else buf[mask].isnan()
    assert bool(out.all()), "elements outside the output were written"


# ---------------------------------------------------------------------------------------------------------------------
# 1. the single-pass cast
# ---------------------------------------------------------------------------------------------------------------------
CAST_SHAPES = [(16, 1), (48, 5), (128, 128), (80, 200), (144, 130), (1040, 333), (4096, 1024)]
MODES = [(r, c) for r in (None, "strip", "block") for c in (None, "strip", "block") if r or c]


def _spread(shape, gen):
    """bf16 data whose magnitudes differ by orders of magnitude between rows and columns: every block gets its own scale."""
    x = torch.randn(shape, generator=gen, device="cuda") * torch.logspace(-3, 3, shape[1], device="cuda")
    return (x * torch.logspace(-2, 2, shape[0], device="cuda")[:, None]).to(BF16)


@pytest.mark.parametrize("fmt", **FMT_IDS)
@pytest.mark.parametrize("shape", CAST_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_cast_block_bit_equal(fmt, shape):
    """Every combination of outputs, into strided views of NaN-filled buffers: data and scales equal the reference bit for
    bit and nothing around them is written."""
    F8, ops = _F8(), _ops()
    R, C = shape
    g = torch.Generator(device="cuda").manual_seed(R + 3 * C)
    xbuf = torch.zeros(R, C + 24, dtype=BF16, device="cuda")
    x = xbuf[:, 8:8 + C] if C % 8 else xbuf[:, :C]  # odd widths also read from an unaligned strided source
    x.copy_(_spread(shape, g))
    x[R // 2, C // 3] = 0
    rb, cb = -(-R // B), -(-C // B)
    for row, col in MODES:
        q_r, sq_r, qt_r, st_r = F8.quantize_blockwise_reference(x, fmt, row, col)
        kw, bufs = {}, []
        for mode, data, scale, names in ((row, (R, C), (cb, R) if row == "strip" else (rb, cb), ("out", "out_scale")),
                                         (col, (C, R), (rb, C) if col == "strip" else (cb, rb), ("out_t", "out_t_scale"))):
            if mode is not None:
                dbuf, kw[names[0]] = guarded(*data, fmt, NAN8)
                sbuf, kw[names[1]] = guarded(*scale, torch.float32, float("nan"), left=4, extra=4)
                bufs += [(dbuf, kw[names[0]]), (sbuf, kw[names[1]])]
        q, sq, qt, st = ops.fp8_cast_block(x, fmt, row=row, col=col, **kw)
        what = f"row={row} col={col}"
        if row:
            assert_bytes_equal(q, q_r, f"q {what}")
            assert_bits_equal(sq.contiguous(), sq_r, f"sq {what}")
        else:
            assert q is None and sq is None
        if col:
            assert_bytes_equal(qt, qt_r, f"qt {what}")
            assert_bits_equal(st.contiguous(), st_r, f"st {what}")
        else:
            assert qt is None and st is None
        for buf, view in bufs:
            guard_intact(buf, view)
    # the dispatching cast takes the native path and allocates its outputs
    q, sq, qt, st = F8.quantize_blockwise(x, fmt, row="strip", col="block")
    q_r, sq_r, qt_r, st_r = F8.quantize_blockwise_reference(x, fmt, "strip", "block")
    assert_bytes_equal(q, q_r, "q")
    assert_bytes_equal(qt, qt_r, "qt")
    assert_bits_equal(sq, sq_r, "sq")
    assert_bits_equal(st, st_r, "st")


@pytest.mark.parametrize("fmt", **FMT_IDS)
@pytest.mark.parametrize("bad", [math.inf, math.nan], ids=["inf", "nan"])
def test_cast_block_zero_and_nonfinite_blocks(fmt, bad):
    x = torch.ones(256, 384, dtype=BF16, device="cuda")
    x[:128, :128] = 0
    x[130, 200] = bad
    for row, col in (("strip", "block"), ("block", "strip")):
        got = _ops().fp8_cast_block(x, fmt, row=row, col=col)
        want = _F8().quantize_blockwise_reference(x, fmt, row, col)
        for t, t_r, what in zip(got, want, ("q", "sq", "qt", "st")):
            if t.dtype == torch.float32:
                assert torch.equal(t.isnan(), t_r.isnan()) and torch.equal(t.nan_to_num(7.0), t_r.nan_to_num(7.0)), what
            else:  # a NaN scale makes NaN bytes (any NaN encoding), everything else is bit-equal
                assert torch.equal(t.float().isnan(), t_r.float().isnan()), what
                keep = ~t_r.float().isnan()
                assert torch.equal(u8(t)[keep], u8(t_r)[keep]), what
    q, sq, qt, st = _ops().fp8_cast_block(x, fmt, row="strip", col="block")
    assert int(sq.isnan().sum()) == 1 and bool(sq[1, 130].isnan()) and bool((sq[0, :128] == 1).all())
    assert int(st.isnan().sum()) == 1 and bool(st[1, 1].isnan()) and float(st[0, 0]) == 1


def test_cast_block_refusals_write_nothing():
    from deepspeed_b200.ops import native as N
    NE = _NE()
    x = torch.randn(48, 64, device="cuda").to(BF16)
    qbuf = torch.full((64, 64), NAN8, dtype=torch.uint8, device="cuda")
    tbuf = torch.full((64, 64), NAN8, dtype=torch.uint8, device="cuda")
    sbuf = torch.full((64, ), 7.0, device="cuda")
    tsbuf = torch.full((64, ), 7.0, device="cuda")

    def cast(R=48, C=64, ld=64, fmt=N.F8E4M3, row=1, q=qbuf, ld_q=64, sq=sbuf, ld_sq=64, col=0, qt=None, ld_t=0, st=None,
             ld_st=0):
        rc = N.cuda().dsb_fp8_cast_block(N.ptr(x), N.c_i64(R), N.c_i64(C), N.c_i64(ld), fmt, row, N.ptr(q), N.c_i64(ld_q),
                                         N.ptr(sq), N.c_i64(ld_sq), col, N.ptr(qt), N.c_i64(ld_t), N.ptr(st), N.c_i64(ld_st),
                                         N.stream())
        N.check(rc, "fp8_cast_block")

    t = dict(col=1, qt=tbuf, ld_t=64, st=tsbuf, ld_st=64)
    bad = [dict(R=0), dict(C=0), dict(ld=32), dict(fmt=N.BF16), dict(row=0), dict(row=3), dict(row=-1), dict(t, col=3),
           dict(q=None), dict(sq=None), dict(ld_q=48), dict(q=qbuf.view(-1)[8:]), dict(ld_sq=40), dict(row=2, ld_sq=0),
           dict(t, R=40),  # R % 16
           dict(t, qt=None), dict(t, st=None), dict(t, ld_t=40), dict(t, ld_t=32), dict(t, qt=tbuf.view(-1)[8:]),
           dict(t, ld_st=48), dict(t, col=2, ld_st=0)]
    for kw in bad:
        with pytest.raises(NE, match="unsupported shape"):
            cast(**kw)
    torch.cuda.synchronize()
    assert bool((qbuf == NAN8).all()) and bool((tbuf == NAN8).all()) and bool((sbuf == 7).all()) and bool((tsbuf == 7).all())
    cast(**t)  # the baseline arguments are accepted
    torch.cuda.synchronize()
    assert not bool((qbuf[:48] == NAN8).all()) and not bool((tbuf[:, :48] == NAN8).all())
    with pytest.raises(NE):
        _ops().fp8_cast_block(x.float(), E4M3)
    with pytest.raises(NE):
        _ops().fp8_cast_block(x, E4M3, row=None, col=None)
    with pytest.raises(NE):
        _ops().fp8_cast_block(x, E4M3, out_scale=torch.empty(2, 48, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------------
# 2. the blockwise GEMM, exact oracle
# ---------------------------------------------------------------------------------------------------------------------
def f8_grid(rows, cols, fmt, gen, emin=-3, emax=3, lo=-2, hi=2):
    """fp8 ``[rows, cols]``: integers in ``[lo, hi]`` times ``2**e_r`` (one exponent per row), exact in both formats."""
    v = torch.randint(lo, hi + 1, (rows, cols), generator=gen, device="cuda", dtype=torch.int32).float()
    e = torch.randint(emin, emax + 1, (rows, ), generator=gen, device="cuda", dtype=torch.int32)
    return torch.ldexp(v, e[:, None]).to(fmt), e


def block_scales(M, rows_b, K, spread=2):
    """Power-of-two ``(sa_inv [ceil(K/128), M], sb_inv [ceil(rows_b/128), ceil(K/128)])`` that differ between any two
    neighbouring rows, k-blocks and n-blocks, so a scale read from a wrong row, k-block or n-block changes the result."""
    kb, nb = -(-K // B), -(-rows_b // B)
    n = 2 * spread + 1
    ia = torch.arange(kb, device="cuda")[:, None] * 3 + torch.arange(M, device="cuda")[None, :]
    ib = torch.arange(nb, device="cuda")[:, None] * 2 + torch.arange(kb, device="cuda")[None, :] * 3
    return torch.ldexp(torch.ones(()).cuda(), (ia % n - spread).int()), torch.ldexp(torch.ones(()).cuda(), (ib % n - spread).int())


def dequant(a, sa, b, sb):
    """float64 ``(A, B)`` with their block scales applied."""
    ad = a.double() * sa.t().double().repeat_interleave(B, dim=1)[:, :a.shape[1]]
    bd = b.double() * sb.double().repeat_interleave(B, dim=0)[:b.shape[0]].repeat_interleave(B, dim=1)[:, :b.shape[1]]
    return ad, bd


def exact_c(a, sa, b, sb, c_old=None):
    """The product in float64.  On :func:`f8_grid` operands with :func:`block_scales` every partial sum is an integer
    multiple of one power of two no more than 24 bits below the largest, so the kernel's fp32 accumulation is exact."""
    ad, bd = dequant(a, sa, b, sb)
    ref = ad @ bd.t()
    return ref if c_old is None else ref + c_old.double()


GEMM_SHAPES = [(128, 128, 128), (1, 8, 16), (7, 24, 48), (200, 136, 400), (300, 520, 272), (513, 264, 1040)]


@pytest.mark.parametrize("afmt", [E4M3, E5M2], ids=["a_e4m3", "a_e5m2"])
@pytest.mark.parametrize("accum", [False, True], ids=["store", "accum"])
@pytest.mark.parametrize("shape", GEMM_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_block_exact(afmt, accum, shape):
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + 7 * N + 13 * K + int(accum))
    a_val, ea = f8_grid(M, K, afmt, g)
    b_val, eb = f8_grid(N, K, E4M3, g)
    abuf, a = guarded(M, K, afmt, NAN8)
    bbuf, b = guarded(N, K, E4M3, NAN8)
    a.copy_(a_val)
    b.copy_(b_val)
    sa_val, sb_val = block_scales(M, N, K)
    # strided scale tensors inside NaN: a read outside them would poison C
    sabuf, sa = guarded(*sa_val.shape, torch.float32, float("nan"), left=4, extra=4)
    sbbuf, sb = guarded(*sb_val.shape, torch.float32, float("nan"), left=4, extra=4)
    sa.copy_(sa_val)
    sb.copy_(sb_val)
    cbuf, c = guarded(M, N, BF16, float("nan"), left=8, extra=8)
    c_old = None
    if accum:
        v = torch.randint(-128, 129, (M, N), generator=g, device="cuda").float()
        c_old = (torch.ldexp(v, ea[:, None] + eb[None, :]) * (2.0**-3)).to(BF16)
        c.copy_(c_old)
    K_ = _K()
    K_.fp8_matmul_block(a, b, sa, sb, out=c, epi=K_.EPI_ACCUM if accum else K_.EPI_STORE)
    ref = exact_c(a_val, sa_val, b_val, sb_val, c_old)
    assert_bits_equal(c, ref.to(BF16), "C")
    assert torch.equal(_F8().matmul_blockwise_reference(a_val, b_val, sa_val, sb_val).double(), exact_c(a_val, sa_val, b_val, sb_val))
    guard_intact(cbuf, c)


@pytest.mark.parametrize("afmt", [E4M3, E5M2], ids=["a_e4m3", "a_e5m2"])
def test_gemm_block_large_k_needs_promotion(afmt):
    """K = 16384 of positive products with per-block scales: the sums reach 2**16 and keep every low bit."""
    M, N, K = 128, 256, 16384
    g = torch.Generator(device="cuda").manual_seed(5)
    a, _ = f8_grid(M, K, afmt, g, emin=0, emax=0, lo=1, hi=4)
    b, _ = f8_grid(N, K, E4M3, g, emin=0, emax=0, lo=1, hi=4)
    sa, sb = block_scales(M, N, K, spread=1)
    c = _K().fp8_matmul_block(a, b, sa, sb)
    ref = exact_c(a, sa, b, sb)
    assert float(ref.max()) > 2.0**16
    assert torch.equal(ref.float().double(), ref), "the exact result fits fp32"
    assert_bits_equal(c, ref.to(BF16), "C")


@pytest.mark.parametrize("shape", [(128, 64, 128), (200, 192, 400), (77, 320, 48), (130, 256, 272)],
                         ids=lambda s: "x".join(map(str, s)))
def test_gemm_block_swiglu_exact(shape):
    """``inter % 128 == 64`` puts a tile's gate rows and up rows at different offsets inside their 128-row scale blocks."""
    M, I, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + I + K)
    a, _ = f8_grid(M, K, E4M3, g)
    w, _ = f8_grid(2 * I, K, E4M3, g)
    sa, sb = block_scales(M, 2 * I, K)
    cbuf, act = guarded(M, I, BF16, float("nan"), left=8, extra=8)
    gbuf, gu = guarded(M, 2 * I, BF16, float("nan"), left=8, extra=8)
    K_ = _K()
    K_.fp8_matmul_block(a, w, sa, sb, out=act, epi=K_.EPI_SWIGLU, out2=gu)
    ref = exact_c(a, sa, w, sb)
    assert_bits_equal(gu, ref.to(BF16), "gate|up")
    want, bound = swiglu_reference(ref[:, :I], ref[:, I:])
    assert_within(act, want, bound, "act")
    guard_intact(cbuf, act)
    guard_intact(gbuf, gu)
    act2 = K_.fp8_matmul_block(a, w, sa, sb, epi=K_.EPI_SWIGLU)
    assert_bits_equal(act2, act.contiguous(), "act without the gate|up save")


@pytest.mark.parametrize("shape", [(128, 128, 128), (200, 72, 400), (64, 520, 48)], ids=lambda s: "x".join(map(str, s)))
def test_gemm_block_dswiglu_exact(shape):
    M, I, K = shape
    g = torch.Generator(device="cuda").manual_seed(3 * M + I + K)
    a, _ = f8_grid(M, K, E5M2, g)
    w, _ = f8_grid(I, K, E4M3, g)
    sa, sb = block_scales(M, I, K)
    gu = (torch.randn(M, 2 * I, generator=g, device="cuda") * 2).to(BF16)
    obuf, out2 = guarded(M, 2 * I, BF16, float("nan"), left=8, extra=8)
    K_ = _K()
    K_.fp8_matmul_block(a, w, sa, sb, epi=K_.EPI_DSWIGLU, aux=gu, out2=out2)
    d = exact_c(a, sa, w, sb)
    dg, dg_b, du, du_b = dswiglu_reference(d, gu[:, :I], gu[:, I:], d_fp32=True)
    assert_within(out2[:, :I], dg, dg_b, "dgate")
    assert_within(out2[:, I:], du, du_b, "dup")
    guard_intact(obuf, out2)


@pytest.mark.parametrize("epi", ["store", "accum", "swiglu", "dswiglu"])
def test_gemm_block_equal_scales_reproduce_tensorwise(epi):
    """With one value in every entry of both scale tensors the blockwise kernel computes what the tensorwise kernel does
    on the same bytes, bit for bit, on random (inexact) data."""
    M, N, K = 392, 384, 1008
    g = torch.Generator(device="cuda").manual_seed(13)
    afmt = E5M2 if epi == "dswiglu" else E4M3
    a = (torch.randn(M, K, generator=g, device="cuda") * 8).to(afmt)
    b = (torch.randn(N, K, generator=g, device="cuda") * 8).to(E4M3)
    K_ = _K()
    sa1, sb1 = torch.tensor([2.0**-7], device="cuda"), torch.tensor([2.0**-6], device="cuda")
    sa = sa1.expand(-(-K // B), M).contiguous()
    sb = sb1.expand(-(-N // B), -(-K // B)).contiguous()
    Nn = N // 2 if epi == "swiglu" else N
    kw_t, kw_b = {}, {}
    if epi == "accum":
        c0 = torch.randn(M, N, generator=g, device="cuda").to(BF16)
        kw_t, kw_b = dict(out=c0.clone(), epi=K_.EPI_ACCUM), dict(out=c0.clone(), epi=K_.EPI_ACCUM)
    elif epi == "swiglu":
        kw_t = dict(epi=K_.EPI_SWIGLU, out2=torch.empty(M, N, dtype=BF16, device="cuda"))
        kw_b = dict(epi=K_.EPI_SWIGLU, out2=torch.empty(M, N, dtype=BF16, device="cuda"))
    elif epi == "dswiglu":
        gu = torch.randn(M, 2 * N, generator=g, device="cuda").to(BF16)
        kw_t = dict(epi=K_.EPI_DSWIGLU, aux=gu, out2=torch.empty(M, 2 * N, dtype=BF16, device="cuda"))
        kw_b = dict(epi=K_.EPI_DSWIGLU, aux=gu, out2=torch.empty(M, 2 * N, dtype=BF16, device="cuda"))
    want = K_.fp8_matmul(a, b, sa1, sb1, **kw_t)
    got = K_.fp8_matmul_block(a, b, sa, sb, **kw_b)
    assert tuple(got.shape) == (M, Nn)
    assert_bits_equal(got.contiguous(), want.contiguous(), "C")
    if "out2" in kw_t:
        assert_bits_equal(kw_b["out2"], kw_t["out2"], "out2")


@pytest.mark.parametrize("epi", ["store", "swiglu"])
def test_gemm_block_cta_counts_bit_identical(epi):
    """Random (inexact) data and scales: 1-7 persistent CTAs and every rasterisation give the same bits."""
    M, N, K = 392, 384, 1008
    g = torch.Generator(device="cuda").manual_seed(11)
    a = (torch.randn(M, K, generator=g, device="cuda") * 8).to(E4M3)
    b = (torch.randn(N, K, generator=g, device="cuda") * 8).to(E4M3)
    sa, sb = block_scales(M, N, K, spread=3)
    K_ = _K()
    e = K_.EPI_SWIGLU if epi == "swiglu" else K_.EPI_STORE
    out2 = torch.empty(M, N, dtype=BF16, device="cuda") if epi == "swiglu" else None
    first = K_.fp8_matmul_block(a, b, sa, sb, epi=e, out2=out2)
    first2 = out2.clone() if out2 is not None else None
    for sms in range(1, 8):
        for gm in (0, 1, 3, 8):
            c = K_.fp8_matmul_block(a, b, sa, sb, epi=e, out2=out2, sms=sms, group_m=gm)
            assert_bits_equal(c, first, f"C sms={sms} group_m={gm}")
            if out2 is not None:
                assert_bits_equal(out2, first2, f"gate|up sms={sms} group_m={gm}")


def test_gemm_block_nan_scale_poisons_its_rows_and_columns_only():
    M, N, K = 200, 392, 400
    a = torch.ones(M, K, device="cuda").to(E4M3)
    b = torch.ones(N, K, device="cuda").to(E4M3)
    sa, sb = block_scales(M, N, K)
    sa[2, 137] = float("nan")  # row 137, third k-block
    c = _K().fp8_matmul_block(a, b, sa, sb)
    nan = c.isnan()
    assert bool(nan[137].all()) and int(nan.sum()) == N, "exactly the row of the NaN strip"
    sa, sb = block_scales(M, N, K)
    sb[1, 3] = float("nan")  # columns 128..255, last (partial) k-block
    nan = _K().fp8_matmul_block(a, b, sa, sb).isnan()
    assert bool(nan[:, 128:256].all()) and int(nan.sum()) == M * 128, "exactly the columns of the NaN block"
    # SwiGLU: a NaN in an up block reaches act and the up half of gate|up, not the gate half
    I = 192
    w = torch.ones(2 * I, K, device="cuda").to(E4M3)
    sa, sb = block_scales(M, 2 * I, K)
    sb[2, 0] = float("nan")  # rows 256..383 of [gate; up] = up features 64..191
    gu = torch.empty(M, 2 * I, dtype=BF16, device="cuda")
    act = _K().fp8_matmul_block(a, w, sa, sb, epi=_K().EPI_SWIGLU, out2=gu)
    assert bool(act[:, 64:].isnan().all()) and not bool(act[:, :64].isnan().any())
    assert bool(gu[:, 256:].isnan().all()) and not bool(gu[:, :256].isnan().any())


def test_gemm_block_refusals_write_nothing():
    """The -2 conditions ``dsb_gemm_fp8_block`` adds to those of ``dsb_gemm_fp8``, and a sample of the shared ones."""
    from deepspeed_b200.ops import native as N
    NE = _NE()
    abuf = torch.ones(256, 256, device="cuda").to(E4M3)
    a5 = torch.ones(256, 256, device="cuda").to(E5M2)
    cbuf = torch.full((256, 256), float("nan"), dtype=BF16, device="cuda")
    s = torch.ones(2, 256, device="cuda")

    def call(a=abuf, b=abuf, c=cbuf, M=64, n=64, K=192, lda=256, ldb=256, ldc=256, fmt=N.F8E4M3, sa=s, ld_sa=256, sb=s,
             ld_sb=256, epi=0, aux_=None, ld_aux=0, out2=None, ld_out2=0):
        rc = N.cuda().dsb_gemm_fp8_block(N.ptr(a), N.ptr(b), N.ptr(c), M, n, K, lda, ldb, ldc, fmt, N.ptr(sa), ld_sa,
                                         N.ptr(sb), ld_sb, epi, N.ptr(aux_), ld_aux, N.ptr(out2), ld_out2, 8, 0, N.stream())
        N.check(rc, "gemm_fp8_block")

    cases = [dict(ld_sa=63), dict(ld_sa=0), dict(ld_sb=1), dict(ld_sb=0), dict(sa=None), dict(sb=None), dict(M=0),
             dict(K=24), dict(n=12), dict(lda=40), dict(ldc=60), dict(a=abuf.view(-1)[8:]), dict(fmt=N.BF16), dict(epi=4),
             dict(epi=2, a=a5, fmt=N.F8E5M2), dict(epi=2, n=72), dict(epi=3)]
    for kw in cases:
        with pytest.raises(NE, match="unsupported shape"):
            call(**kw)
    torch.cuda.synchronize()
    assert bool(cbuf.isnan().all()), "a refused call wrote C"
    call()  # the baseline arguments are accepted
    torch.cuda.synchronize()
    assert not bool(cbuf[:64, :64].isnan().any())
    K_ = _K()
    a, b = abuf[:64, :192], abuf[:128, :192]
    sa, sb = torch.ones(2, 64, device="cuda"), torch.ones(1, 2, device="cuda")
    K_.fp8_matmul_block(a, b, sa, sb)
    for bad_sa, bad_sb in ((sa[:1], sb), (sa, sb[:, :1]), (sa.t().contiguous(), sb), (sa, torch.ones(2, 2, device="cuda")),
                           (sa.double(), sb), (torch.ones(1, device="cuda"), torch.ones(1, device="cuda"))):
        with pytest.raises(NE, match="do not fit"):
            K_.fp8_matmul_block(a, b, bad_sa, bad_sb)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the autograd nodes
# ---------------------------------------------------------------------------------------------------------------------
# As in the tensorwise tests: inside a k-block the fp8 tensor core keeps about 14 bits of the products it adds; the bound
# allows 2**-11 of the magnitudes for the blocks, plus the fp32 promotion and the bf16 rounding.
FP8_BLOCK_REL = 2.0**-11


def _bounded(got, ad, bd, what):
    """``got`` (bf16) within the kernel's accumulation error of ``ad @ bd^T`` (float64 dequantised operands)."""
    ref, mag = ad @ bd.t(), ad.abs() @ bd.abs().t()
    acc = FP8_BLOCK_REL * mag + 2 * (ad.shape[1] // B + 1) * U * mag
    err = (got.double() - ref).abs() - ulp(ref.abs(), BF16)
    print(f"[fp8 blockwise accumulation] {what}: worst |C - exact| beyond one bf16 ulp = "
          f"2**{math.log2(max(float((err / mag.clamp_min(1e-300)).max()), 2**-60)):.1f} of the magnitudes")
    assert_within(got, ref, ulp(ref.abs() + acc, BF16) + acc, what)


def test_fp8_blockwise_linear_node():
    from deepspeed_b200.ops.linear import fp8_linear
    F8 = _F8()
    g = torch.Generator(device="cuda").manual_seed(1)
    T, Kd, Nd = 400, 528, 368  # partial blocks in every dimension
    x = _spread((T, Kd), g).view(2, T // 2, Kd).requires_grad_(True)
    w = (torch.randn(Nd, Kd, generator=g, device="cuda") * 0.03).to(BF16).requires_grad_(True)
    dy = _spread((T, Nd), g).view(2, T // 2, Nd)
    y = fp8_linear(x, w, recipe="blockwise")
    x8t, sxt = y.grad_fn.saved_tensors
    y.backward(dy)
    x2, dy2 = x.detach().reshape(T, Kd), dy.reshape(T, Nd)
    x8, sx, x8t_r, sxt_r = F8.quantize_blockwise_reference(x2, E4M3, "strip", "block")
    w8, sw, w8t, swt = F8.quantize_blockwise_reference(w.detach(), E4M3, "block", "block")
    dy8, sdy, dy8t, sdyt = F8.quantize_blockwise_reference(dy2, E5M2, "strip", "strip")
    assert_bytes_equal(x8t, x8t_r, "saved x^T")
    assert_bits_equal(sxt, sxt_r, "saved scale_inv")
    _bounded(y.detach().reshape(T, Nd), *dequant(x8, sx, w8, sw), "y")
    _bounded(x.grad.reshape(T, Kd), *dequant(dy8, sdy, w8t, swt), "dx")
    _bounded(w.grad, *dequant(dy8t, sdyt, x8t_r, sxt_r), "dw")


def test_fp8_blockwise_swiglu_node_against_reference_path(monkeypatch):
    from deepspeed_b200.ops import linear
    F8 = _F8()
    g = torch.Generator(device="cuda").manual_seed(2)
    T, H, I = 528, 272, 448  # I % 128 == 64
    x0 = torch.randn(T, H, generator=g, device="cuda").to(BF16)
    wgu0 = (torch.randn(2 * I, H, generator=g, device="cuda") * H**-0.5).to(BF16)
    wd0 = (torch.randn(H, I, generator=g, device="cuda") * I**-0.5).to(BF16)
    dy = torch.randn(T, H, generator=g, device="cuda").to(BF16)

    def run():
        x, wgu, wd = (t.clone().requires_grad_(True) for t in (x0, wgu0, wd0))
        y = linear.fp8_swiglu_mlp(x, wgu, wd, recipe="blockwise")
        saved = [t.clone() for t in y.grad_fn.saved_tensors]
        y.backward(dy)
        return y.detach(), x.grad, wgu.grad, wd.grad, saved

    y, dx, dwgu, dwd, (x8t, sxt, gu, act8t, sat) = run()
    monkeypatch.setattr(linear, "_fp8_native", lambda *a, **k: False)
    y_r, dx_r, dwgu_r, dwd_r, (x8t_r, sxt_r, gu_r, act8t_r, sat_r) = run()
    assert_bytes_equal(x8t, x8t_r, "x^T")
    assert_bits_equal(sxt, sxt_r, "x^T scale_inv")
    x8, sx, _, _ = F8.quantize_blockwise_reference(x0, E4M3, "strip")
    wgu8, sgu, _, _ = F8.quantize_blockwise_reference(wgu0, E4M3, "block")
    _bounded(gu, *dequant(x8, sx, wgu8, sgu), "gate|up")
    # the forward output and the gradients pass through silu (``__expf`` against ``torch.exp``) and a cast whose rounding
    # can flip where the two differ in the last bit: compare the two paths in norm
    for got, want, what in ((y, y_r, "y"), (dx, dx_r, "dx"), (dwgu, dwgu_r, "dW_gate_up"), (dwd, dwd_r, "dW_down")):
        rel = float((got.float() - want.float()).norm() / want.float().norm())
        assert rel < 2e-2, (what, rel)


def test_fp8_blockwise_nodes_make_no_host_sync():
    from deepspeed_b200.ops.linear import fp8_linear, fp8_swiglu_mlp
    x = torch.randn(256, 256, device="cuda").to(BF16).requires_grad_(True)
    w = (torch.randn(512, 256, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    wd = (torch.randn(256, 256, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    fp8_swiglu_mlp(fp8_linear(x, wd, recipe="blockwise"), w, wd, recipe="blockwise").sum().backward()  # modules loaded
    x.grad = w.grad = wd.grad = None
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = fp8_swiglu_mlp(fp8_linear(x, wd, recipe="blockwise"), w, wd, recipe="blockwise")
        y.sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for t in (x.grad, w.grad, wd.grad):
        assert bool(torch.isfinite(t).all()) and bool(t.any())


# ---------------------------------------------------------------------------------------------------------------------
# 4. training
# ---------------------------------------------------------------------------------------------------------------------
def _llama(recipe, vocab=1024, **kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    fp8 = dict(fp8=True, fp8_recipe=recipe) if recipe else {}
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=vocab, num_hidden_layers=2, max_position_embeddings=512, **fp8, **kw)
    with torch.device("cuda"):
        return LlamaForCausalLM(cfg).to(BF16)


def _engine(model, stage, lr=1e-3, gas=1):
    import deepspeed_b200 as ds
    cfg = {"train_micro_batch_size_per_gpu": 2, "gradient_accumulation_steps": gas, "bf16": {"enabled": True},
           "optimizer": {"type": "AdamW", "params": {"lr": lr}}, "zero_optimization": {"stage": stage}}
    engine, _, _, _ = ds.initialize(model=model, config=cfg)
    return engine


def _blockwise_llama_zero3():
    """ZeRO-3 with two micro steps per step: dW is stored into the flat gradient views on the first micro step and
    accumulated by the GEMM epilogue on the second; the gradients match the bf16 model's on the same weights."""
    from deepspeed_b200.ops import linear, native
    ran = {"accum": 0, "store": 0}
    real = linear._weight_grad_sink

    def weight_grad(w, dtype, into, *a, **k):
        # every projection of this model is an FP8 node, whose sink writes with a partial of the FP8 GEMM
        zo = linear._zo_of(w)
        assert zo is not None and into.keywords.get("block") is True, "dW goes into the flat view, blockwise"
        ran["store" if zo.grad_is_fresh(w) else "accum"] += 1
        return real(w, dtype, into, *a, **k)

    linear._weight_grad_sink = weight_grad
    engine = _engine(_llama("blockwise", checkpoint_layers=1), 3, gas=2)
    ids = torch.randint(0, 1024, (2, 256), generator=torch.Generator().manual_seed(1)).cuda()
    before = native.launch_count
    losses = []
    for _ in range(6):
        for _ in range(2):
            loss = engine(ids, labels=ids)
            engine.backward(loss)
            engine.step()
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses), losses
    assert losses[-1] < losses[0] - 0.5, losses
    assert native.launch_count > before
    assert ran["store"] > 0 and ran["accum"] > 0, ran


def test_fp8_blockwise_llama_zero3_stores_then_accumulates_dw():
    run_distributed(_blockwise_llama_zero3, 1, ())


def test_fp8_blockwise_weight_grad_store_then_accumulate():
    """dW into a bf16 gradient view: stored, then accumulated in the GEMM epilogue (one rounding of old + product)."""
    F8 = _F8()
    g = torch.Generator(device="cuda").manual_seed(3)
    T, Kd, Nd = 384, 272, 400
    dy, x = _spread((T, Nd), g), _spread((T, Kd), g)
    _, _, dy8t, sdyt = F8.quantize_blockwise(dy, E5M2, row=None, col="strip")
    _, _, x8t, sxt = F8.quantize_blockwise(x, E4M3, row=None, col="block")
    gbuf, gv = guarded(Nd, Kd, BF16, float("nan"), left=8, extra=8)
    F8.gemm(dy8t, x8t, sdyt, sxt, True, out=gv, block=True)
    first = gv.clone()
    ad, bd = dequant(dy8t, sdyt, x8t, sxt)
    _bounded(first, ad, bd, "dW stored")
    F8.gemm(dy8t, x8t, sdyt, sxt, True, out=gv, accumulate=True, block=True)
    ref, mag = ad @ bd.t() + first.double(), ad.abs() @ bd.abs().t() + first.double().abs()
    acc = FP8_BLOCK_REL * mag + 2 * (T // B + 2) * U * mag
    assert_within(gv, ref, ulp(ref.abs() + acc, BF16) + acc, "dW accumulated")
    guard_intact(gbuf, gv)


# Final losses on the bigram stream of the tensorwise test (mean of the last 10 of 120 steps).  Measured on an H100 80GB
# HBM3 at 700 W: bf16 3.0230, tensorwise 3.0540, blockwise 3.0203 (entropy floor 2.535).  The tolerance against bf16 is the
# one that test uses for the tensorwise recipe.
CONVERGENCE_GAP = 0.1


def _bigram_batches(steps, vocab=256, Bsz=2, S=256, seed=0):
    """Token streams from a fixed random bigram table (each token has a few likely successors): learnable, with a known
    entropy floor."""
    g = torch.Generator().manual_seed(seed)
    probs = torch.softmax(torch.randn(vocab, vocab, generator=g) * 3, -1)
    floor = float(-(probs * probs.log()).sum(-1).mean())
    out = []
    for _ in range(steps):
        ids = torch.empty(Bsz, S, dtype=torch.long)
        ids[:, 0] = torch.randint(0, vocab, (Bsz, ), generator=g)
        for t in range(1, S):
            ids[:, t] = torch.multinomial(probs[ids[:, t - 1]], 1, generator=g).squeeze(1)
        out.append(ids)
    return out, floor


def _convergence():
    batches, floor = _bigram_batches(120)
    finals = {}
    for recipe in (None, "tensorwise", "blockwise"):
        engine = _engine(_llama(recipe, vocab=256), 3, lr=2e-3)
        losses = []
        for ids in batches:
            ids = ids.cuda()
            loss = engine(ids, labels=ids)
            engine.backward(loss)
            engine.step()
            losses.append(float(loss))
        finals[recipe or "bf16"] = sum(losses[-10:]) / 10
        del engine
    gap = finals["blockwise"] - finals["bf16"]
    print(f"[fp8 blockwise convergence] bf16 {finals['bf16']:.4f} tensorwise {finals['tensorwise']:.4f} "
          f"blockwise {finals['blockwise']:.4f} (blockwise - bf16 {gap:+.4f}) entropy floor {floor:.4f}")
    assert finals["bf16"] < math.log(256) - 1.0, finals  # the runs learned the bigrams
    assert abs(gap) <= CONVERGENCE_GAP, (finals, gap)


def test_fp8_blockwise_convergence_matches_bf16():
    run_distributed(_convergence, 1, ())
