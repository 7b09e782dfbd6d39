"""FP8 training on the wgmma kernels: the amax / cast(-transpose) kernels bit for bit against the torch recipe, the FP8
GEMM under an exact oracle, the two autograd nodes against float64, and FP8 Llama training under ZeRO-3.

Exact oracle.  Operands are small integers on fp8 grids times a power of two per row, and the scale inverses are powers of
two.  While every partial sum fits fp32's significand, an fp32 accumulation is exact in any order, so C must be bit-equal
to the float64 product rounded once to bf16 (ACCUM: ``C_old + exact``, rounded once).  Hopper's fp8 wgmma accumulates
with fewer bits than fp32; the kernel promotes every 128 products into an fp32 accumulator, and the large-K case checks
that: its partial sums grow past 2**14, where an unpromoted accumulation loses low bits."""
import math

import pytest
import torch

from tests.common import run_distributed
from tests.numerics import (U, assert_bits_equal, assert_within, dswiglu_reference, gemm_bound, swiglu_reference, ulp)

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FMAX = {E4M3: 448.0, E5M2: 57344.0}
NAN8 = 0x7F  # a NaN byte in both formats


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


def guarded_f8(rows, cols, fmt, top=2, left=16, extra=32):
    """A ``[rows, cols]`` fp8 view into a NaN-filled buffer (16-byte aligned rows and start): returns (buffer, view)."""
    ld = -(-(left + cols + extra) // 16) * 16
    buf = torch.full((rows + top + 3, ld), NAN8, dtype=torch.uint8, device="cuda").view(fmt)
    return buf, buf[top:top + rows, left:left + cols]


def guard_intact_f8(buf, view):
    mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    r0 = (view.data_ptr() - buf.data_ptr()) // buf.stride(0)
    c0 = (view.data_ptr() - buf.data_ptr()) % buf.stride(0)
    mask[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = False
    assert bool((u8(buf)[mask] == NAN8).all()), "bytes outside the output were written"


# ---------------------------------------------------------------------------------------------------------------------
# 1. amax and cast(-transpose)
# ---------------------------------------------------------------------------------------------------------------------
CAST_SHAPES = [(1, 1), (3, 5), (16, 7), (64, 64), (80, 200), (33, 130), (1040, 333), (4096, 1024)]


@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("shape", CAST_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_cast_bit_equal(fmt, shape):
    R, C = shape
    g = torch.Generator(device="cuda").manual_seed(R * 1000 + C)
    big = torch.full((R + 4, C + 11), float("nan"), dtype=BF16, device="cuda")
    x = big[1:1 + R, 3:3 + C]
    x.copy_((torch.randn(R, C, generator=g, device="cuda") * torch.logspace(-4, 4, C, device="cuda")).to(BF16))
    amax = _ops().fp8_amax(x)
    assert float(amax) == float(x.float().abs().max())
    q_ref, qt_ref, si_ref = _F8().quantize_reference(x, fmt, rowwise=True, colwise=True)
    qbuf, q = guarded_f8(R, C, fmt)
    colwise = R % 16 == 0
    tbuf, qt = guarded_f8(C, R, fmt) if colwise else (None, None)
    _, _, si = _ops().fp8_cast(x, amax, fmt, rowwise=True, colwise=colwise, out=q, out_t=qt)
    assert_bits_equal(si, si_ref, "scale_inv")
    assert_bytes_equal(q, q_ref, "q")
    guard_intact_f8(qbuf, q)
    if colwise:
        assert_bytes_equal(qt, qt_ref, "qt")
        assert_bytes_equal(qt, q.t(), "qt vs q^T")
        guard_intact_f8(tbuf, qt)
        # the transposed output alone is the same bytes
        _, qt2, _ = _ops().fp8_cast(x, amax, fmt, rowwise=False, colwise=True)
        assert_bytes_equal(qt2, qt_ref, "qt alone")
    # the front door picks the kernels here and matches the reference
    d, dt, s = _F8().quantize_tensorwise(x, fmt, rowwise=True, colwise=colwise)
    assert_bytes_equal(d, q_ref, "quantize_tensorwise")
    assert_bits_equal(s, si_ref, "quantize_tensorwise scale_inv")
    # contiguous rows (the vectorised loads and stores the training step uses)
    d, dt, s = _F8().quantize_tensorwise(x.contiguous(), fmt, rowwise=True, colwise=colwise)
    assert_bytes_equal(d, q_ref, "contiguous q")
    if colwise:
        assert_bytes_equal(dt, qt_ref, "contiguous qt")


@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_cast_all_zero(fmt):
    x = torch.zeros(64, 96, dtype=BF16, device="cuda")
    q, qt, si = _F8().quantize_tensorwise(x, fmt, rowwise=True, colwise=True)
    assert float(si) == 1.0 and not bool(u8(q).any()) and not bool(u8(qt).any())


@pytest.mark.parametrize("fmt", [E4M3, E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("bad", [math.inf, -math.inf, math.nan], ids=["inf", "-inf", "nan"])
def test_cast_nonfinite_is_nan(fmt, bad):
    x = torch.randn(48, 80, device="cuda").to(BF16)
    x[17, 33] = bad
    amax = _ops().fp8_amax(x)
    assert math.isnan(float(amax)) if math.isnan(bad) else float(amax) == math.inf
    q, qt, si = _F8().quantize_tensorwise(x, fmt, rowwise=True, colwise=True)
    q_ref, qt_ref, si_ref = _F8().quantize_reference(x, fmt, rowwise=True, colwise=True)
    assert math.isnan(float(si))
    assert bool(q.float().isnan().all()) and bool(qt.float().isnan().all())
    assert_bytes_equal(q, q_ref, "q")
    assert_bytes_equal(qt, qt_ref, "qt")


def test_cast_refusals_write_nothing():
    from deepspeed_b200.ops import native as N
    NE = _NE()
    x = torch.randn(40, 64, device="cuda").to(BF16)
    amax = _ops().fp8_amax(x)
    qbuf = torch.full((64, 64), NAN8, dtype=torch.uint8, device="cuda")
    si = torch.full((1, ), 7.0, device="cuda")

    def cast(R=40, C=64, ld=64, amax_p=amax, fmt=N.F8E4M3, q=qbuf, ld_q=64, qt=None, ld_t=0, si_p=si):
        rc = N.cuda().dsb_fp8_cast(N.ptr(x), N.c_i64(R), N.c_i64(C), N.c_i64(ld), N.ptr(amax_p), fmt, N.ptr(q),
                                   N.c_i64(ld_q), N.ptr(qt), N.c_i64(ld_t), N.ptr(si_p), N.stream())
        N.check(rc, "fp8_cast")

    bad = [dict(R=0), dict(C=0), dict(ld=32), dict(amax_p=None), dict(si_p=None), dict(fmt=N.BF16), dict(q=None),
           dict(ld_q=48), dict(q=qbuf.view(-1)[8:]), dict(q=None, qt=qbuf, ld_t=48),  # R % 16
           dict(R=32, q=None, qt=qbuf, ld_t=40), dict(R=32, q=None, qt=qbuf, ld_t=16),
           dict(R=32, q=None, qt=qbuf.view(-1)[8:], ld_t=64)]
    for kw in bad:
        with pytest.raises(NE, match="unsupported shape"):
            cast(**kw)
    torch.cuda.synchronize()
    assert bool((qbuf == NAN8).all()) and float(si) == 7.0
    with pytest.raises(NE):
        N.check(N.cuda().dsb_fp8_amax(N.ptr(x), N.c_i64(40), N.c_i64(64), N.c_i64(32), N.ptr(amax), N.stream()), "amax")
    with pytest.raises(NE):
        _ops().fp8_cast(x.float(), amax, E4M3)


# ---------------------------------------------------------------------------------------------------------------------
# 2. FP8 GEMM, exact oracle
# ---------------------------------------------------------------------------------------------------------------------
def f8_grid(rows, cols, fmt, gen, emin=-3, emax=3, lo=-4, hi=4):
    """fp8 ``[rows, cols]``: integers in ``[lo, hi]`` times ``2**e_r`` (one exponent per row), exact in both formats."""
    v = torch.randint(lo, hi + 1, (rows, cols), generator=gen, device="cuda", dtype=torch.int32).float()
    e = torch.randint(emin, emax + 1, (rows, ), generator=gen, device="cuda", dtype=torch.int32)
    return torch.ldexp(v, e[:, None]).to(fmt), e


def pow2(e):
    return torch.tensor([2.0**e], dtype=torch.float32, device="cuda")


def exact_c(a, b, sa, sb, c_old=None):
    ref = (a.double() @ b.double().t()) * (float(sa) * float(sb))
    if c_old is not None:
        ref = ref + c_old.double()
    return ref


def guarded_c(M, N):
    buf = torch.full((M + 16, N + 24), float("nan"), dtype=BF16, device="cuda")
    return buf, buf[8:8 + M, 8:8 + N]


def guard_intact_c(buf, view):
    mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    r0 = (view.data_ptr() - buf.data_ptr()) // (2 * buf.stride(0))
    c0 = (view.data_ptr() - buf.data_ptr()) // 2 % buf.stride(0)
    mask[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = False
    assert bool(buf[mask].isnan().all()), "elements outside the output were written"


GEMM_SHAPES = [(128, 128, 128), (1, 8, 16), (7, 24, 48), (200, 136, 400), (300, 520, 272), (513, 264, 1040)]


@pytest.mark.parametrize("afmt", [E4M3, E5M2], ids=["a_e4m3", "a_e5m2"])
@pytest.mark.parametrize("accum", [False, True], ids=["store", "accum"])
@pytest.mark.parametrize("shape", GEMM_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_exact(afmt, accum, shape):
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + 7 * N + 13 * K + int(accum))
    a_val, ea = f8_grid(M, K, afmt, g)
    b_val, eb = f8_grid(N, K, E4M3, g)
    abuf, a = guarded_f8(M, K, afmt)
    bbuf, b = guarded_f8(N, K, E4M3)
    a.copy_(a_val)
    b.copy_(b_val)
    sa, sb = pow2(-5), pow2(3)
    cbuf, c = guarded_c(M, N)
    c_old = None
    if accum:
        v = torch.randint(-128, 129, (M, N), generator=g, device="cuda").float()
        c_old = (torch.ldexp(v, ea[:, None] + eb[None, :]) * (2.0**-2)).to(BF16)
        c.copy_(c_old)
    K_ = _K()
    K_.fp8_matmul(a, b, sa, sb, out=c, epi=K_.EPI_ACCUM if accum else K_.EPI_STORE)
    assert_bits_equal(c, exact_c(a_val, b_val, sa, sb, c_old).to(BF16), "C")
    guard_intact_c(cbuf, c)


@pytest.mark.parametrize("afmt", [E4M3, E5M2], ids=["a_e4m3", "a_e5m2"])
def test_gemm_large_k_needs_promotion(afmt):
    """K = 16384 of positive products: row sums reach 2**16-2**17, so every partial sum past 2**14 must keep its low bits.
    The kernel is exact; cuBLAS's fast-accumulate FP8 GEMM (no promotion) on the same data is not."""
    M, N, K = 128, 256, 16384
    g = torch.Generator(device="cuda").manual_seed(5)
    a, _ = f8_grid(M, K, afmt, g, emin=0, emax=0, lo=1, hi=4)
    b, _ = f8_grid(N, K, E4M3, g, emin=0, emax=0, lo=1, hi=4)
    sa, sb = pow2(0), pow2(0)
    c = _K().fp8_matmul(a, b, sa, sb)
    ref = exact_c(a, b, sa, sb)
    assert float(ref.max()) > 2.0**16
    assert_bits_equal(c, ref.to(BF16), "C")
    # fp32-representable exactness: compare in fp32 as well (the bf16 rounding could hide small losses)
    c32 = torch._scaled_mm(a, b.t(), scale_a=sa, scale_b=sb, out_dtype=torch.float32, use_fast_accum=False)
    assert torch.equal(c32.double(), ref), "cuBLAS promoted accumulation is exact on this data"
    fast = torch._scaled_mm(a, b.t(), scale_a=sa, scale_b=sb, out_dtype=torch.float32, use_fast_accum=True)
    assert not torch.equal(fast.double(), ref), "this data would not tell an unpromoted accumulation apart"


@pytest.mark.parametrize("afmt", [E4M3, E5M2], ids=["a_e4m3", "a_e5m2"])
def test_gemm_equals_scaled_mm(afmt):
    M, N, K = 384, 256, 1024
    g = torch.Generator(device="cuda").manual_seed(9)
    a, _ = f8_grid(M, K, afmt, g)
    b, _ = f8_grid(N, K, E4M3, g)
    sa, sb = pow2(-4), pow2(-1)
    c = _K().fp8_matmul(a, b, sa, sb)
    ref = torch._scaled_mm(a, b.t(), scale_a=sa, scale_b=sb, out_dtype=BF16, use_fast_accum=False)
    assert_bits_equal(c, ref, "C vs torch._scaled_mm")


@pytest.mark.parametrize("shape", [(128, 64, 128), (200, 192, 400), (77, 128, 48)], ids=lambda s: "x".join(map(str, s)))
def test_gemm_swiglu_exact(shape):
    M, I, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + I + K)
    a, _ = f8_grid(M, K, E4M3, g)
    w, _ = f8_grid(2 * I, K, E4M3, g)
    sa, sb = pow2(-4), pow2(-2)
    cbuf, act = guarded_c(M, I)
    gbuf, gu = guarded_c(M, 2 * I)
    K_ = _K()
    K_.fp8_matmul(a, w, sa, sb, out=act, epi=K_.EPI_SWIGLU, out2=gu)
    ref = exact_c(a, w, sa, sb)
    assert_bits_equal(gu, ref.to(BF16), "gate|up")
    want, bound = swiglu_reference(ref[:, :I], ref[:, I:])
    assert_within(act, want, bound, "act")
    guard_intact_c(cbuf, act)
    guard_intact_c(gbuf, gu)


@pytest.mark.parametrize("shape", [(128, 128, 128), (200, 72, 400), (64, 520, 48)], ids=lambda s: "x".join(map(str, s)))
def test_gemm_dswiglu_exact(shape):
    M, I, K = shape
    g = torch.Generator(device="cuda").manual_seed(3 * M + I + K)
    a, _ = f8_grid(M, K, E5M2, g)
    w, _ = f8_grid(I, K, E4M3, g)
    sa, sb = pow2(-6), pow2(-3)
    gu = (torch.randn(M, 2 * I, generator=g, device="cuda") * 2).to(BF16)
    obuf, out2 = guarded_c(M, 2 * I)
    K_ = _K()
    K_.fp8_matmul(a, w, sa, sb, epi=K_.EPI_DSWIGLU, aux=gu, out2=out2)
    d = exact_c(a, w, sa, sb)
    dg, dg_b, du, du_b = dswiglu_reference(d, gu[:, :I], gu[:, I:], d_fp32=True)
    assert_within(out2[:, :I], dg, dg_b, "dgate")
    assert_within(out2[:, I:], du, du_b, "dup")
    guard_intact_c(obuf, out2)


@pytest.mark.parametrize("epi", ["store", "swiglu"])
def test_gemm_cta_counts_bit_identical(epi):
    """Random (inexact) data: 1-7 persistent CTAs and every rasterisation give the same bits."""
    M, N, K = 392, 384, 1008
    g = torch.Generator(device="cuda").manual_seed(11)
    a = (torch.randn(M, K, generator=g, device="cuda") * 8).to(E4M3)
    b = (torch.randn(N, K, generator=g, device="cuda") * 8).to(E4M3)
    sa, sb = pow2(-7), pow2(-6)
    K_ = _K()
    e = K_.EPI_SWIGLU if epi == "swiglu" else K_.EPI_STORE
    out2 = torch.empty(M, N, dtype=BF16, device="cuda") if epi == "swiglu" else None
    first = K_.fp8_matmul(a, b, sa, sb, epi=e, out2=out2)
    first2 = out2.clone() if out2 is not None else None
    if epi == "store":
        _bounded(first, a.double(), b.double(), 2.0**-13, "C random")
    for sms in range(1, 8):
        for gm in (0, 1, 3, 8):
            c = K_.fp8_matmul(a, b, sa, sb, epi=e, out2=out2, sms=sms, group_m=gm)
            assert_bits_equal(c, first, f"C sms={sms} group_m={gm}")
            if out2 is not None:
                assert_bits_equal(out2, first2, f"gate|up sms={sms} group_m={gm}")


def test_gemm_nan_scale_gives_nan():
    a = torch.ones(128, 64, device="cuda").to(E4M3)
    b = torch.ones(128, 64, device="cuda").to(E4M3)
    c = _K().fp8_matmul(a, b, torch.tensor([float("nan")], device="cuda"), pow2(0))
    assert bool(c.isnan().all())


def test_gemm_refusals_write_nothing():
    """Every -2 condition of ``dsb_gemm_fp8`` raises NativeOpError and leaves C untouched."""
    from deepspeed_b200.ops import native as N
    NE = _NE()
    abuf = torch.ones(256, 256, device="cuda").to(E4M3)
    a5 = torch.ones(256, 256, device="cuda").to(E5M2)
    cbuf = torch.full((256, 256), float("nan"), dtype=BF16, device="cuda")
    aux = torch.zeros(256, 256, dtype=BF16, device="cuda")
    s = pow2(0)

    def call(a=abuf, b=abuf, c=cbuf, M=64, n=64, K=64, lda=256, ldb=256, ldc=256, fmt=N.F8E4M3, sa=s, sb=s, epi=0,
             aux_=None, ld_aux=0, out2=None, ld_out2=0):
        rc = N.cuda().dsb_gemm_fp8(N.ptr(a), N.ptr(b), N.ptr(c), M, n, K, lda, ldb, ldc, fmt, N.ptr(sa), N.ptr(sb), epi,
                                   N.ptr(aux_), ld_aux, N.ptr(out2), ld_out2, 8, 0, N.stream())
        N.check(rc, "gemm_fp8")

    cases = [
        dict(M=0), dict(n=0), dict(K=0), dict(K=24), dict(n=12), dict(lda=40), dict(ldb=40), dict(lda=48, K=64),
        dict(ldc=60), dict(ldc=32, n=64), dict(a=abuf.view(-1)[8:]), dict(b=abuf.view(-1)[8:]), dict(c=cbuf.view(-1)[4:]),
        dict(sa=None), dict(sb=None), dict(fmt=N.BF16), dict(fmt=N.F8E4M3 + 7), dict(epi=4), dict(epi=-1),
        dict(epi=2, a=a5, fmt=N.F8E5M2), dict(epi=2, n=72), dict(epi=3),  # DSWIGLU with an e4m3 A
        dict(epi=3, a=a5, fmt=N.F8E5M2, out2=cbuf, ld_out2=256), dict(epi=3, a=a5, fmt=N.F8E5M2, aux_=aux, ld_aux=256),
        dict(epi=3, a=a5, fmt=N.F8E5M2, aux_=aux, ld_aux=252, out2=cbuf, ld_out2=256),
        dict(epi=3, a=a5, fmt=N.F8E5M2, aux_=aux.view(-1)[4:], ld_aux=256, out2=cbuf, ld_out2=256),
    ]
    for kw in cases:
        with pytest.raises(NE, match="unsupported shape"):
            call(**kw)
    torch.cuda.synchronize()
    assert bool(cbuf.isnan().all()), "a refused call wrote C"
    call()  # the baseline arguments are accepted
    torch.cuda.synchronize()
    assert not bool(cbuf[:64, :64].isnan().any())
    # shapes that do not fit together are refused by the wrapper before any tensor map is built
    K_ = _K()
    for args in ((abuf[:, :64], abuf[:, :32]), (abuf.to(torch.float32)[:64, :64], abuf[:64, :64]),
                 (abuf[:64, :64], a5[:64, :64])):
        with pytest.raises(NE, match="do not fit"):
            K_.fp8_matmul(*args, s, s)
    with pytest.raises(NE, match="do not fit"):
        K_.fp8_matmul(a5[:64, :64], abuf[:64, :64], s, s, epi=K_.EPI_DSWIGLU)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the autograd nodes
# ---------------------------------------------------------------------------------------------------------------------
def _deq(t8):
    return t8.double()


# Inside one k-block the fp8 tensor core accumulates with fewer bits than fp32 (products aligned to the largest one, about
# 14 bits kept): on data that is not on a common small-integer grid, a block's partial sum errs by a small multiple of
# 2**-14 of its magnitudes (the worst these tests saw on an H100 80GB HBM3 at 700 W was 2**-13.0; they print it).  The
# blocks then add in fp32.  The bound allows 2**-11 for the blocks, plus the fp32 additions and the bf16 rounding.
FP8_BLOCK_REL = 2.0**-11


def fp8_gemm_bound(ref, mag, K):
    acc = FP8_BLOCK_REL * mag + 2 * (K // 128 + 1) * U * mag
    return ulp(ref.abs() + acc, BF16) + acc


worst = {}


def _bounded(got, a, b, s, what):
    """``got`` (bf16) within :func:`fp8_gemm_bound` of ``s * a @ b^T`` (float64 operands)."""
    ref = (a @ b.t()) * s
    mag = (a.abs() @ b.abs().t()) * s
    err = (got.double() - ref).abs() - ulp(ref.abs(), BF16)
    worst[what] = float((err / mag.clamp_min(1e-300)).max())
    print(f"[fp8 accumulation] {what}: worst |C - exact| beyond one bf16 ulp = 2**{math.log2(max(worst[what], 2**-60)):.1f} "
          f"of the magnitudes")
    assert_within(got, ref, fp8_gemm_bound(ref, mag, a.shape[1]), what)


def test_fp8_linear_node():
    from deepspeed_b200.ops.linear import fp8_linear
    F8 = _F8()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(2, 256, 512, generator=g, device="cuda").to(BF16).requires_grad_(True)
    w = (torch.randn(384, 512, generator=g, device="cuda") * 0.03).to(BF16).requires_grad_(True)
    dy = torch.randn(2, 256, 384, generator=g, device="cuda").to(BF16)
    y = fp8_linear(x, w)
    x8t, sx = y.grad_fn.saved_tensors
    y.backward(dy)
    x2, dy2 = x.detach().reshape(-1, 512), dy.reshape(-1, 384)
    x8r, x8tr, sxr = F8.quantize_reference(x2, E4M3, True, True)
    w8r, w8tr, swr = F8.quantize_reference(w.detach(), E4M3, True, True)
    dy8r, dy8tr, sdyr = F8.quantize_reference(dy2, E5M2, True, True)
    assert_bytes_equal(x8t, x8tr, "saved x^T")
    assert_bits_equal(sx, sxr, "saved scale_inv")
    _bounded(y.detach().reshape(-1, 384), _deq(x8r), _deq(w8r), float(sxr * swr), "y")
    _bounded(x.grad.reshape(-1, 512), _deq(dy8r), _deq(w8tr), float(sdyr * swr), "dx")
    _bounded(w.grad, _deq(dy8tr), _deq(x8tr), float(sdyr * sxr), "dw")


def test_fp8_swiglu_node_against_reference_path(monkeypatch):
    from deepspeed_b200.ops import linear
    F8 = _F8()
    g = torch.Generator(device="cuda").manual_seed(2)
    T, H, I = 512, 256, 384
    x0 = torch.randn(T, H, generator=g, device="cuda").to(BF16)
    wgu0 = (torch.randn(2 * I, H, generator=g, device="cuda") * H**-0.5).to(BF16)
    wd0 = (torch.randn(H, I, generator=g, device="cuda") * I**-0.5).to(BF16)
    dy = torch.randn(T, H, generator=g, device="cuda").to(BF16)

    def run():
        x, wgu, wd = (t.clone().requires_grad_(True) for t in (x0, wgu0, wd0))
        y = linear.fp8_swiglu_mlp(x, wgu, wd)
        saved = [t.clone() for t in y.grad_fn.saved_tensors]
        y.backward(dy)
        return y.detach(), x.grad, wgu.grad, wd.grad, saved

    y, dx, dwgu, dwd, (x8t, sx, gu, act8t, sa) = run()
    monkeypatch.setattr(linear, "_fp8_native", lambda *a, **k: False)
    y_r, dx_r, dwgu_r, dwd_r, (x8t_r, sx_r, gu_r, act8t_r, sa_r) = run()
    # the casts of the inputs are bit-equal to the torch reference
    assert_bytes_equal(x8t, x8t_r, "x^T")
    assert_bits_equal(sx, sx_r, "x scale_inv")
    wgu8 = F8.quantize_reference(wgu0, E4M3)
    wd8 = F8.quantize_reference(wd0, E4M3, True, True)
    dy8 = F8.quantize_reference(dy, E5M2, True, True)
    # gate|up and y: fp32 accumulations of the quantised operands
    _bounded(gu, _deq(x8t.t()), _deq(wgu8[0]), float(sx * wgu8[2]), "gate|up")
    _bounded(y, _deq(act8t.t()), _deq(wd8[0]), float(sa * wd8[2]), "y")
    _bounded(dwd, _deq(dy8[1]), _deq(act8t), float(dy8[2] * sa), "dW_down")
    # dX and dW_gate_up pass through the dSwiGLU epilogue (silu through __expf) and the e5m2 cast of its output, whose
    # rounding can flip where the reference path's torch.exp differs in the last bit: compare with the reference path
    for got, want, what in ((dx, dx_r, "dx"), (dwgu, dwgu_r, "dW_gate_up"), (y, y_r, "y vs reference path")):
        rel = float((got.float() - want.float()).norm() / want.float().norm())
        assert rel < 2e-2, (what, rel)


def _sync_free():
    from deepspeed_b200.ops.linear import fp8_linear, fp8_swiglu_mlp
    x = torch.randn(256, 256, device="cuda").to(BF16).requires_grad_(True)
    w = (torch.randn(512, 256, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    wd = (torch.randn(256, 256, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = fp8_swiglu_mlp(fp8_linear(x, wd), w, wd)
        y.sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for t in (x.grad, w.grad, wd.grad):
        assert bool(torch.isfinite(t).all()) and bool(t.any())


def test_fp8_nodes_make_no_host_sync():
    _sync_free()


def _first_backward_on_autograd_thread():
    from deepspeed_b200.ops.linear import fp8_linear, fp8_swiglu_mlp
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(256, 256, generator=g, device="cuda").to(BF16).requires_grad_(True)
    w = (torch.randn(768, 256, generator=g, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    wd = (torch.randn(256, 384, generator=g, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    wl = (torch.randn(256, 256, generator=g, device="cuda") * 0.05).to(BF16).requires_grad_(True)
    y = fp8_swiglu_mlp(fp8_linear(x, wl), w, wd)
    torch.cuda.synchronize()
    y.backward(torch.ones_like(y))
    for t in (x.grad, w.grad, wd.grad, wl.grad):
        assert t is not None and bool(torch.isfinite(t).all()) and bool(t.any())


def test_fp8_backward_first_on_autograd_thread():
    run_distributed(_first_backward_on_autograd_thread, 1, ())


# ---------------------------------------------------------------------------------------------------------------------
# 4. training
# ---------------------------------------------------------------------------------------------------------------------
def _llama(fp8, vocab=1024, **kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=vocab, num_hidden_layers=2, max_position_embeddings=512, fp8=fp8, **kw)
    with torch.device("cuda"):
        return LlamaForCausalLM(cfg).to(BF16)


def _engine(model, stage, lr=1e-3, gas=1):
    import deepspeed_b200 as ds
    cfg = {"train_micro_batch_size_per_gpu": 2, "gradient_accumulation_steps": gas, "bf16": {"enabled": True},
           "optimizer": {"type": "AdamW", "params": {"lr": lr}}, "zero_optimization": {"stage": stage}}
    engine, _, _, _ = ds.initialize(model=model, config=cfg)
    return engine


def _fp8_llama_zero3():
    from deepspeed_b200.ops import native
    engine = _engine(_llama(True, checkpoint_layers=1), 3, gas=2)
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


def test_fp8_llama_trains_zero3():
    run_distributed(_fp8_llama_zero3, 1, ())


# Final-loss gap, FP8 minus bf16, on the bigram stream below (mean of the last 10 of 120 steps).  Measured on an H100
# 80GB HBM3 at 700 W: bf16 3.0230, FP8 3.0540, gap +0.031 (entropy floor 2.535).  The bound is about 3x that.
CONVERGENCE_GAP = 0.1


def _bigram_batches(steps, vocab=256, B=2, S=256, seed=0):
    """Token streams from a fixed random bigram table (each token has a few likely successors): learnable, with a known
    entropy floor."""
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(vocab, vocab, generator=g) * 3
    probs = torch.softmax(logits, -1)
    floor = float(-(probs * probs.log()).sum(-1).mean())
    out = []
    for _ in range(steps):
        ids = torch.empty(B, S, dtype=torch.long)
        ids[:, 0] = torch.randint(0, vocab, (B, ), generator=g)
        for t in range(1, S):
            ids[:, t] = torch.multinomial(probs[ids[:, t - 1]], 1, generator=g).squeeze(1)
        out.append(ids)
    return out, floor


def _convergence():
    batches, floor = _bigram_batches(120)
    finals = {}
    for fp8 in (False, True):
        engine = _engine(_llama(fp8, vocab=256), 3, lr=2e-3)
        losses = []
        for ids in batches:
            ids = ids.cuda()
            loss = engine(ids, labels=ids)
            engine.backward(loss)
            engine.step()
            losses.append(float(loss))
        finals[fp8] = sum(losses[-10:]) / 10
        del engine
    gap = finals[True] - finals[False]
    print(f"[fp8 convergence] bf16 {finals[False]:.4f} fp8 {finals[True]:.4f} gap {gap:+.4f} entropy floor {floor:.4f}")
    assert finals[False] < math.log(256) - 1.0, finals  # both runs learned the bigrams
    assert abs(gap) <= CONVERGENCE_GAP, (finals, gap)


def test_fp8_convergence_matches_bf16():
    run_distributed(_convergence, 1, (), timeout=600)
