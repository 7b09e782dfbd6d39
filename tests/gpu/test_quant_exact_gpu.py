"""The group quantization kernels of ``csrc/cuda/quant.cu`` per element against the exact emulations in
``tests/numerics.py``: int8/int4 quantize / dequantize (ZeRO++ qwZ, qgZ), the qgZ dequantize-reduce-requantize, LoCo
error feedback, MoQ fake quantization and the FP8/FP6/FP4/FP12 codec.  Codes, scales, offsets, error buffers and
dequantized values must be bit-exact; every output is written into a buffer with sentinel guard bands."""
import ctypes
import types

import numpy as np
import pytest
import torch

from tests import numerics as R
from deepspeed_b200.ops import native as N
from deepspeed_b200.ops.quantizer import quantizer as Q

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
FORMS = [(4, True), (4, False), (8, True), (8, False)]
GUARD = 256


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


class Guarded:
    """``n`` elements inside a sentinel-filled buffer with ``GUARD`` elements on each side."""

    def __init__(self, n, dtype, sentinel=None):
        if sentinel is None:
            sentinel = 0x5A if dtype in (torch.int8, torch.uint8) else -1234.5
        self.buf = torch.full((n + 2 * GUARD, ), sentinel, dtype=dtype, device="cuda")
        self.ref = self.buf.clone()
        self.t = self.buf[GUARD:GUARD + n]

    def guards_intact(self):
        torch.cuda.synchronize()
        return torch.equal(self.buf[:GUARD], self.ref[:GUARD]) and torch.equal(self.buf[-GUARD:], self.ref[-GUARD:])

    def untouched(self):
        torch.cuda.synchronize()
        return torch.equal(self.buf, self.ref)


def _same(out, ref, what):
    """Bit-equal, except that a NaN only has to meet a NaN: the contract for a non-finite group is its NaNs, not their
    payloads."""
    if out.dtype.is_floating_point:
        nan = torch.isnan(out.float())
        assert torch.equal(nan, torch.isnan(ref.float())), f"{what}: NaNs in different places"
        out, ref = out.masked_fill(nan, 0), ref.masked_fill(nan, 0)
    R.assert_bits_equal(out, ref, what)


def _i(v):
    return ctypes.c_int64(v)


def quantize(x, groups, bits, sym, perm=None, stochastic=False, seed=0):
    n = x.numel()
    q = Guarded(n if bits == 8 else n // 2, torch.int8)
    p = Guarded(groups * (1 if sym else 2), torch.float32)
    rc = N.cuda().dsb_quantize(P(x), P(q.t), P(p.t), _i(groups), n // groups, bits, int(sym), N.dt(x), P(perm),
                               int(stochastic), ctypes.c_uint32(seed), N.stream())
    N.check(rc, "quantize")
    assert q.guards_intact() and p.guards_intact()
    return q.t, p.t


def dequantize(q, params, groups, bits, sym, dtype):
    n = q.numel() * (1 if bits == 8 else 2)
    out = Guarded(n, dtype)
    rc = N.cuda().dsb_dequantize(P(q), P(params), P(out.t), _i(groups), n // groups, bits, int(sym), N.dt(out.t),
                                 N.stream())
    N.check(rc, "dequantize")
    assert out.guards_intact()
    return out.t


def _codes_params(x, groups, bits, sym):
    codes, scale, offset = R.int_quant_reference(x, groups, bits, sym)
    packed = torch.from_numpy(R.pack_int(codes, bits, sym)).reshape(-1)
    params = torch.from_numpy(scale if sym else np.stack([scale, offset], 1).reshape(-1))
    return codes, scale, offset, packed, params


def _assert_quant(x, groups, bits, sym, q, p, what):
    codes, scale, offset, packed, params = _codes_params(x.cpu(), groups, bits, sym)
    _same(q.cpu(), packed, f"{what} codes")
    _same(p.cpu(), params, f"{what} params")
    return codes, scale, offset


def _deq_ref(codes, scale, offset, dtype):
    return torch.from_numpy(R.int_dequant_reference(codes, scale, offset)).to(dtype).reshape(-1)


# ---- quantize / dequantize --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gs", [8, 16, 2040, 2048, 2056, "cap"])
@pytest.mark.parametrize("bits,sym", FORMS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_quantize_dequantize_exact(dtype, bits, sym, gs):
    """One vector per thread (8, 16), partial last passes (2040, 2056), every register slot (the 8192 16-bit and 4096
    fp32 caps), with ties, +-amax, constant / zero / negative-only / tiny / huge groups."""
    if gs == "cap":
        gs = 4096 if dtype == torch.float32 else 8192
    gen = torch.Generator().manual_seed(gs + bits + 100 * sym)
    groups = 9
    x = R.quant_cases(groups, gs, dtype, bits, sym, gen).cuda()
    q, p = quantize(x, groups, bits, sym)
    codes, scale, offset = _assert_quant(x, groups, bits, sym, q, p, "quantize")
    out = dequantize(q, p, groups, bits, sym, dtype)
    _same(out.cpu(), _deq_ref(codes, scale, offset, dtype), "dequantize")


@pytest.mark.parametrize("groups,gs", [(1, 8), (100_000, 8), (3000, 40)])
@pytest.mark.parametrize("bits,sym", FORMS)
def test_quantize_group_counts(groups, gs, bits, sym):
    gen = torch.Generator().manual_seed(groups)
    x = R.quant_cases(groups, gs, torch.bfloat16, bits, sym, gen).cuda()
    q, p = quantize(x, groups, bits, sym)
    codes, scale, offset = _assert_quant(x, groups, bits, sym, q, p, "quantize")
    out = dequantize(q, p, groups, bits, sym, torch.bfloat16)
    _same(out.cpu(), _deq_ref(codes, scale, offset, torch.bfloat16), "dequantize")


def test_four_bit_nibble_order_and_sign_extension():
    """Codes -8..7 at known positions: element 2i is the low nibble of byte i, and a set bit 3 reads back negative."""
    k = torch.arange(-8, 8, dtype=torch.float32).repeat(2)  # amax 8 -> scale 1, +8 absent so codes are k themselves
    x = k.clone()
    x[0] = -8.0
    q, p = quantize(x.cuda(), 1, 4, True)
    assert float(p.cpu()[0]) == 1.0
    b = q.cpu().view(torch.uint8).to(torch.int32)
    lo, hi = b & 0xF, b >> 4
    assert torch.equal(lo, (k[0::2].to(torch.int32) & 0xF)) and torch.equal(hi, (k[1::2].to(torch.int32) & 0xF))
    out = dequantize(q, p, 1, 4, True, torch.float32)
    assert torch.equal(out.cpu(), k)


@pytest.mark.parametrize("nodes,devs", [(1, 8), (2, 4), (4, 2)])
@pytest.mark.parametrize("bits", [4, 8])
def test_swizzled_quantize_places_groups_by_perm(nodes, devs, bits):
    gen = torch.Generator().manual_seed(nodes)
    groups, gs = 8 * 6, 64
    x = R.quant_cases(groups, gs, torch.bfloat16, bits, True, gen).cuda()
    perm = Q.swizzle_perm(groups, nodes, devs, "cuda")
    q, p = quantize(x, groups, bits, True, perm=perm)
    _, _, _, packed, params = _codes_params(x.cpu(), groups, bits, True)
    inv = torch.empty(groups, dtype=torch.long)
    inv[perm.cpu().long()] = torch.arange(groups)
    _same(q.cpu().view(groups, -1), packed.view(groups, -1)[inv], "swizzled codes")
    _same(p.cpu(), params[inv], "swizzled scales")
    assert sorted(perm.cpu().tolist()) == list(range(groups))


def test_dequantize_beyond_int32_indexes():
    """int8 codes to bf16 over more than 2^31 elements: the flat index must be 64-bit."""
    gs = 2048
    groups = 2**31 // gs + 3
    q = torch.randint(-128, 128, (groups * gs, ), dtype=torch.int8, device="cuda")
    s = torch.rand(groups, device="cuda") + 0.5
    out = dequantize(q, s, groups, 8, True, torch.bfloat16)
    for lo in (0, 2**31 - gs, groups * gs - 3 * gs):  # the first group, across 2^31, the last groups
        want = (q[lo:lo + 3 * gs].float().view(3, gs) * s[lo // gs:lo // gs + 3, None]).bfloat16().reshape(-1)
        assert torch.equal(out[lo:lo + 3 * gs], want), lo
    del out, q


# ---- dequant-reduce (qgZ) ---------------------------------------------------------------------------------------------
def dequant_reduce(q, params, peers, out_groups, gs, bits, sym, err=None, beta=0.0):
    oq = Guarded(out_groups * gs // (1 if bits == 8 else 2), torch.int8)
    op = Guarded(out_groups * (1 if sym else 2), torch.float32)
    rc = N.cuda().dsb_dequant_reduce(P(q), P(params), P(oq.t), P(op.t), peers, out_groups, gs, bits, int(sym), P(err),
                                     ctypes.c_float(beta), N.stream())
    N.check(rc, "dequant_reduce")
    assert oq.guards_intact() and op.guards_intact()
    return oq.t, op.t


@pytest.mark.parametrize("with_err", [False, True])
@pytest.mark.parametrize("bits,sym", FORMS)
@pytest.mark.parametrize("peers", [2, 4, 8])
def test_dequant_reduce_exact(peers, bits, sym, with_err):
    gen = torch.Generator().manual_seed(peers * 7 + bits)
    out_groups, gs = 7, 2048
    x = torch.randn(peers, out_groups, gs, generator=gen) * torch.exp2(torch.randint(-8, 8, (peers, out_groups, 1),
                                                                                       generator=gen).float())
    # one peer's NaN or inf, at the first, a middle or the last position, makes that output group non-finite
    x[1, 3, 17], x[0, 4, 0], x[peers - 1, 6, -1] = float("nan"), float("inf"), -float("inf")
    x[:, 5] = x[:, 5] / x[:, 5].abs().max() * 1e-38  # tiny: 1/scale overflows in every peer and in the sum
    x[:, 5, ::3] = 0.0
    bad = [3, 4, 6]
    codes, scale, offset, packed, params = _codes_params(x.reshape(-1), peers * out_groups, bits, sym)
    err = (torch.randn(out_groups * gs, generator=gen) * 0.01) if with_err else None
    derr = err.cuda() if with_err else None
    oq, op = dequant_reduce(packed.cuda(), params.cuda(), peers, out_groups, gs, bits, sym, derr, 0.7)
    c2, s2, o2, new = R.reduce_reference(codes, scale, offset, peers, bits, sym, err, 0.7)
    _same(oq.cpu(), torch.from_numpy(R.pack_int(c2, bits, sym)).reshape(-1), "codes")
    want_p = s2 if sym else np.stack([s2, o2], 1).reshape(-1)
    _same(op.cpu(), torch.from_numpy(want_p), "params")
    assert np.isnan(s2[bad]).all() and np.isfinite(np.delete(s2, bad)).all()
    if sym and not with_err:
        assert (c2[5, ::3] == 0).all()  # the tiny group's zeros stay zero
    if with_err:
        _same(derr.cpu(), torch.from_numpy(new).reshape(-1), "error buffer")
        assert torch.equal(derr.cpu().view(out_groups, gs)[bad], err.view(out_groups, gs)[bad])


def test_dequant_reduce_shared_memory_limit():
    """12288 fp32 accumulators fill the 48 KB of dynamic shared memory: accepted and exact; 12290 is refused."""
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(2 * 12288, generator=gen)
    codes, scale, offset, packed, params = _codes_params(x, 2, 8, True)
    oq, op = dequant_reduce(packed.cuda(), params.cuda(), 2, 1, 12288, 8, True)
    c2, s2, _, _ = R.reduce_reference(codes, scale, offset, 2, 8, True)
    _same(oq.cpu(), torch.from_numpy(R.pack_int(c2, 8, True)).reshape(-1), "codes")
    _same(op.cpu(), torch.from_numpy(s2), "scale")
    q = torch.zeros(2 * 12290, dtype=torch.int8, device="cuda")
    oq, op = Guarded(12290, torch.int8), Guarded(1, torch.float32)
    with pytest.raises(N.NativeOpError):
        N.check(N.cuda().dsb_dequant_reduce(P(q), P(torch.ones(2, device="cuda")), P(oq.t), P(op.t), 2, 1, 12290, 8, 1,
                                            P(None), ctypes.c_float(0.0), N.stream()), "dequant_reduce")
    assert oq.untouched() and op.untouched()


# ---- LoCo ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("reset", [False, True])
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_loco_quantize_exact(dtype, bits, reset):
    """Codes, scales and the error update bit-exact; a group holding a NaN or an inf keeps its error slice."""
    gen = torch.Generator().manual_seed(bits)
    groups, gs = 37, 2048
    x = R.quant_cases(groups, gs, dtype, bits, True, gen).view(groups, gs)
    x[10, 0], x[11, gs // 2], x[12, -1] = float("nan"), float("inf"), -float("inf")
    err0 = torch.randn(groups * gs, generator=gen) * 0.05
    err0.view(groups, gs)[4] *= 1e-38  # keep the tiny group tiny
    err = Guarded(groups * gs, torch.float32)
    err.t.copy_(err0)
    err.ref[GUARD:GUARD + groups * gs].copy_(err0)
    q = Guarded(groups * gs // (1 if bits == 8 else 2), torch.int8)
    p = Guarded(groups, torch.float32)
    xd = x.cuda().reshape(-1).contiguous()
    rc = N.cuda().dsb_loco_quantize(P(xd), P(err.t), P(q.t), P(p.t), _i(groups), gs,
                                    bits, N.dt(x), ctypes.c_float(0.8), int(reset), N.stream())
    N.check(rc, "loco_quantize")
    assert err.guards_intact() and q.guards_intact() and p.guards_intact()
    codes, scale, new = R.loco_reference(x, err0, groups, bits, 0.8, reset)
    _same(q.t.cpu(), torch.from_numpy(R.pack_int(codes, bits, True)).reshape(-1), "codes")
    _same(p.t.cpu(), torch.from_numpy(scale), "scales")
    _same(err.t.cpu(), torch.from_numpy(new).reshape(-1), "error buffer")
    assert torch.equal(err.t.cpu().view(groups, gs)[10:13], err0.view(groups, gs)[10:13])


# ---- fake quantization (MoQ) -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sym", [True, False])
@pytest.mark.parametrize("bits", list(range(2, 17)))
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fake_quantize_exact(dtype, bits, sym):
    gen = torch.Generator().manual_seed(bits)
    groups, gs = 8, 1024
    x = R.quant_cases(groups, gs, dtype, min(bits, 8), sym, gen).view(groups, gs)
    x[7, 5] = float("nan")
    y = x.cuda().reshape(-1).contiguous()
    rc = N.cuda().dsb_fake_quantize(P(y), _i(groups), gs, bits, int(sym), N.dt(y), 0, ctypes.c_uint32(0), N.stream())
    N.check(rc, "fake_quantize")
    codes, scale, offset = R.int_quant_reference(x, groups, bits, sym)
    _same(y.cpu(), _deq_ref(codes, scale, offset, dtype), "fake_quantize")
    assert torch.isnan(y.view(groups, gs)[7].float()).all()


# ---- minifloat codec -------------------------------------------------------------------------------------------------------
def fp_quantize(x, groups, fmt, stochastic=False, seed=0):
    bits, m = R.FP_FORMATS[fmt]
    gs = x.numel() // groups
    bpg = (gs * bits + 7) // 8
    q = Guarded(groups * bpg, torch.uint8)
    s = Guarded(groups, torch.float32)
    rc = N.cuda().dsb_fp_quantize(P(x), P(q.t), P(s.t), _i(groups), gs, bits, m, N.dt(x), int(stochastic),
                                  ctypes.c_uint32(seed), N.stream())
    N.check(rc, "fp_quantize")
    assert q.guards_intact() and s.guards_intact()
    return q.t, s.t


def fp_dequantize(q, scales, out_groups, gs, fmt, dtype, rows=None, groups_per_row=1):
    bits, m = R.FP_FORMATS[fmt]
    out = Guarded(out_groups * gs, dtype)
    rc = N.cuda().dsb_fp_dequantize(P(q), P(scales), P(out.t), _i(out_groups), gs, bits, m, N.dt(out.t), P(rows),
                                    groups_per_row, N.stream())
    N.check(rc, "fp_dequantize")
    assert out.guards_intact()
    return out.t


@pytest.mark.parametrize("gs", [4, 12, 100, 132, 1028, 4096])
@pytest.mark.parametrize("fmt", list(R.FP_FORMATS))
def test_fp_quantize_dequantize_exact(fmt, gs):
    """Codes packed little-endian across byte boundaries, the lane tail (group sizes that are not a multiple of
    32 lanes x codes per lane), scales and dequantized values, bit-exact, fp32 and bf16 inputs."""
    bits, _ = R.FP_FORMATS[fmt]
    gen = torch.Generator().manual_seed(gs)
    groups = 6
    for dtype in (torch.float32, torch.bfloat16):
        x = R.fp_cases(fmt, groups, gs, gen).to(dtype)
        q, s = fp_quantize(x.cuda(), groups, fmt)
        codes, scale = R.fp_quant_reference(x, groups, fmt)
        _same(s.cpu(), torch.from_numpy(scale), f"{fmt} scales")
        _same(q.cpu(), torch.from_numpy(R.pack_bits(codes, bits)).reshape(-1), f"{fmt} codes")
        out = fp_dequantize(q, s, groups, gs, fmt, torch.bfloat16)
        want = torch.from_numpy(R.fp_dequant_reference(codes, scale, fmt)).bfloat16().reshape(-1)
        _same(out.cpu(), want, f"{fmt} dequantize")
        assert (out.view(groups, gs)[1] == 0).all() and (out.view(groups, gs)[2, ::3] == 0).all()


@pytest.mark.parametrize("fmt", list(R.FP_FORMATS))
def test_fp_selective_dequantize_rows(fmt):
    """Repeated and out-of-order row indexes, two groups per row."""
    gen = torch.Generator().manual_seed(3)
    rows_n, gpr, gs = 6, 2, 64
    x = torch.randn(rows_n * gpr * gs, generator=gen)
    q, s = fp_quantize(x.cuda(), rows_n * gpr, fmt)
    rows = torch.tensor([4, 0, 4, 5, 1, 1], dtype=torch.int32)
    out = fp_dequantize(q, s, rows.numel() * gpr, gs, fmt, torch.float32, rows=rows.cuda(), groups_per_row=gpr)
    codes, scale = R.fp_quant_reference(x, rows_n * gpr, fmt)
    full = torch.from_numpy(R.fp_dequant_reference(codes, scale, fmt)).reshape(rows_n, -1)
    _same(out.cpu(), full[rows.long()].reshape(-1), "selective dequantize")


# ---- stochastic rounding ------------------------------------------------------------------------------------------------
def _stoch_check(draws, lo, hi, target, what):
    """Every draw is one of the two neighbours ``lo``/``hi`` of ``target`` (all in the same units), and the mean over
    the draws (rows) is within 6 binomial standard deviations of ``target``."""
    n = draws.shape[0]
    assert ((draws == lo) | (draws == hi)).all(), f"{what}: a draw is not a neighbour"
    p = np.where(hi > lo, (target - lo) / np.where(hi > lo, hi - lo, 1), 0.0)
    sd = (hi - lo) * np.sqrt(p * (1 - p) / n)
    dev = np.abs(draws.mean(0) - target)
    assert (dev <= 6 * sd + 1e-12 * np.abs(target)).all(), \
        f"{what}: mean off by {dev.max():.3g} (worst {(dev / np.maximum(sd, 1e-300)).max():.1f} sigma)"


DRAWS = 4096


def test_stochastic_int_quantize_and_fake_quantize():
    gen = torch.Generator().manual_seed(0)
    gs = 64
    base = torch.randn(gs, generator=gen)
    base[0] = 4.0  # amax 4 -> int4 scale 0.5
    x = base.repeat(DRAWS).cuda()
    q, p = quantize(x, DRAWS, 4, True, stochastic=True, seed=11)
    q2, _ = quantize(x, DRAWS, 4, True, stochastic=True, seed=11)
    q3, _ = quantize(x, DRAWS, 4, True, stochastic=True, seed=12)
    assert torch.equal(q, q2) and not torch.equal(q, q3)
    out = dequantize(q, p, DRAWS, 4, True, torch.float32).cpu().view(DRAWS, gs).double().numpy() / 0.5
    t = (base.double().numpy() / 0.5)
    _stoch_check(out, np.clip(np.floor(t), -8, 7), np.clip(np.floor(t) + 1, -8, 7), np.minimum(t, 7), "int4 quantize")
    y = x.clone()
    N.check(N.cuda().dsb_fake_quantize(P(y), _i(DRAWS), gs, 4, 1, N.dt(y), 1, ctypes.c_uint32(5), N.stream()), "fq")
    _stoch_check(y.cpu().view(DRAWS, gs).double().numpy() / 0.5, np.clip(np.floor(t), -8, 7),
                 np.clip(np.floor(t) + 1, -8, 7), np.minimum(t, 7), "fake_quantize")


@pytest.mark.parametrize("fmt", list(R.FP_FORMATS))
def test_stochastic_fp_quantize(fmt):
    """Values across the format, its subnormal band and exact grid values at binade boundaries (which must come back
    unchanged): each draw is a neighbour, the mean is unbiased, seeds reproduce."""
    gen = torch.Generator().manual_seed(1)
    vals, _ = R.fp_grid(fmt)
    fmax = vals[-1]
    sub = vals[1:int(np.searchsorted(vals, vals[1] * 2**R.FP_FORMATS[fmt][1]))]  # the subnormal band
    gs = 128
    pick = np.concatenate([vals[-1:], vals[np.searchsorted(vals, 2.0**np.arange(-3, 3))],  # exact powers of two
                           np.linspace(0, sub[-1] * 1.3, 40)[1:],  # subnormal band and just above
                           np.random.default_rng(0).uniform(0, fmax, gs)])[:gs].astype(np.float32)
    pick[1::2] *= -1
    pick[0] = fmax
    base = torch.from_numpy(pick)
    x = base.repeat(DRAWS).cuda()
    q, s = fp_quantize(x, DRAWS, fmt, stochastic=True, seed=3)
    q2, _ = fp_quantize(x, DRAWS, fmt, stochastic=True, seed=3)
    q3, _ = fp_quantize(x, DRAWS, fmt, stochastic=True, seed=4)
    assert torch.equal(q, q2) and not torch.equal(q, q3)
    assert float(s[0]) == 1.0
    out = fp_dequantize(q, s, DRAWS, gs, fmt, torch.float32).cpu().view(DRAWS, gs).double().numpy()
    a = np.abs(pick.astype(np.float64))
    i = np.clip(np.searchsorted(vals, a, side="right") - 1, 0, len(vals) - 1)
    lo = vals[i]
    hi = np.where(lo == a, lo, vals[np.minimum(i + 1, len(vals) - 1)])
    sign = np.where(pick < 0, -1.0, 1.0)
    _stoch_check(out * sign, lo, hi, a, fmt)


# ---- non-finite groups ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", ["nan", "inf", "-inf"])
def test_nonfinite_group_dequantizes_nonfinite_in_every_kernel(bad):
    """A NaN or an inf at the first, a middle and the last position of a group: that group comes back all NaN and its
    scale is NaN, in every kernel; the neighbouring groups stay bit-exact."""
    v = float(bad)
    gen = torch.Generator().manual_seed(0)
    groups, gs = 6, 256
    x = (torch.randn(groups, gs, generator=gen)).to(torch.bfloat16)
    x[1, 0], x[3, gs // 2], x[5, -1] = v, v, v
    bad_g = [1, 3, 5]
    for bits, sym in FORMS:
        q, p = quantize(x.cuda().reshape(-1), groups, bits, sym)
        codes, scale, offset = _assert_quant(x.reshape(-1), groups, bits, sym, q, p, f"quantize {bits} {sym}")
        out = dequantize(q, p, groups, bits, sym, torch.float32).cpu().view(groups, gs)
        assert torch.isnan(out[bad_g]).all() and torch.isfinite(out[[0, 2, 4]]).all()
        assert np.isnan(scale[bad_g]).all()
    for bits in (2, 8, 16):
        y = x.cuda().reshape(-1).contiguous()
        N.check(N.cuda().dsb_fake_quantize(P(y), _i(groups), gs, bits, 1, N.dt(y), 0, ctypes.c_uint32(0), N.stream()), "fq")
        codes, scale, offset = R.int_quant_reference(x, groups, bits, True)
        _same(y.cpu(), _deq_ref(codes, scale, offset, torch.bfloat16), "fake_quantize")
        assert torch.isnan(y.view(groups, gs)[bad_g].float()).all()
    for fmt in R.FP_FORMATS:
        q, s = fp_quantize(x.cuda().reshape(-1), groups, fmt)
        out = fp_dequantize(q, s, groups, gs, fmt, torch.float32).cpu().view(groups, gs)
        assert torch.isnan(out[bad_g]).all() and torch.isnan(s.cpu()[bad_g]).all(), fmt
        codes, scale = R.fp_quant_reference(x.reshape(-1), groups, fmt)
        want = torch.from_numpy(R.fp_dequant_reference(codes, scale, fmt))
        _same(out[[0, 2, 4]], want[[0, 2, 4]], f"{fmt} neighbours")


@pytest.mark.parametrize("bits", [4, 8])
def test_asymmetric_range_beyond_fp32_is_nonfinite(bits):
    """Finite values whose asymmetric range hi - lo overflows fp32 (+-3e38): no finite scale spans them, so the group is
    treated like a non-finite one (NaN scale, all NaN) in quantize and fake quantize; its neighbours stay exact."""
    gen = torch.Generator().manual_seed(bits)
    groups, gs = 3, 64
    x = torch.randn(groups, gs, generator=gen)
    x[1, 0], x[1, -1] = 3e38, -3e38
    q, p = quantize(x.cuda().reshape(-1), groups, bits, False)
    codes, scale, offset = _assert_quant(x.reshape(-1), groups, bits, False, q, p, "quantize")
    out = dequantize(q, p, groups, bits, False, torch.float32).cpu().view(groups, gs)
    assert np.isnan(scale[1]) and torch.isnan(out[1]).all() and torch.isfinite(out[[0, 2]]).all()
    _same(out.reshape(-1), _deq_ref(codes, scale, offset, torch.float32), "dequantize")
    y = x.cuda().reshape(-1).contiguous()
    N.check(N.cuda().dsb_fake_quantize(P(y), _i(groups), gs, bits, 0, N.dt(y), 0, ctypes.c_uint32(0), N.stream()), "fq")
    _same(y.cpu(), _deq_ref(codes, scale, offset, torch.float32), "fake_quantize")


# ---- refusals --------------------------------------------------------------------------------------------------------------
def test_refused_arguments_raise_and_leave_outputs_untouched():
    x = torch.randn(1 << 16, device="cuda")
    xb = x.bfloat16()
    q, p = Guarded(1 << 16, torch.int8), Guarded(1 << 12, torch.float32)
    err = Guarded(1 << 16, torch.float32)

    def refused(rc):
        with pytest.raises(N.NativeOpError):
            N.check(rc, "refused")
        assert q.untouched() and p.untouched() and err.untouched()

    for t, gs, bits in [(x, 4100, 8), (x, 6, 8), (x, 8192, 8), (xb, 8200, 8), (xb, 12, 8), (xb, 16, 5), (xb, 16, 2)]:
        refused(N.cuda().dsb_quantize(P(t), P(q.t), P(p.t), _i(2), gs, bits, 1, N.dt(t), P(None), 0, ctypes.c_uint32(0),
                                      N.stream()))
        refused(N.cuda().dsb_loco_quantize(P(t), P(err.t), P(q.t), P(p.t), _i(2), gs, bits, N.dt(t),
                                           ctypes.c_float(0.8), 0, N.stream()))
    for bits in (1, 17):
        refused(N.cuda().dsb_fake_quantize(P(q.t), _i(2), 16, bits, 1, N.dt(xb), 0, ctypes.c_uint32(0), N.stream()))
    for gs, bits in [(15, 8), (12290, 8), (16, 6)]:
        refused(N.cuda().dsb_dequant_reduce(P(q.t), P(p.t), P(q.t), P(p.t), 2, 1, gs, bits, 1, P(None),
                                            ctypes.c_float(0.0), N.stream()))
    for bits, m, gs in [(5, 2, 16), (8, 4, 16), (6, 3, 16), (12, 2, 16), (8, 3, 18)]:
        refused(N.cuda().dsb_fp_quantize(P(x), P(q.t), P(p.t), _i(2), gs, bits, m, N.dt(x), 0, ctypes.c_uint32(0),
                                         N.stream()))
        refused(N.cuda().dsb_fp_dequantize(P(q.t), P(p.t), P(err.t), _i(2), gs, bits, m, N.dt(x), P(None), 1,
                                           N.stream()))
    refused(N.cuda().dsb_dequantize(P(q.t), P(p.t), P(err.t), _i(2), 16, 3, 1, N.dt(x), N.stream()))


# ---- ZeRO++ composition on one GPU ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("n", [3, 37, 1003, 4101, 2**20 + 5])
def test_qgz_exchange_and_reduce_per_rank(monkeypatch, world, n):
    """qgZ for ``world`` emulated ranks: ``_rank_chunks``, each rank's int4 ``quantize``, a receive buffer sliced from
    every sender's payload, ``_exchange_and_reduce`` with the all-to-all replaced by a copy of that buffer; each rank's
    slice equals the mean of the exactly dequantized chunks.  Rank 0 sends a NaN: the rank that owns that element gets
    NaN exactly across the quantization group around it, and every other element stays finite."""
    from deepspeed_b200.runtime.comm import coalesced_collectives as CC
    gen = torch.Generator().manual_seed(n + world)
    grads = [torch.randn(n, generator=gen).bfloat16() for _ in range(world)]
    i_nan = n // 2
    grads[0][i_nan] = float("nan")
    sent, ref_codes = [], []
    for g in grads:
        flat, per0, per, gs = CC._rank_chunks(g.cuda(), world)
        groups = (per // gs) * world
        q, p = Q.quantize(flat.contiguous(), groups, 4, Q.Symmetric)
        codes, scale, _, packed, params = _codes_params(flat.cpu(), groups, 4, True)
        _same(q.cpu(), packed, "rank payload")
        _same(p.cpu(), params, "rank scales")
        sent.append((q, p))
        ref_codes.append((codes, scale))
    gpr = per // gs  # groups per chunk
    for k in range(world):
        q_recv = torch.cat([q.view(world, -1)[k] for q, _ in sent])
        p_recv = torch.cat([p.view(world, -1)[k] for _, p in sent])
        calls = iter([q_recv, p_recv])
        monkeypatch.setattr(CC.dist, "all_to_all_single", lambda out, inp, group=None: out.copy_(next(calls)))
        got = CC._exchange_and_reduce(sent[k][0], sent[k][1], world, k, per0, per, gs, n, 4, torch.bfloat16, None)
        deq = np.stack([R.int_dequant_reference(c[k * gpr:(k + 1) * gpr], s[k * gpr:(k + 1) * gpr], None).reshape(-1)
                        for c, s in ref_codes])
        want = torch.from_numpy(deq).cuda().view(world, per).sum(0).div_(world)
        valid = max(0, min(per0, n - k * per0))
        _same(got, want[:valid].bfloat16(), f"rank {k}")
        nan = torch.zeros(valid, dtype=torch.bool)
        if k == i_nan // per0:
            g0 = (i_nan - k * per0) // gs
            nan[g0 * gs:(g0 + 1) * gs] = True
        assert torch.equal(torch.isnan(got.cpu()), nan) and torch.isfinite(got.cpu()[~nan]).all(), f"rank {k}"


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("n", [3, 37, 1003, 4101, 2**20 + 5])
def test_qwz_quantized_gather_per_rank(monkeypatch, world, n):
    """qwZ ``_quantized_gather`` with the all-gather replaced by the concatenation of every rank's payload: the other
    ranks' ranges are their exact int8 round trips, this rank's own range is its shard unchanged."""
    from deepspeed_b200.runtime.zero import sharded as S
    gen = torch.Generator().manual_seed(n)
    shards = [torch.randn(n, generator=gen).bfloat16().cuda() for _ in range(world)]
    gs = Q.aligned_group_size(n)
    padded = (n + gs - 1) // gs * gs
    payloads = [Q.quantize(torch.nn.functional.pad(s, (0, padded - n)), padded // gs, 8, Q.Symmetric) for s in shards]
    for r in range(world):
        calls = iter([torch.cat([q.reshape(-1) for q, _ in payloads]), torch.cat([p.reshape(-1) for _, p in payloads])])
        monkeypatch.setattr(S.dist, "all_gather_into_tensor", lambda out, inp, group=None: out.copy_(next(calls)))
        u = types.SimpleNamespace(shard_numel=n, shard_range=lambda rank: (rank * n, (rank + 1) * n))
        me = types.SimpleNamespace(shard_world=world, dp_group=None, shard_rank=r)
        full = torch.empty(world * n, dtype=torch.bfloat16, device="cuda")
        S.ZeroShardedOptimizer._quantized_gather(me, full, shards[r], u)
        for k in range(world):
            if k == r:
                assert torch.equal(full[k * n:(k + 1) * n], shards[r])
                continue
            src = torch.nn.functional.pad(shards[k].cpu(), (0, padded - n))
            codes, scale, _ = R.int_quant_reference(src, padded // gs, 8, True)
            want = torch.from_numpy(R.int_dequant_reference(codes, scale)).reshape(-1)[:n].bfloat16()
            _same(full[k * n:(k + 1) * n].cpu(), want, f"rank {r} sees rank {k}")
