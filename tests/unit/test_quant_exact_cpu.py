"""Host paths of the group quantizers (the CPU tier ZeRO++ runs on in most tests) against the exact references of
``tests/numerics.py``, self-checks of those references, and the group-size policy every caller must keep."""
import fractions

import numpy as np
import pytest
import torch

from tests import numerics as R
from deepspeed_b200.ops.quantizer import quantizer as Q
from deepspeed_b200.ops.fp_quantizer.quantize import FP_Quantize, _host_codec

DTYPES = [torch.bfloat16, torch.float16, torch.float32]


def _eq(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    same = (got == want) | (np.isnan(got) & np.isnan(want)) if got.dtype.kind == "f" else got == want
    if not same.all():
        k = int(np.flatnonzero(~same.reshape(-1))[0])
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.size} differ; first at {k}: "
                             f"got {got.reshape(-1)[k]!r}, want {want.reshape(-1)[k]!r}")


# ---- the references themselves ---------------------------------------------------------------------------------------
def test_minifloat_grids_match_known_constants():
    assert R.fp_max("e4m3") == 448.0 and R.fp_max("e5m2") == 57344.0 and R.fp_max("e3m2") == 28.0
    assert R.fp_max("e4m7") == 510.0
    assert list(R.fp_grid("e2m1")[0]) == [0, 0.5, 1, 1.5, 2, 3, 4, 6]
    assert len(R.fp_grid("e2m1")[0]) == 8 and len(R.fp_grid("e3m2")[0]) == 32 and len(R.fp_grid("e4m7")[0]) == 2048
    assert R.fp_grid("e4m3")[0][1] == 2.0**-9 and R.fp_grid("e5m2")[0][1] == 2.0**-16  # subnormal steps
    for fmt in R.FP_FORMATS:
        v, c = R.fp_grid(fmt)
        assert (np.diff(v) > 0).all() and (np.diff(c) > 0).all()


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_fp8_rounding_reference_matches_torch_conversion(fmt):
    """Ties to even at every midpoint of the grid and random values: the same as torch's float8 cast."""
    vals, _ = R.fp_grid(fmt)
    mids = (vals[:-1] + vals[1:]) / 2
    near = np.concatenate([mids, np.nextafter(mids.astype(np.float32), 0), np.nextafter(mids.astype(np.float32), 1e9),
                           vals, np.random.default_rng(0).uniform(0, vals[-1], 4096)]).astype(np.float32)
    v = np.concatenate([near, -near])
    dt = torch.float8_e4m3fn if fmt == "e4m3" else torch.float8_e5m2
    want = torch.from_numpy(v).to(dt).view(torch.uint8).numpy().astype(np.int64)
    _eq(R.fp_round(v, fmt), want, fmt)


def test_fmaf_reference_is_correctly_rounded():
    rng = np.random.default_rng(1)
    a = rng.standard_normal(4000).astype(np.float32)
    b = (rng.standard_normal(4000) * 2.0**rng.integers(-30, 30, 4000)).astype(np.float32)
    c = (rng.standard_normal(4000) * 2.0**rng.integers(-60, 60, 4000)).astype(np.float32)
    # midpoint cases: a*b lands half an fp32 ulp from c, plus a tiny c below it
    a[:3], b[:3], c[:3] = np.float32(1 + 2**-23), np.float32(1 + 2**-23), np.float32(-2.0**-46)
    got = R.fmaf(a, b, c)
    for i in range(4000):
        exact = fractions.Fraction(float(a[i])) * fractions.Fraction(float(b[i])) + fractions.Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [lo, np.nextafter(lo, np.float32(-np.inf)), np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda z: (abs(fractions.Fraction(float(z)) - exact),
                                         int(np.array(z).view(np.int32)) & 1))
        assert got[i] == best, (i, a[i], b[i], c[i], got[i], best)


def test_host_fma_is_correctly_rounded():
    """The host tier's ``_fma32`` (asymmetric dequantize, LoCo update) equals the correctly rounded reference, also where
    the float64 sum itself rounds onto an fp32 midpoint (205 * 10475530 * 2^-55 + 1 is just above one)."""
    rng = np.random.default_rng(3)
    a = rng.integers(-255, 256, 20000).astype(np.float32)
    b = (rng.standard_normal(20000) * 2.0**rng.integers(-60, 10, 20000)).astype(np.float32)
    c = (rng.standard_normal(20000) * 2.0**rng.integers(-10, 10, 20000)).astype(np.float32)
    a[0], b[0], c[0] = 205.0, np.float32(10475530 * 2.0**-55), 1.0
    got = Q._fma32(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(c)).numpy()
    assert got[0] == np.nextafter(np.float32(1), np.float32(2))
    _eq(got, R.fmaf(a, b, c), "_fma32")


def test_host_codec_matches_grid_rounding_in_every_format():
    """``_host_codec`` finds exponents with ``floor(log2)``: it must agree with the enumerated grid, also just below a
    power of two and across the subnormal band."""
    rng = np.random.default_rng(2)
    for fmt, (bits, m) in R.FP_FORMATS.items():
        vals, _ = R.fp_grid(fmt)
        mids = (vals[:-1] + vals[1:]) / 2
        pw = 2.0**np.arange(-20, 16)
        v = np.concatenate([vals, mids, np.nextafter(pw.astype(np.float32), 0), rng.uniform(0, vals[-1] * 1.1, 8192)])
        v = np.concatenate([v, -v]).astype(np.float32)
        got = _host_codec(torch.from_numpy(v), bits, m).double().numpy()
        _eq(got, R.fp_decode(R.fp_round(v, fmt), fmt), fmt)


# ---- host paths against the references --------------------------------------------------------------------------------
@pytest.mark.parametrize("bits,sym", [(4, True), (4, False), (8, True), (8, False)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_host_quantize_dequantize_exact(bits, sym, dtype):
    gen = torch.Generator().manual_seed(bits * 10 + sym)
    groups, gs = 11, 40
    x = R.quant_cases(groups, gs, dtype, bits, sym, gen)
    qt = Q.Symmetric if sym else Q.Asymmetric
    q, p = Q.quantize(x, groups, bits, qt)
    codes, scale, offset = R.int_quant_reference(x, groups, bits, sym)
    _eq(q.view(groups, -1).numpy(), R.pack_int(codes, bits, sym), "codes")
    _eq(p.reshape(groups, -1)[:, 0].numpy(), scale, "scale")
    if not sym:
        _eq(p[:, 1].numpy(), offset, "offset")
    out = Q.dequantize(q, p, groups, bits, qt, dtype=dtype)
    want = torch.from_numpy(R.int_dequant_reference(codes, scale, offset)).to(dtype).reshape(-1)
    R.assert_bits_equal(out, want, "dequantize")
    # the ties went to even codes; zeros stay zero, in the tiny group too (symmetric codes have an exact zero)
    assert float(scale[0]) == 2.0**-3 and (codes[0, 1:-1] % 2 == 0).all()
    if sym:
        assert (out.view(groups, gs)[2] == 0).all() and (out.view(groups, gs)[4][::3] == 0).all()


@pytest.mark.parametrize("bits,sym", [(4, True), (4, False), (8, True), (8, False)])
def test_host_nonfinite_group_is_nan_and_neighbours_exact(bits, sym):
    gen = torch.Generator().manual_seed(5)
    groups, gs = 7, 16
    x = R.quant_cases(groups, gs, torch.float32, bits, sym, gen).view(groups, gs)
    x[1, 0], x[3, gs // 2], x[5, -1] = float("nan"), float("inf"), -float("inf")
    if not sym:  # finite values whose range hi - lo overflows fp32: no finite scale spans them either
        x[6, 0], x[6, 1] = 3e38, -3e38
    qt = Q.Symmetric if sym else Q.Asymmetric
    q, p = Q.quantize(x.reshape(-1), groups, bits, qt)
    out = Q.dequantize(q, p, groups, bits, qt, dtype=torch.float32).view(groups, gs)
    codes, scale, offset = R.int_quant_reference(x, groups, bits, sym)
    want = R.int_dequant_reference(codes, scale, offset)
    for g in (1, 3, 5) if sym else (1, 3, 5, 6):
        assert torch.isnan(out[g]).all(), g
    _eq(out.numpy(), want, "dequantize")
    _eq(q.view(groups, -1).numpy(), R.pack_int(codes, bits, sym), "codes")


@pytest.mark.parametrize("bits", [4, 8])
def test_host_loco_quantize_exact_and_keeps_error_of_nonfinite_group(bits):
    gen = torch.Generator().manual_seed(bits)
    groups, gs = 9, 24
    x = R.quant_cases(groups, gs, torch.bfloat16, bits, True, gen).view(groups, gs)
    x[7, 3] = float("nan")
    x[8, 0] = float("inf")
    err = torch.randn(groups * gs, generator=gen) * 0.05
    err0 = err.clone()
    q, p = Q.loco_quantize(x.reshape(-1), err, groups, num_bits=bits, beta=0.8)
    codes, scale, upd = R.loco_reference(x, err0, groups, bits, 0.8, False)
    _eq(q.view(groups, -1).numpy(), R.pack_int(codes, bits, True), "codes")
    _eq(p.numpy(), scale, "scale")
    _eq(err.view(groups, gs).numpy(), upd, "error buffer")
    assert torch.equal(err.view(groups, gs)[7:], err0.view(groups, gs)[7:])


@pytest.mark.parametrize("bits,sym", [(4, True), (4, False), (8, True), (8, False)])
@pytest.mark.parametrize("with_err", [False, True])
def test_host_quantized_reduction_exact(bits, sym, with_err):
    gen = torch.Generator().manual_seed(3)
    peers, out_groups, gs = 4, 5, 32
    qt = Q.Symmetric if sym else Q.Asymmetric
    x = torch.randn(peers * out_groups * gs, generator=gen)
    x.view(peers, out_groups, gs)[2, 4, 5] = float("nan")
    q, p = Q.quantize(x, peers * out_groups, bits, qt)
    err = torch.randn(out_groups * gs, generator=gen) * 0.01 if with_err else None
    err0 = err.clone() if with_err else None
    oq, op = Q.quantized_reduction(q, p, peers * out_groups, out_groups, bits, qt, err=err, err_beta=0.5)
    codes, scale, offset = R.int_quant_reference(x, peers * out_groups, bits, sym)
    c2, s2, o2, new = R.reduce_reference(codes, scale, offset, peers, bits, sym, err0, 0.5)
    _eq(oq.view(out_groups, -1).numpy(), R.pack_int(c2, bits, sym), "codes")
    _eq(op.reshape(out_groups, -1)[:, 0].numpy(), s2, "scale")
    assert np.isnan(s2[4]) and not np.isnan(s2[:4]).any()
    if with_err:
        _eq(err.view(out_groups, gs).numpy(), new, "error buffer")


@pytest.mark.parametrize("sym", [True, False])
@pytest.mark.parametrize("bits", [2, 3, 8, 12, 16])
def test_host_fake_quantize_exact(bits, sym):
    gen = torch.Generator().manual_seed(bits)
    groups, gs = 8, 32
    x = R.quant_cases(groups, gs, torch.float32, min(bits, 8), sym, gen)
    x.view(groups, gs)[7, 1] = float("nan")
    y = Q.fake_quantize(x.clone(), groups, bits, Q.Symmetric if sym else Q.Asymmetric)
    codes, scale, offset = R.int_quant_reference(x, groups, bits, sym)
    _eq(y.view(groups, gs).numpy(), R.int_dequant_reference(codes, scale, offset), "fake_quantize")


@pytest.mark.parametrize("fmt", list(R.FP_FORMATS))
def test_host_fp_quantize_exact(fmt):
    bits, m = R.FP_FORMATS[fmt]
    gen = torch.Generator().manual_seed(bits)
    gs = 64
    x = torch.randn(6, gs, generator=gen) * torch.exp2(torch.linspace(-12, 2, gs))  # spans the subnormal band
    x[1] = 0.0
    x[2] *= 1e-38  # tiny amax: 1/scale overflows
    x[2, ::4] = 0.0
    x[3, 7] = float("nan")
    x[4, 0] = -float("inf")
    fq = FP_Quantize(group_size=gs)
    vals = fq.quantize(x, q_bits=bits, q_mantisa_bits=m)
    codes, scale = R.fp_quant_reference(x, 6, fmt)
    _eq(fq.get_scales().numpy(), scale, "scale")
    fin = np.isfinite(scale)
    _eq(vals.view(6, gs).double().numpy()[fin], R.fp_decode(codes, fmt)[fin], "codes")
    out = fq.dequantize(vals).float().view(6, gs).numpy()
    want = R.fp_dequant_reference(codes, scale, fmt)
    _eq(out[fin], want[fin], "dequantize")
    assert np.isnan(out[~fin]).all() and (out[1] == 0).all() and (out[2, ::4] == 0).all()


# ---- group-size policy -------------------------------------------------------------------------------------------------
def _group_ok(gs, dtype):
    """``group_ok`` in quant.cu: a multiple of one 16-byte vector, at most 4 vectors per thread of 256 threads."""
    per = 4 if dtype == torch.float32 else 8
    return gs % per == 0 and gs <= 4 * 256 * per and gs % 2 == 0


def test_every_chosen_group_size_is_one_the_kernels_accept():
    from deepspeed_b200.runtime.zero.gather_handles import CUDAQuantizer
    cq = CUDAQuantizer()
    for dtype in DTYPES:
        for n in list(range(8, 20000, 8)) + [4104, 8200, 65536 + 8, 2**20, 2**22 + 8 * 3 * 5 * 7]:
            g = cq._groups_for(n, dtype)
            assert n % g == 0 and _group_ok(n // g, dtype), (dtype, n, n // g)
        for n in (1, 7, 8, 13, 2047, 2048, 2049, 10**6):
            assert _group_ok(Q.aligned_group_size(n), dtype), (dtype, n)
    assert _group_ok(FP_Quantize().group_size, torch.bfloat16)  # the fp quantizer only needs a multiple of 4
    assert FP_Quantize().group_size % 4 == 0


# ---- the checks reject plausible codec bugs ------------------------------------------------------------------------------
def _unpack_int(packed, bits, sym, sign_extend=True):
    """Codes back from ``quantize``'s bytes (``[groups, bytes]``), the way ``dequant_one`` reads them."""
    if bits == 8:
        return packed.astype(np.int64) + (0 if sym else 128)
    b = packed.view(np.uint8).astype(np.int64)
    v = np.stack([b & 0xF, b >> 4], axis=2).reshape(b.shape[0], -1)
    return np.where(sign_extend & sym & (v >= 8), v - 16, v)


def _pack_bits_big_endian(codes, bits):
    c = np.asarray(codes, np.int64).reshape(codes.shape[0], -1)
    bitarr = ((c[:, :, None] >> np.arange(bits)[::-1]) & 1).reshape(c.shape[0], -1)
    return (bitarr.reshape(c.shape[0], -1, 8) << np.arange(8)[::-1]).sum(axis=2).astype(np.uint8)


def _rejected(got, want):
    """True when the bit-exact comparison the GPU tests make refuses ``got``."""
    try:
        R.assert_bits_equal(torch.from_numpy(np.ascontiguousarray(got)), torch.from_numpy(np.ascontiguousarray(want)), "")
    except AssertionError:
        return True
    return False


def test_exact_checks_reject_plausible_codec_bugs():
    """Emulations of a kernel with one plausible bug each produce the outputs the GPU tests compare (packed codes,
    scales, dequantized values) on the inputs those tests use; the same bit-exact comparison against the references
    refuses every mutant and accepts the unmutated emulation."""
    gen = torch.Generator().manual_seed(0)
    groups, gs = 9, 2048
    for bits in (4, 8):
        x = R.quant_cases(groups, gs, torch.bfloat16, bits, True, gen)
        codes, scale, _ = R.int_quant_reference(x, groups, bits, True)
        packed = R.pack_int(codes, bits, True)
        deq = R.int_dequant_reference(_unpack_int(packed, bits, True), scale)
        assert not _rejected(packed, packed) and not _rejected(deq, R.int_dequant_reference(codes, scale))
        trunc, _, _ = R.int_quant_reference(x, groups, bits, True, rint=np.trunc)
        assert _rejected(R.pack_int(trunc, bits, True), packed), f"int{bits}: truncation instead of rint"
        assert _rejected((scale * 2).astype(np.float32), scale), f"int{bits}: scale x2 (params)"
        assert _rejected(R.int_dequant_reference(codes, scale * 2), deq), f"int{bits}: scale x2 (dequantize)"
        if bits == 4:
            u = packed.view(np.uint8)
            swapped = ((u >> 4) | (u << 4)).astype(np.uint8).view(np.int8)
            assert _rejected(swapped, packed), "swapped nibbles"
            no_sign = R.int_dequant_reference(_unpack_int(packed, 4, True, sign_extend=False), scale)
            assert _rejected(no_sign, deq), "no 4-bit sign extension"
    for fmt, bits in (("e4m3", 8), ("e5m2", 8), ("e3m2", 6)):
        x = R.fp_cases(fmt, 6, 1028, gen)
        codes, scale = R.fp_quant_reference(x, 6, fmt)
        packed = R.pack_bits(codes, bits)
        assert not _rejected(packed, R.pack_bits(codes, bits))
        if bits == 8:
            g = R._np32(x).reshape(6, -1)
            away = R.fp_round(R.to_grid(g, scale[:, None]), fmt, ties_even=False)
            assert _rejected(R.pack_bits(away, 8), packed), f"{fmt}: ties away from zero"
        else:
            assert _rejected(_pack_bits_big_endian(codes, 6), packed), "6-bit codes packed big-endian"


# ---- a NaN gradient through qgZ reaches the step skip ------------------------------------------------------------------------
def _nan_gradient_run(zero_extra):
    """ZeRO-3 bf16 with clipping on 2 ranks; rank 1 plants a NaN in one activation gradient at step 1.  Returns, per step,
    the global norm, and whether the skipped step left every bf16 weight and fp32 master bit-unchanged."""
    import math
    import torch.distributed as td
    import deepspeed_b200 as ds
    from tests.unit.simple_model import SimpleModel, base_config, make_batch
    if td.get_backend() == "gloo":  # gloo ranks exchange host tensors: run on the host tier even where a GPU is visible
        from deepspeed_b200.accelerator.host_accelerator import HostAccelerator
        from deepspeed_b200.accelerator.real_accelerator import set_accelerator
        set_accelerator(HostAccelerator())
    torch.manual_seed(0)
    model = SimpleModel()
    cfg = base_config(3, "bf16", 1, 1.0)
    cfg["zero_optimization"].update(zero_extra)
    eng, *_ = ds.initialize(model=model, config=cfg)
    zo = eng.optimizer
    r, w = ds.comm.get_rank(), ds.comm.get_world_size()
    inject = {"on": False}

    def plant(g):
        if inject["on"] and r == 1:
            g = g.clone()
            g.view(-1)[0] = math.nan
        return g

    model.layers[0].register_forward_hook(lambda mod, inp, out: (out.register_hook(plant), out)[1])

    def snapshot():
        return [(zo._piece_lp(rt, s, e).clone(), zo._piece_master(rt, s, e).clone()) for rt, gi, s, e in zo.pieces
                if gi >= 0]

    gen = torch.Generator().manual_seed(1)
    norms, unchanged = [], None
    for it in range(3):
        inject["on"] = it == 1
        x, y = make_batch(w, 4, gen)
        loss = eng(x[r * 4:(r + 1) * 4].bfloat16().to(eng.device), y[r * 4:(r + 1) * 4].to(eng.device))
        eng.backward(loss)
        before = snapshot()
        eng.step()
        if it == 1:
            unchanged = all(torch.equal(a0, a1) and torch.equal(m0, m1) for (a0, m0), (a1, m1) in zip(before, snapshot()))
        norms.append(eng.get_global_grad_norm())
    return norms, unchanged


def _nan_gradient_with_and_without_qgz():
    import math
    for extra in ({}, {"zero_quantized_gradients": True}):
        norms, unchanged = _nan_gradient_run(extra)
        assert math.isfinite(norms[0]) and math.isfinite(norms[2]), (extra, norms)
        assert norms[1] == math.inf, (extra, norms)  # the NaN reached the norm pass: the step was skipped
        assert unchanged, f"{extra}: the skipped step changed weights or masters"


def test_nan_gradient_skips_the_step_with_and_without_qgz():
    """A NaN gradient on one rank ends the same way with ``zero_quantized_gradients`` as without: qgZ's int4 round trip
    keeps it non-finite, so the norm is inf and the step leaves weights and masters bit-unchanged.  On the host tier over
    gloo, or through the kernels over NCCL where two GPUs are present."""
    from tests.common import run_distributed
    run_distributed(_nan_gradient_with_and_without_qgz, 2)
