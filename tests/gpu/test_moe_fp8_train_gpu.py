"""GPU tier: FP8 dropless MoE experts -- the ragged forms of the FP8 wgmma GEMM (``dsb_gemm_fp8_ragged``,
``dsb_gemm_fp8_ragged_wgrad``), the FP8 ragged SwiGLU node (``ops/linear.py`` ``_FP8RaggedSwiGLUFn``), the dropless MoE
layer with FP8 experts and ``MixtralConfig(fp8_experts=True)`` under the engine.

Kernel checks are exact: fp8 operands on a power-of-two integer grid and power-of-two scales that differ between any two
neighbouring strips and blocks, so every promoted sum is exact and a correct result is bit-equal to the float64 product
rounded once.  Row operands hold NaN bytes (and blockwise scales NaN) outside the experts' segments, outputs sit inside
NaN guard bands, and rows outside the segments must keep their bits."""
import math
import zlib

import pytest
import torch

from tests.common import run_distributed
from tests.gpu.test_fp8_blockwise_gpu import NAN8, _bigram_batches, f8_grid
from tests.gpu.test_gemm_gpu import Guarded
from tests.gpu.test_moe_grouped_train_gpu import COUNTS, GuardedStack, check_rows_untouched, dev_offsets
from tests.numerics import assert_bits_equal, assert_within, dswiglu_reference, swiglu_reference

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
B = 128
NAN = float("nan")
RECIPES = ["tensorwise", "blockwise"]
SMS = (0, 1, 3, 7)


def _K():
    from deepspeed_b200.ops.kernels import gemm_sm100
    return gemm_sm100


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(("moe-fp8", ) + key).encode()))


def layout(counts, lead=0, tail=0):
    """Offsets of 128-row aligned segments after ``lead`` rows (a multiple of 128), and the row count with ``tail``."""
    off = [lead]
    for c in counts:
        off.append(off[-1] + -(-c // B) * B)
    return off, off[-1] + tail


def seg_rows(counts, off, R, cols, fmt, gen):
    """fp8 ``[R, cols]``: expert e's ``counts[e]`` grid rows, zeros on its padding, NaN bytes elsewhere."""
    x = torch.full((R, cols), NAN8, dtype=torch.uint8, device="cuda").view(fmt)
    for e, c in enumerate(counts):
        x[off[e]:off[e + 1]].view(torch.uint8).zero_()
        if c:
            x[off[e]:off[e] + c] = f8_grid(c, cols, fmt, gen)[0]
    return x


def seg_cols(counts, off, R, rows, fmt, gen):
    """The transposed layout ``[rows, R]`` of :func:`seg_rows`, with per-row exponents (returned) for exact addends."""
    v, ex = f8_grid(rows, R, fmt, gen)
    x = torch.full((rows, R), NAN8, dtype=torch.uint8, device="cuda").view(fmt)
    for e, c in enumerate(counts):
        x[:, off[e]:off[e + 1]].view(torch.uint8).zero_()
        x[:, off[e]:off[e] + c] = v[:, off[e]:off[e] + c]
    return x, ex


def scales(block, a_shape, b_shape, gen, a_cols_nan=None):
    """``(sa, sb)``: tensorwise two power-of-two scalars; blockwise strips ``[ceil(K/128), rows of A]`` and blocks of B
    that differ between neighbours.  ``a_cols_nan``: columns of ``sa`` (rows of A) set to NaN."""
    if not block:
        e = torch.randint(-3, 4, (2, ), generator=gen, device="cuda").float()
        return torch.ldexp(torch.ones(1, device="cuda"), e[:1].int()), torch.ldexp(torch.ones(1, device="cuda"), e[1:].int())
    (ma, ka), (nb, kbb) = a_shape, b_shape
    ia = torch.arange(-(-ka // B), device="cuda")[:, None] * 3 + torch.arange(ma, device="cuda")[None, :]
    ib = torch.arange(-(-nb // B), device="cuda")[:, None] * 2 + torch.arange(-(-kbb // B), device="cuda")[None, :] * 3
    one = torch.ones((), device="cuda")
    sa, sb = torch.ldexp(one, (ia % 5 - 2).int()), torch.ldexp(one, (ib % 5 - 2).int())
    if a_cols_nan is not None:
        sa[:, a_cols_nan] = NAN
    return sa, sb


def deq(t, s, block, mode):
    """float64 values of the cast ``t`` with scales ``s`` (mode "strip": ``s [ceil(C/128), R]``; "block")."""
    if not block:
        return t.double() * float(s)
    R, C = t.shape
    if mode == "strip":
        return t.double() * s.t().double().repeat_interleave(B, dim=1)[:, :C]
    return t.double() * s.double().repeat_interleave(B, dim=0)[:R].repeat_interleave(B, dim=1)[:, :C]


def outside(counts, off, R):
    """Row indices outside the experts' segments."""
    m = torch.ones(R, dtype=torch.bool)
    m[off[0]:off[-1]] = False
    return m.nonzero().flatten().cuda()


# ---------------------------------------------------------------------------------------------------------------------
# 1. exact oracle per form
# ---------------------------------------------------------------------------------------------------------------------
def run_forward(counts, Nn, Kd, epi, block, gen, lead=0, tail=0, sms=0):
    """forward: a e4m3 [R, K], b the stacked weight [E Nb, K] (SwiGLU: Nb = 2 Nn), expert e's rows at e Nb."""
    K_ = _K()
    E = len(counts)
    off, R = layout(counts, lead, tail)
    Nb = 2 * Nn if epi == K_.EPI_SWIGLU else Nn
    a = seg_rows(counts, off, R, Kd, E4M3, gen)
    b = f8_grid(E * Nb, Kd, E4M3, gen)[0]
    sa, sb = scales(block, (R, Kd), (E * Nb, Kd), gen, outside(counts, off, R))
    what = f"fp8 ragged forward epi={epi} block={block} E={E} N={Nn} K={Kd} lead={lead} tail={tail} sms={sms}"
    Ad, Bd = deq(a, sa, block, "strip"), deq(b, sb, block, "block")
    out = Guarded(R, Nn)
    gu = Guarded(R, 2 * Nn) if epi == K_.EPI_SWIGLU else None
    K_.fp8_ragged_matmul(a, b, dev_offsets(off), sa, sb, E, out=out.view, epi=epi, out2=gu.view if gu else None,
                         block=block, sms=sms)
    for e, c in enumerate(counts):
        if c:
            s = slice(off[e], off[e] + c)
            ref = Ad[s] @ Bd[e * Nb:(e + 1) * Nb].t()
            if gu is None:
                assert_bits_equal(out.view[s], ref.to(BF16), f"{what} expert {e}")
            else:
                assert_bits_equal(gu.view[s], ref.to(BF16), f"{what} gate|up expert {e}")
                want, bound = swiglu_reference(ref[:, :Nn], ref[:, Nn:])
                assert_within(out.view[s], want, bound, f"{what} act expert {e}")
    res = out.view.clone()
    check_rows_untouched(out, counts, off, what)
    if gu is not None:
        check_rows_untouched(gu, counts, off, what + " gate|up")
    return res


def run_dgrad(counts, Nn, Kd, epi, block, gen, lead=0, tail=0, sms=0):
    """dgrad: a e5m2 [R, K], b the transposed cast [N, E K], expert e's slab at column e K."""
    K_ = _K()
    E = len(counts)
    off, R = layout(counts, lead, tail)
    a = seg_rows(counts, off, R, Kd, E5M2, gen)
    b = f8_grid(Nn, E * Kd, E4M3, gen)[0]
    sa, sb = scales(block, (R, Kd), (Nn, E * Kd), gen, outside(counts, off, R))
    what = f"fp8 ragged dgrad epi={epi} block={block} E={E} N={Nn} K={Kd} lead={lead} tail={tail} sms={sms}"
    Ad, Bd = deq(a, sa, block, "strip"), deq(b, sb, block, "block")
    if epi == K_.EPI_DSWIGLU:
        aux = torch.full((R, 2 * Nn), NAN, dtype=BF16, device="cuda")
        for e, c in enumerate(counts):
            aux[off[e]:off[e + 1]] = 0
            aux[off[e]:off[e] + c] = (torch.randn(c, 2 * Nn, generator=gen, device="cuda") * 2).to(BF16)
        out = Guarded(R, 2 * Nn)
        K_.fp8_ragged_matmul(a, b, dev_offsets(off), sa, sb, E, out=out.view[:, :Nn], epi=epi, aux=aux, out2=out.view,
                             block=block, sms=sms)
    else:
        out = Guarded(R, Nn)
        K_.fp8_ragged_matmul(a, b, dev_offsets(off), sa, sb, E, out=out.view, block=block, sms=sms)
    for e, c in enumerate(counts):
        if c:
            s = slice(off[e], off[e] + c)
            ref = Ad[s] @ Bd[:, e * Kd:(e + 1) * Kd].t()
            if epi == K_.EPI_DSWIGLU:
                dg, dg_b, du, du_b = dswiglu_reference(ref, aux[s, :Nn], aux[s, Nn:], d_fp32=True)
                assert_within(out.view[s, :Nn], dg, dg_b, f"{what} dgate expert {e}")
                assert_within(out.view[s, Nn:], du, du_b, f"{what} dup expert {e}")
            else:
                assert_bits_equal(out.view[s], ref.to(BF16), f"{what} expert {e}")
    res = out.view.clone()
    check_rows_untouched(out, counts, off, what)
    return res


def run_wgrad(counts, M, Nn, accumulate, block, gen, lead=0, tail=0, sms=0):
    """out[e] (+)= a[:, rows of e] b[:, rows of e]^T, a e5m2 [M, R], b e4m3 [N, R]."""
    K_ = _K()
    E = len(counts)
    off, R = layout(counts, lead, tail)
    a, ea = seg_cols(counts, off, R, M, E5M2, gen)
    b, eb = seg_cols(counts, off, R, Nn, E4M3, gen)
    sa, sb = scales(block, (M, R), (Nn, R), gen)
    Ad, Bd = deq(a, sa, block, "strip"), deq(b, sb, block, "block")
    c_old = None
    if accumulate:
        v = torch.randint(-128, 129, (E, M, Nn), generator=gen, device="cuda").float()
        c_old = (torch.ldexp(v, (ea[:, None] + eb[None, :])[None]) * 2.0**-3).to(BF16)
    out = GuardedStack(E, M, Nn, fill=c_old)
    K_.fp8_ragged_wgrad(a, b, dev_offsets(off), sa, sb, E, out=out.view, accumulate=accumulate, block=block, sms=sms)
    what = f"fp8 ragged wgrad acc={accumulate} block={block} E={E} M={M} N={Nn} sms={sms}"
    for e, c in enumerate(counts):
        if c:
            s = slice(off[e], off[e + 1])
            ref = Ad[:, s] @ Bd[:, s].t()
            if accumulate:
                ref = ref + c_old[e].double()
            assert_bits_equal(out.view[e] + 0.0, ref.to(BF16) + 0.0, f"{what} expert {e}")
        elif accumulate:
            assert_bits_equal(out.view[e], c_old[e], f"{what}: empty expert {e} under ACCUM")
        else:
            assert bool((out.view[e] == 0).all()), f"{what}: empty expert {e} under STORE is not zero"
    out.check_guards(what)
    return out.view.clone()


CASES = sorted(COUNTS)
BLOCKS = dict(argvalues=[False, True], ids=["tensorwise", "blockwise"])


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("block", **BLOCKS)
def test_fp8_ragged_forward_store_exact(case, block):
    """The down projection: expert e's rows of the stacked [E H, I] weight."""
    run_forward(COUNTS[case], 256, 192, _K().EPI_STORE, block, _gen("fwd", case, block), lead=128, tail=37)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("block", **BLOCKS)
def test_fp8_ragged_forward_swiglu_exact(case, block):
    """gate|up (+) SwiGLU: gate rows at e 2I + col0, up rows at e 2I + I + col0; I % 128 == 64 puts the up rows at an
    offset inside their 128-row scale block."""
    run_forward(COUNTS[case], 192, 256, _K().EPI_SWIGLU, block, _gen("swiglu", case, block), lead=0, tail=5)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("block", **BLOCKS)
def test_fp8_ragged_dgrad_store_exact(case, block):
    """dX of gate|up: the transposed cast [H, E 2I], expert e's W^T the column slab at e 2I."""
    run_dgrad(COUNTS[case], 200, 384, _K().EPI_STORE, block, _gen("dgrad", case, block), lead=128, tail=64)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("block", **BLOCKS)
def test_fp8_ragged_dgrad_dswiglu_exact(case, block):
    """down dX (+) dSwiGLU: the transposed cast [I, E H], expert e's slab at column e H."""
    run_dgrad(COUNTS[case], 192, 256, _K().EPI_DSWIGLU, block, _gen("dswiglu", case, block), lead=0, tail=128)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("accumulate", [False, True], ids=["store", "accum"])
@pytest.mark.parametrize("block", **BLOCKS)
def test_fp8_ragged_wgrad_exact(case, accumulate, block):
    """Variable-K dW: each tile sums its expert's k-blocks only; empty experts store zeros or keep C; M and N tails."""
    M, Nn = (200, 328) if case != "e256" else (136, 136)
    run_wgrad(COUNTS[case], M, Nn, accumulate, block, _gen("wgrad", case, accumulate, block), lead=128, tail=16)


@pytest.mark.parametrize("block", **BLOCKS)
def test_fp8_ragged_forms_grid_independent(block):
    """Each tile's k loop runs in one CTA in a fixed order: every form is bit-identical over CTA counts and relaunches."""
    K_ = _K()
    counts = COUNTS["edges"]
    forms = (("fwd", lambda g, s: run_forward(counts, 256, 192, K_.EPI_STORE, block, g, 128, 9, s)),
             ("swiglu", lambda g, s: run_forward(counts, 192, 256, K_.EPI_SWIGLU, block, g, 0, 3, s)),
             ("dgrad", lambda g, s: run_dgrad(counts, 200, 384, K_.EPI_STORE, block, g, 0, 0, s)),
             ("dswiglu", lambda g, s: run_dgrad(counts, 192, 256, K_.EPI_DSWIGLU, block, g, 128, 0, s)),
             ("wgrad", lambda g, s: run_wgrad(counts, 200, 328, False, block, g, 0, 0, s)),
             ("wgrad-acc", lambda g, s: run_wgrad(counts, 200, 328, True, block, g, 0, 0, s)))
    for name, fn in forms:
        first = None
        for sms in SMS:
            for _ in range(2 if sms == 0 else 1):
                got = fn(_gen("grid", name, block), sms)
                if first is None:
                    first = got
                else:
                    assert_bits_equal(got, first, f"{name} block={block} sms={sms}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. refused arguments
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", ["unaligned", "decreasing", "past_rows"])
@pytest.mark.parametrize("form", ["fwd", "dgrad", "wgrad"])
def test_fp8_ragged_malformed_offsets_write_nothing(bad, form):
    """Device offsets that are not non-decreasing multiples of 128 inside [0, R]: the kernel checks them before anything
    else and every CTA leaves, writing nothing."""
    K_ = _K()
    g = _gen("malformed", bad, form)
    R, E, H = 512, 3, 256
    off = {"unaligned": [0, 64, 256, 384], "decreasing": [0, 256, 128, 384], "past_rows": [0, 128, 256, 640]}[bad]
    sa, sb = torch.ones(1, device="cuda"), torch.ones(1, device="cuda")
    if form == "wgrad":
        a, b = f8_grid(H, R, E5M2, g)[0], f8_grid(H, R, E4M3, g)[0]
        out = GuardedStack(E, H, H)
        K_.fp8_ragged_wgrad(a, b, dev_offsets(off), sa, sb, E, out=out.view)
        torch.cuda.synchronize()
        assert bool(out.view.isnan().all()), f"{form} {bad}: written"
        out.check_guards(f"{form} {bad}")
        return
    fmt = E4M3 if form == "fwd" else E5M2
    a = f8_grid(R, H, fmt, g)[0]
    b = f8_grid(E * H, H, E4M3, g)[0] if form == "fwd" else f8_grid(H, E * H, E4M3, g)[0]
    out = Guarded(R, H)
    K_.fp8_ragged_matmul(a, b, dev_offsets(off), sa, sb, E, out=out.view)
    torch.cuda.synchronize()
    out.check_untouched(f"{form} {bad}: the output")


def _refusal(case):
    K_ = _K()
    g = _gen("refusal", case)
    R, E, H, I = 256, 2, 256, 128
    off = dev_offsets([0, 128, 256])
    one = torch.ones(1, device="cuda")
    x8 = f8_grid(R, H, E4M3, g)[0]
    w13 = f8_grid(E * 2 * I, H, E4M3, g)[0]
    w2t = f8_grid(I, E * H, E4M3, g)[0]
    dy8 = f8_grid(R, H, E5M2, g)[0]
    sa_b = torch.ones(2, R, device="cuda")
    sb_b = torch.ones(E * 2 * I // B, H // B, device="cuda")
    mm = K_.fp8_ragged_matmul
    return {
        "block_sa_shape": (lambda o: mm(x8, w13, off, torch.ones(1, R, device="cuda"), sb_b, E, out=o, epi=K_.EPI_SWIGLU,
                                        block=True), (R, I)),
        "block_sb_shape": (lambda o: mm(x8, w13, off, sa_b, torch.ones(3, 2, device="cuda"), E, out=o,
                                        epi=K_.EPI_SWIGLU, block=True), (R, I)),
        "tensor_scale_shape": (lambda o: mm(x8, w13, off, sa_b, one, E, out=o, epi=K_.EPI_SWIGLU), (R, I)),
        "wrong_e": (lambda o: mm(x8, w13, off, one, one, 3, out=o, epi=K_.EPI_SWIGLU), (R, I)),
        "dgrad_k_mod128": (lambda o: mm(f8_grid(R, 192, E5M2, g)[0], f8_grid(I, E * 192, E4M3, g)[0], off, one, one, E,
                                        out=o), (R, I)),
        "fwd_dswiglu": (lambda o: mm(x8, f8_grid(E * I, H, E4M3, g)[0], off, one, one, E, out=o, epi=K_.EPI_DSWIGLU,
                                     aux=torch.zeros(R, 2 * I, dtype=BF16, device="cuda"),
                                     out2=torch.zeros(R, 2 * I, dtype=BF16, device="cuda")), (R, I)),
        "dgrad_swiglu": (lambda o: mm(dy8, w2t, off, one, one, E, out=o, epi=K_.EPI_SWIGLU), (R, I)),
        "e257": (lambda o: mm(x8, f8_grid(257 * 16, H, E4M3, g)[0], dev_offsets([0] * 258), one, one, 257, out=o),
                 (R, 16)),
        "wgrad_sa_shape": (lambda o: K_.fp8_ragged_wgrad(f8_grid(H, R, E5M2, g)[0], f8_grid(H, R, E4M3, g)[0], off,
                                                         torch.ones(1, H, device="cuda"), torch.ones(2, 2, device="cuda"),
                                                         E, out=o.view(E, H, H), block=True), (E * H, H)),
        "wgrad_b_rows": (lambda o: K_.fp8_ragged_wgrad(f8_grid(H, R, E5M2, g)[0], f8_grid(H, R - 16, E4M3, g)[0], off,
                                                       one, one, E, out=o.view(E, H, H)), (E * H, H)),
    }[case]


@pytest.mark.parametrize("case", ["block_sa_shape", "block_sb_shape", "tensor_scale_shape", "wrong_e", "dgrad_k_mod128",
                                  "fwd_dswiglu", "dgrad_swiglu", "e257", "wgrad_sa_shape", "wgrad_b_rows"])
def test_fp8_ragged_refused_arguments_raise_and_write_nothing(case):
    from deepspeed_b200.ops.native import NativeOpError
    call, (rows, cols) = _refusal(case)
    out = torch.full((rows, cols), NAN, dtype=BF16, device="cuda")
    with pytest.raises(NativeOpError):
        call(out)
    torch.cuda.synchronize()
    assert bool(out.isnan().all()), f"{case}: written by a refused call"


# ---------------------------------------------------------------------------------------------------------------------
# 3. against the dense FP8 GEMM per expert
# ---------------------------------------------------------------------------------------------------------------------
def test_fp8_ragged_tensorwise_bit_equal_to_fp8_matmul_per_expert():
    """Random (not grid) operands: every ragged form with given scalar scales is bit-equal to ``fp8_matmul`` run on each
    expert's rows and weight slab with the same scales (the same tile, k order and promotion)."""
    K_ = _K()
    g = _gen("vs-dense")
    counts = [300, 0, 17, 256, 129]
    E, H, I = len(counts), 256, 192
    off, R = layout(counts, 128, 64)
    offs = dev_offsets(off)
    rnd = lambda *s, fmt: (torch.randn(*s, generator=g, device="cuda") * 8).to(fmt)
    sa, sb = torch.tensor([2.0**-3], device="cuda"), torch.tensor([2.0**-5], device="cuda")
    x8, w13, w2 = rnd(R, H, fmt=E4M3), rnd(E * 2 * I, H, fmt=E4M3), rnd(E * H, I, fmt=E4M3)
    dy8, w2t, w13t = rnd(R, H, fmt=E5M2), rnd(I, E * H, fmt=E4M3), rnd(H, E * 2 * I, fmt=E4M3)
    gu_aux = (torch.randn(R, 2 * I, generator=g, device="cuda")).to(BF16)
    act8 = rnd(R, I, fmt=E4M3)
    a_t, b_t = rnd(H, R, fmt=E5M2), rnd(I, R, fmt=E4M3)
    gu = torch.empty(R, 2 * I, dtype=BF16, device="cuda")
    act = K_.fp8_ragged_matmul(x8, w13, offs, sa, sb, E, epi=K_.EPI_SWIGLU, out2=gu)
    y = K_.fp8_ragged_matmul(act8, w2, offs, sa, sb, E)
    dgu = torch.empty(R, 2 * I, dtype=BF16, device="cuda")
    K_.fp8_ragged_matmul(dy8, w2t, offs, sa, sb, E, epi=K_.EPI_DSWIGLU, aux=gu_aux, out2=dgu)
    dgu8 = dgu.to(E5M2)
    dx = K_.fp8_ragged_matmul(dgu8, w13t, offs, sa, sb, E)
    dw = K_.fp8_ragged_wgrad(a_t, b_t, offs, sa, sb, E)
    for e, c in enumerate(counts):
        s = slice(off[e], off[e + 1])
        if not c:
            assert not bool(dw[e].any())
            continue
        gu_e = torch.empty(off[e + 1] - off[e], 2 * I, dtype=BF16, device="cuda")
        act_e = K_.fp8_matmul(x8[s], w13[e * 2 * I:(e + 1) * 2 * I], sa, sb, epi=K_.EPI_SWIGLU, out2=gu_e)
        assert_bits_equal(act[s], act_e, f"act expert {e}")
        assert_bits_equal(gu[s], gu_e, f"gate|up expert {e}")
        assert_bits_equal(y[s], K_.fp8_matmul(act8[s], w2[e * H:(e + 1) * H], sa, sb), f"y expert {e}")
        d_e = torch.empty(off[e + 1] - off[e], 2 * I, dtype=BF16, device="cuda")
        K_.fp8_matmul(dy8[s], w2t[:, e * H:(e + 1) * H], sa, sb, epi=K_.EPI_DSWIGLU, aux=gu_aux[s], out2=d_e)
        assert_bits_equal(dgu[s], d_e, f"dgate|dup expert {e}")
        assert_bits_equal(dx[s], K_.fp8_matmul(dgu8[s], w13t[:, e * 2 * I:(e + 1) * 2 * I], sa, sb), f"dx expert {e}")
        assert_bits_equal(dw[e], K_.fp8_matmul(a_t[:, s], b_t[:, s], sa, sb), f"dW expert {e}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. the node
# ---------------------------------------------------------------------------------------------------------------------
def _node_case(counts, H, I, seed, lead=0, tail=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = len(counts)
    off, R = layout(counts, lead, tail)
    x = torch.zeros(R, H, dtype=BF16, device="cuda")
    dy = torch.zeros(R, H, dtype=BF16, device="cuda")
    for e, c in enumerate(counts):
        x[off[e]:off[e] + c] = (torch.randn(c, H, generator=g, device="cuda") * (1 + e)).to(BF16)
        dy[off[e]:off[e] + c] = torch.randn(c, H, generator=g, device="cuda").to(BF16)
    w13 = (torch.randn(E, 2 * I, H, generator=g, device="cuda") * H**-0.5).to(BF16)
    w2 = (torch.randn(E, H, I, generator=g, device="cuda") * I**-0.5).to(BF16)
    return off, x, dy, w13, w2


def test_fp8_ragged_blockwise_node_bit_equal_to_dense_node_per_expert():
    """With 128-row segments every strip and block of the blockwise recipe coincides with the one the dense node casts on
    the expert's padded segment: the same arithmetic in the same order, so y, dx, dW13 and dW2 are bit-equal."""
    from deepspeed_b200.ops.linear import fp8_ragged_swiglu_mlp, fp8_ragged_swiglu_native, fp8_swiglu_mlp
    counts = [300, 0, 17, 256, 1, 129]
    E, H, I = len(counts), 256, 320
    off, x0, dy, w13_0, w2_0 = _node_case(counts, H, I, 11, lead=0, tail=0)
    offs = dev_offsets(off)
    assert fp8_ragged_swiglu_native(x0, offs, w13_0, w2_0)
    x, w13, w2 = (t.clone().requires_grad_(True) for t in (x0, w13_0, w2_0))
    y = fp8_ragged_swiglu_mlp(x, offs, w13, w2, recipe="blockwise")
    y.backward(dy)
    for e, c in enumerate(counts):
        s = slice(off[e], off[e + 1])
        if not c:
            assert not bool(w13.grad[e].any()) and not bool(w2.grad[e].any()), f"empty expert {e}"
            continue
        xe, we13, we2 = (t.clone().requires_grad_(True) for t in (x0[s], w13_0[e], w2_0[e]))
        ye = fp8_swiglu_mlp(xe, we13, we2, recipe="blockwise")
        ye.backward(dy[s])
        assert_bits_equal(y[s], ye, f"y expert {e}")
        assert_bits_equal(x.grad[s], xe.grad, f"dx expert {e}")
        assert_bits_equal(w13.grad[e], we13.grad, f"dW13 expert {e}")
        assert_bits_equal(w2.grad[e], we2.grad, f"dW2 expert {e}")


@pytest.mark.parametrize("recipe", RECIPES)
def test_fp8_ragged_node_against_reference_path(recipe, monkeypatch):
    """The wgmma path against the node's torch reference of the same recipe (offsets read on the host): the bound of the
    dense FP8 node tests, in norm (silu is ``__expf`` against ``torch.exp``, and a cast can flip on a last-bit difference)."""
    from deepspeed_b200.ops import linear
    counts = [200, 0, 130, 384]
    off, x0, dy, w13_0, w2_0 = _node_case(counts, 256, 448, 12, lead=128, tail=128)
    offs = dev_offsets(off)

    def run():
        x, w13, w2 = (t.clone().requires_grad_(True) for t in (x0, w13_0, w2_0))
        y = linear.fp8_ragged_swiglu_mlp(x, offs, w13, w2, recipe=recipe)
        y.backward(dy)
        return y.detach()[off[0]:off[-1]], x.grad[off[0]:off[-1]], w13.grad, w2.grad

    got = run()
    monkeypatch.setattr(linear, "fp8_ragged_swiglu_native", lambda *a, **k: False)
    want = run()
    for g_, w_, what in zip(got, want, ("y", "dx", "dW13", "dW2")):
        assert bool(torch.isfinite(g_).all()), what
        rel = float((g_.float() - w_.float()).norm() / w_.float().norm())
        assert rel < 2e-2, (what, rel)


def _layer_no_sync_first_backward_on_autograd_thread(recipe):
    """A fresh process: the dropless layer with FP8 experts runs forward and backward (its first backward, on the
    autograd worker thread) with no host synchronisation, and stays close to the bf16 experts on the same weights."""
    from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
    from deepspeed_b200.moe.layer import MoE
    E, H, I, T = 4, 256, 256, 384
    layers = []
    for fp8 in (recipe, None):
        torch.manual_seed(0)
        layers.append(MoE(H, GroupedSwiGLUExperts(E, H, I, fp8_recipe=fp8), num_experts=E, k=2, min_capacity=4,
                          drop_tokens=False, use_rts=False).cuda().to(BF16))
    g = torch.Generator(device="cuda").manual_seed(1)
    x0 = torch.randn(T, H, generator=g, device="cuda").to(BF16)
    gy = torch.randn(T, H, generator=g, device="cuda").to(BF16)
    outs = []
    for i, layer in enumerate(layers):
        x = x0.clone().requires_grad_(True)
        torch.cuda.synchronize()
        if i == 0:
            torch.cuda.set_sync_debug_mode("error")
        try:
            y, _, _ = layer(x)
            (y.float() * gy.float()).sum().backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        ex = layer.deepspeed_moe.experts
        outs.append((y, x.grad, ex.w13.grad, ex.w2.grad))
    for a, b, what in zip(*outs, ("y", "dx", "dW13", "dW2")):
        assert a is not None and bool(torch.isfinite(a).all()) and bool(a.any()), what
        rel = float((a.float() - b.float()).norm() / b.float().norm())
        assert rel < 0.1, (recipe, what, rel)


@pytest.mark.parametrize("recipe", RECIPES)
def test_fp8_dropless_layer_no_sync_and_autograd_thread(recipe):
    run_distributed(_layer_no_sync_first_backward_on_autograd_thread, 1, (recipe, ))


# ---------------------------------------------------------------------------------------------------------------------
# 5. engine and convergence
# ---------------------------------------------------------------------------------------------------------------------
def _mixtral(recipe, vocab=1024):
    from deepspeed_b200.models.mixtral import MixtralForCausalLM, mixtral_config
    torch.manual_seed(0)
    fp8 = dict(fp8_experts=True, fp8_recipe=recipe) if recipe else {}
    cfg = mixtral_config("tiny-moe", hidden_size=256, intermediate_size=256, num_attention_heads=4, num_key_value_heads=2,
                         vocab_size=vocab, num_hidden_layers=2, num_local_experts=4, max_position_embeddings=512,
                         drop_tokens=False, **fp8)
    with torch.device("cuda"):
        return MixtralForCausalLM(cfg).to(BF16)


def _engine_losses(recipe, stage, experts_only, two_phase, steps=6):
    import deepspeed_b200 as ds
    model = _mixtral(recipe)
    if experts_only:
        for n, p in model.named_parameters():
            p.requires_grad_(n.endswith(("experts.w13", "experts.w2")))
    config = {"train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
              "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}}, "zero_optimization": {"stage": stage}}
    if two_phase:
        config["gradient_clipping"] = 1e6  # a clip that never bites keeps the step out of backward
    engine, _, _, _ = ds.initialize(model=model, config=config)
    ids = torch.randint(0, 1024, (2, 256), generator=torch.Generator().manual_seed(1)).cuda()
    losses = []
    for _ in range(steps):
        loss = engine(ids, labels=ids)
        engine.backward(loss)
        engine.step()
        losses.append(float(loss))
    return losses


def _engine_fp8_experts(recipe, stage):
    from deepspeed_b200.ops import linear, native
    calls = {"n": 0}
    real = linear._FP8RaggedSwiGLUFn.apply

    def node(*a):
        assert a[-1] is True, "the FP8 experts run the wgmma kernels"
        calls["n"] += 1
        return real(*a)

    linear._FP8RaggedSwiGLUFn.apply = node
    before = native.launch_count
    losses = _engine_losses(recipe, stage, False, False)
    assert calls["n"] > 0 and native.launch_count > before
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0] - 0.5, losses
    # experts only: w13 / w2 are their unit's last gradients, so marking them ready reduces the unit (ZeRO-3 releases
    # its weights; the fused step rewrites them): the step fused into backward gives the two-phase step's losses
    fused = _engine_losses(recipe, stage, True, False)
    two_phase = _engine_losses(recipe, stage, True, True)
    for a, b in zip(fused, two_phase):
        assert abs(a - b) <= 2e-3 * abs(b), (fused, two_phase)
    print(f"[fp8 experts engine] {recipe} ZeRO-{stage}: {losses}")


@pytest.mark.parametrize("stage", [2, 3])
@pytest.mark.parametrize("recipe", RECIPES)
def test_mixtral_fp8_experts_engine_trains(recipe, stage):
    run_distributed(_engine_fp8_experts, 1, (recipe, stage), timeout=600)


# Final losses (mean of the last 10 of 120 steps) on the bigram stream of the FP8 Llama tests, 2-layer Mixtral-shaped model
# (H 256, I 256, 4 experts, top-2, dropless), ZeRO-3.  Measured on an H100 80GB HBM3 at 700 W: bf16 3.0959, tensorwise
# 3.2011, blockwise 3.1163 (entropy floor 2.535).  Blockwise keeps the FP8 Llama tests' tolerance against bf16; tensorwise
# experts, whose activations, gradients and stacked weights share one scale across all experts, end 0.105 above bf16, so
# they are held to a wider bound that still catches a recipe that stops learning.
CONVERGENCE_GAP = 0.1
TENSORWISE_CONVERGENCE_GAP = 0.15


def _convergence():
    import deepspeed_b200 as ds
    batches, floor = _bigram_batches(120)
    finals = {}
    for recipe in (None, "tensorwise", "blockwise"):
        model = _mixtral(recipe, vocab=256)
        cfg = {"train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
               "optimizer": {"type": "AdamW", "params": {"lr": 2e-3}}, "zero_optimization": {"stage": 3}}
        engine, _, _, _ = ds.initialize(model=model, config=cfg)
        losses = []
        for ids in batches:
            ids = ids.cuda()
            loss = engine(ids, labels=ids)
            engine.backward(loss)
            engine.step()
            losses.append(float(loss))
        finals[recipe or "bf16"] = sum(losses[-10:]) / 10
        del engine
    print(f"[fp8 experts convergence] bf16 {finals['bf16']:.4f} tensorwise {finals['tensorwise']:.4f} "
          f"blockwise {finals['blockwise']:.4f} entropy floor {floor:.4f}")
    assert finals["bf16"] < math.log(256) - 1.0, finals
    assert abs(finals["blockwise"] - finals["bf16"]) <= CONVERGENCE_GAP, finals
    assert abs(finals["tensorwise"] - finals["bf16"]) <= TENSORWISE_CONVERGENCE_GAP, finals


def test_fp8_experts_convergence_matches_bf16():
    run_distributed(_convergence, 1, (), timeout=900)
