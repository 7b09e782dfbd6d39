"""GPU tier: the wgmma GEMM (``csrc/cuda/gemm_sm90.cu``) and its front door (``ops/gemm.py``).

Two kinds of check, both per element:

* exact -- operands from :func:`tests.numerics.exact_grid` keep every fp32 partial sum exact, so a correct kernel's
  output is bit-equal to the float64 product rounded once to bf16, whatever its summation order.  Every row and column
  has its own scale, so a value stored in the wrong row, column or tile cannot pass.  cuBLAS must be bit-equal on the
  same data, which checks the premise itself;
* bounded -- random-normal operands against float64 with :func:`tests.numerics.gemm_bound`, which holds only for an fp32
  accumulation.

Operands are views into NaN-filled buffers (a read outside an operand's extent makes C NaN), and outputs are views inside
NaN-filled guard bands on all four sides (a write outside the view changes a guard; an element inside left unwritten
stays NaN).
"""
import json
import os
import zlib

import pytest
import torch

from deepspeed_b200.ops import gemm
from deepspeed_b200.ops.kernels import gemm_sm100 as K
from deepspeed_b200.ops.native import NativeOpError
from tests.numerics import (assert_bits_equal, assert_gemm_bounded, assert_gemm_exact, assert_within, dswiglu_reference,
                            exact_addend, exact_grid, gemm_accum_error, gemm_reference, swiglu_reference, ulp)

pytestmark = pytest.mark.gpu

NAN = float("nan")
BF16 = torch.bfloat16
STORE, ACCUM, SWIGLU, DSWIGLU = K.EPI_STORE, K.EPI_ACCUM, K.EPI_SWIGLU, K.EPI_DSWIGLU
_TABLE = os.path.join(os.path.dirname(gemm.__file__), "gemm_table.json")
with open(_TABLE) as _f:
    STEP_KEYS = sorted(json.load(_f)["shapes"])


def _gen(*seed):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(seed).encode()))


def _randn(rows, cols, gen, scale=1.0):
    return (torch.randn(rows, cols, generator=gen, device="cuda") * scale).to(BF16)


def poisoned(t, top=8, left=8, bottom=64, right=64):
    """``t`` copied into a view of a NaN-filled buffer: ``bottom`` rows past the last row and ``right`` elements past
    every row hold NaN, so a read beyond the view's extent (a K tail, M / N padding) reaches the result.  ``left`` is a
    multiple of 8 and the row stride is rounded up to one, so the view stays 16-byte aligned."""
    R, C = t.shape
    right += (-(left + C + right)) % 8
    buf = torch.full((top + R + bottom, left + C + right), NAN, dtype=t.dtype, device=t.device)
    v = buf[top:top + R, left:left + C]
    v.copy_(t)
    return v


class Guarded:
    """An ``[R, C]`` bf16 output view inside a NaN-filled buffer with guard bands on all four sides (wide enough to
    hold the rest of a 128 x 256 tile), optionally initialised with ``fill``."""

    def __init__(self, R, C, fill=None, top=8, left=8, bottom=136, right=264):
        right += (-(left + C + right)) % 8
        self.buf = torch.full((top + R + bottom, left + C + right), NAN, dtype=BF16, device="cuda")
        self.rs, self.cs = slice(top, top + R), slice(left, left + C)
        self.view = self.buf[self.rs, self.cs]
        if fill is not None:
            self.view.copy_(fill)
        self.before = self.buf.clone()

    def check_guards(self, what):
        """Every element outside the view keeps its bit pattern."""
        after = self.buf.clone()
        after[self.rs, self.cs] = self.before[self.rs, self.cs]
        assert_bits_equal(after, self.before, f"{what}: guard band")

    def check_untouched(self, what):
        """A refused call wrote nothing at all."""
        assert_bits_equal(self.buf, self.before, f"{what}: output written by a refused call")


def operands(M, N, Kd, a_mn, b_mn, gen, exact=True, pad=True):
    """Exact-grid (or random-normal) ``A [M, K]`` and ``B [N, K]``, stored K-major or MN-major (``[K, M]`` / ``[K, N]``)
    as the kernel is told.  Returns ``(a, b, A, B, ea, eb)``: the stored tensors, the logical views of them the
    reference multiplies, and the row exponents of the exact grid (None for random data)."""
    if exact:
        A, ea = exact_grid(M, Kd, gen)
        B, eb = exact_grid(N, Kd, gen)
    else:
        (A, B), ea, eb = (_randn(M, Kd, gen), _randn(N, Kd, gen)), None, None
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    if pad:
        a, b = poisoned(a), poisoned(b)
    return a, b, (a.t() if a_mn else a), (b.t() if b_mn else b), ea, eb


def assert_cublas_exact(A, B, what):
    """The exactness premise: cuBLAS on the same exact-grid operands is bit-equal to the once-rounded exact product."""
    assert_gemm_exact(torch.mm(A, B.t()), A, B, what=f"{what}: cuBLAS control (the exact-grid premise)")


def run_exact(M, N, Kd, a_mn, b_mn, epi, gen, sms=0, group_m=8, control=True):
    """One STORE / ACCUM launch on poisoned exact-grid operands into a guarded output, checked bit for bit."""
    a, b, A, B, ea, eb = operands(M, N, Kd, a_mn, b_mn, gen)
    c_old = exact_addend(ea, eb, gen) if epi == ACCUM else None
    out = Guarded(M, N, fill=c_old)
    K.matmul_2cta(a, b, bool(a_mn), bool(b_mn), out=out.view, epi=epi, sms=sms, group_m=group_m)
    what = f"a_mn={a_mn} b_mn={b_mn} epi={epi} {M}x{N}x{Kd} sms={sms} group_m={group_m}"
    assert_gemm_exact(out.view, A, B, c_old, what=what)
    out.check_guards(what)
    if control:
        assert_cublas_exact(A, B, what)


# ---------------------------------------------------------------------------------------------------------------------
# 1. exact oracle: layouts, epilogues, edges
# ---------------------------------------------------------------------------------------------------------------------
# (M, N, K) covering M in {8, 64, 127, 128, 129, 255, 257, 1000}, N in {8, 120, 128, 136, 256, 264, 520} and
# K in {8, 16, 56, 64, 72, 200, 264}; an MN-major A needs M % 8 == 0
_SHAPES = [(8, 8, 8), (64, 120, 16), (127, 128, 56), (128, 136, 64), (129, 256, 72), (255, 264, 200), (257, 520, 264),
           (1000, 8, 72), (127, 520, 8), (129, 120, 264), (1000, 264, 56), (64, 256, 200), (257, 136, 16), (255, 8, 64),
           (128, 520, 264), (8, 264, 200)]
_SHAPES_MN_A = [(8, 8, 8), (64, 120, 16), (128, 128, 56), (128, 136, 64), (1000, 256, 72), (64, 264, 200), (8, 520, 264),
                (1000, 8, 264), (128, 520, 8), (1000, 136, 200)]
_LAYOUT_CASES = [(a_mn, b_mn) + s for a_mn in (0, 1) for b_mn in (0, 1) for s in (_SHAPES_MN_A if a_mn else _SHAPES)]


@pytest.mark.parametrize("epi", [STORE, ACCUM])
@pytest.mark.parametrize("a_mn,b_mn,M,N,Kd", _LAYOUT_CASES)
def test_gemm_layouts_exact(a_mn, b_mn, M, N, Kd, epi):
    """All four operand layouts with STORE and ACCUM: partial M / N tiles, K tails, one-tile and many-tile problems.
    ACCUM's reference adds C_old to the exact sum and rounds once: rounding the accumulator first fails."""
    run_exact(M, N, Kd, a_mn, b_mn, epi, _gen(a_mn, b_mn, M, N, Kd, epi))


@pytest.mark.parametrize("shape", [(128, 256, 64), (256, 512, 128), (384, 768, 320), (1000, 1000, 264),
                                   (2048, 6144, 4096), (4096, 4096, 14336)])
def test_gemm_nt_matches_fp32(shape):
    """The plain NT entry point (``dsb_gemm_nt_bf16``, column-major tile order): exact on the grid, bounded on random
    data."""
    M, N, Kd = shape
    gen = _gen("nt", *shape)
    for exact in (True, False):
        a, b, A, B, _, _ = operands(M, N, Kd, 0, 0, gen, exact=exact)
        out = Guarded(M, N)
        K.matmul_nt(a, b, out=out.view)
        (assert_gemm_exact if exact else assert_gemm_bounded)(out.view, A, B, what=f"nt {shape} exact={exact}")
        out.check_guards(f"nt {shape}")
        if exact:
            assert_cublas_exact(A, B, f"nt {shape}")


def test_gemm_strided_views_and_fewer_sms():
    """Row-strided operand views (stride 1024, K = 512 and a K tail of 456) on 7 CTAs."""
    gen = _gen("strided")
    big_a, _ = exact_grid(512, 1024, gen)
    big_b, _ = exact_grid(1024, 1024, gen)
    for k0, k1 in ((128, 640), (136, 592)):
        a, b = big_a[:, k0:k1], big_b[:, k0 + 120:k1 + 120]
        assert K.supports(a, b)
        out = Guarded(512, 1024)
        K.matmul_nt(a, b, out=out.view, sms=7)
        assert_gemm_exact(out.view, a, b, what=f"strided K={k1 - k0}")
        out.check_guards("strided")


@pytest.mark.parametrize("shape", [(256, 256, 64), (128, 256, 64), (512, 512, 128), (384, 768, 320), (1000, 1000, 264),
                                   (2048, 6144, 4096), (4096, 4096, 14336), (8192, 28672, 4096)])
def test_gemm_2cta_matches_fp32(shape):
    """General entry point (``dsb_gemm_nt_bf16_2cta``), M / N edges included: exact, then bounded and bit-identical over
    repeated launches on random data."""
    M, N, Kd = shape
    gen = _gen("2cta", *shape)
    a, b, A, B, _, _ = operands(M, N, Kd, 0, 0, gen, pad=M * Kd < 2**25)
    out = Guarded(M, N)
    K.matmul_nt_2cta(a, b, out=out.view)
    assert_gemm_exact(out.view, A, B, what=f"2cta {shape}")
    out.check_guards(f"2cta {shape}")
    del a, b, A, B, out
    a, b, A, B, _, _ = operands(M, N, Kd, 0, 0, gen, exact=False, pad=False)
    c = K.matmul_nt_2cta(a, b)
    assert_gemm_bounded(c, A, B, what=f"2cta {shape} random")
    for _ in range(3):
        assert_bits_equal(K.matmul_nt_2cta(a, b), c, f"2cta {shape} relaunch")


@pytest.mark.parametrize("shape", [(256, 256, 64), (512, 384, 192), (1000, 520, 264), (8192, 4096, 6144), (4096, 14336, 8192)])
def test_gemm_2cta_nn_tn_match_cublas(shape):
    """NN (dX = dY W) and TN (dW = dY^T X) through ``matmul_nn`` / ``matmul_tn``, into guarded views of larger buffers."""
    M, N, Kd = shape
    gen = _gen("nntn", *shape)
    for a_mn, fn in ((0, K.matmul_nn), (1, K.matmul_tn)):
        a, b, A, B, _, _ = operands(M, N, Kd, a_mn, 1, gen, pad=M * Kd < 2**25)
        out = Guarded(M, N)
        fn(a, b, out=out.view)
        what = f"a_mn={a_mn} b_mn=1 {shape}"
        assert_gemm_exact(out.view, A, B, what=what)
        out.check_guards(what)
        assert_cublas_exact(A, B, what)
        del a, b, A, B, out
        a, b, A, B, _, _ = operands(M, N, Kd, a_mn, 1, gen, exact=False, pad=False)
        assert_gemm_bounded(fn(a, b), A, B, what=what + " random")


@pytest.mark.parametrize("shape", [(512, 384, 256), (1000, 520, 264), (6144, 4096, 8192)])
def test_gemm_2cta_accumulate_epilogue(shape):
    """EPI_ACCUM, C += A^T B (the dW accumulation of micro-batch 2..GAS) and C += A B^T: exact, then bounded."""
    M, N, Kd = shape
    gen = _gen("acc", *shape)
    for a_mn, b_mn in ((1, 1), (0, 0)):
        run_exact(M, N, Kd, a_mn, b_mn, ACCUM, gen, control=False)
        a, b, A, B, _, _ = operands(M, N, Kd, a_mn, b_mn, gen, exact=False, pad=False)
        c_old = _randn(M, N, gen, 8.0)
        c = c_old.clone()
        K.matmul_2cta(a, b, bool(a_mn), bool(b_mn), out=c, epi=ACCUM)
        assert_gemm_bounded(c, A, B, c_old, what=f"accum {a_mn}{b_mn} {shape} random")


# ---------------------------------------------------------------------------------------------------------------------
# fused SwiGLU / dSwiGLU epilogues
# ---------------------------------------------------------------------------------------------------------------------
def _check_swiglu(act, gu, x, w, I, exact, what):
    """gate|up (when saved) against the product, act against :func:`swiglu_reference` of the fp32 accumulators."""
    Kd = x.shape[1]
    if gu is not None:
        (assert_gemm_exact if exact else assert_gemm_bounded)(gu, x, w, what=f"{what} gate|up")
    blocks = zip(gemm_reference(x, w[:I], magnitudes=not exact), gemm_reference(x, w[I:], magnitudes=not exact))
    for (rs, cs, g, mg), (_, _, u, mu) in blocks:
        err = (0.0, 0.0) if exact else (gemm_accum_error(mg, Kd), gemm_accum_error(mu, Kd))
        ref, bound = swiglu_reference(g, u, *err)
        assert_within(act[rs, cs], ref, bound, f"{what} act[{rs.start}:, {cs.start}:]")


def run_swiglu(T, H, I, gen, exact=True, pad=True, save=True, sms=0):
    if exact:  # scales up to 2**0: |gate| stays small enough for silu's (|g| + 8) U relative bound to bite
        x, _ = exact_grid(T, H, gen, -6, 0)
        w, _ = exact_grid(2 * I, H, gen, -6, 0)
    else:
        x, w = _randn(T, H, gen, 0.5), _randn(2 * I, H, gen, H**-0.5)
    if pad:
        x, w = poisoned(x), poisoned(w)
    act = Guarded(T, I)
    gu = Guarded(T, 2 * I) if save else None
    K.matmul_2cta(x, w, False, False, out=act.view, epi=SWIGLU, out2=gu.view if save else None, inter=I, sms=sms)
    what = f"swiglu T={T} H={H} I={I} exact={exact}"
    _check_swiglu(act.view, gu.view if save else None, x, w, I, exact, what)
    act.check_guards(what + " act")
    if save:
        gu.check_guards(what + " gate|up")
    return x, w, act.view


@pytest.mark.parametrize("T,H,I", [(256, 128, 128), (1000, 320, 384), (4096, 4096, 14336), (127, 72, 128), (129, 8, 256),
                                   (8, 264, 384)])
def test_gemm_swiglu_epilogue(T, H, I):
    """EPI_SWIGLU: gate|up saved from the accumulators bit-exact, act = silu(gate) * up from the fp32 accumulators; the
    launch without the save writes the same act."""
    gen = _gen("swiglu", T, H, I)
    x, w, act = run_swiglu(T, H, I, gen)
    act2 = Guarded(T, I)
    K.matmul_2cta(x, w, False, False, out=act2.view, epi=SWIGLU, inter=I)
    assert_bits_equal(act2.view, act, "swiglu without the save")
    act2.check_guards("swiglu without the save")
    run_swiglu(T, H, I, gen, exact=False, pad=False)


def _check_dswiglu(dgu, dy, B, aux, I, exact, what):
    Kd = dy.shape[1]
    for rs, cs, d, mag in gemm_reference(dy, B, magnitudes=not exact):
        d_err = 0.0 if exact else gemm_accum_error(mag, Kd)
        g, u = aux[rs, cs], aux[rs, I + cs.start:I + cs.stop]
        dgate, dgate_bound, dup, dup_bound = dswiglu_reference(d, g, u, d_fp32=True, d_err=d_err)
        assert_within(dgu[rs, cs], dgate, dgate_bound, f"{what} dgate[{rs.start}:, {cs.start}:]")
        assert_within(dgu[rs, I + cs.start:I + cs.stop], dup, dup_bound, f"{what} dup[{rs.start}:, {cs.start}:]")


def run_dswiglu(T, H, I, b_mn, gen, exact=True, pad=True):
    """dgate|dup = dSwiGLU(dY W_down, gate|up); W_down stored [H, I] (MN-major, the step's form) or [I, H]."""
    a, b, dy, B, _, _ = operands(T, I, H, 0, b_mn, gen, exact=exact, pad=pad)
    aux = _randn(T, 2 * I, gen, 2.0)
    if pad:
        aux = poisoned(aux)
    dgu = Guarded(T, 2 * I)
    K.matmul_2cta(a, b, False, bool(b_mn), out=dgu.view[:, :I], epi=DSWIGLU, aux=aux, out2=dgu.view, inter=I)
    what = f"dswiglu T={T} H={H} I={I} b_mn={b_mn} exact={exact}"
    _check_dswiglu(dgu.view, dy, B, aux, I, exact, what)
    dgu.check_guards(what)


@pytest.mark.parametrize("T,H,I", [(256, 128, 256), (1000, 320, 392), (4096, 4096, 14336), (127, 72, 136), (129, 8, 8)])
def test_gemm_dswiglu_epilogue(T, H, I):
    """EPI_DSWIGLU with W_down stored [H, I] (the step's form) and [I, H]: the accumulator dY W_down is exact on the
    grid, so only the epilogue's arithmetic is bounded (dswiglu_reference with an fp32 d); then random data."""
    for b_mn in (1, 0):
        gen = _gen("dswiglu", T, H, I, b_mn)
        run_dswiglu(T, H, I, b_mn, gen)
        run_dswiglu(T, H, I, b_mn, gen, exact=False, pad=False)


# ---------------------------------------------------------------------------------------------------------------------
# persistent schedule and rasterisation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Kd", [8, 136, 256, 264, 520])  # num_k = 1, 3, 4, 5, 9 against a 4-stage ring
@pytest.mark.parametrize("sms", [1, 2, 3, 7])
def test_persistent_schedule_exact(sms, Kd):
    """24 tiles (8 x 3) on 1-7 persistent CTAs, so the ring's stage and phase wrap across tile boundaries, under every
    rasterisation: column-major (0), 1, a ragged last group (3 of 8 m-blocks), 8 and more than num_m."""
    a_mn, b_mn = [(0, 0), (0, 1), (1, 1), (1, 0)][(sms + Kd) % 4]
    for group_m in (0, 1, 3, 8, 11):
        run_exact(1000, 520, Kd, a_mn, b_mn, STORE, _gen("sched", sms, Kd, group_m), sms=sms, group_m=group_m,
                  control=False)


@pytest.mark.parametrize("group_m", [0, 1, 3, 8, 20])
def test_gemm_2cta_rasterisation_groups(group_m):
    """Grouped (L2 super-block) tile order visits every tile exactly once: 15 x 6 tiles, a ragged last group and edge
    tiles."""
    run_exact(256 * 7 + 40, 256 * 5 + 24, 192, 0, 0, STORE, _gen("raster", group_m), group_m=group_m, control=False)


@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1), (1, 0)])
def test_grid_independence_random(a_mn, b_mn):
    """Each tile's K loop runs in one CTA in a fixed order, so C is bit-identical whatever the CTA count, the
    rasterisation and the launch: any difference is a race or a phase bug."""
    M, N, Kd = 1832, 1304, 520
    a, b, A, B, _, _ = operands(M, N, Kd, a_mn, b_mn, _gen("grid", a_mn, b_mn), exact=False)
    c = K.matmul_2cta(a, b, bool(a_mn), bool(b_mn))
    assert_gemm_bounded(c, A, B, what=f"grid {a_mn}{b_mn}")
    for sms in (0, 1, 3, 7):
        for group_m in (0, 1, 3, 8, 20):
            for _ in range(2 if sms == 0 else 1):
                c2 = K.matmul_2cta(a, b, bool(a_mn), bool(b_mn), sms=sms, group_m=group_m)
                assert_bits_equal(c2, c, f"grid {a_mn}{b_mn} sms={sms} group_m={group_m}")


# ---------------------------------------------------------------------------------------------------------------------
# grouped (MoE) form
# ---------------------------------------------------------------------------------------------------------------------
def run_grouped(counts, N, Kd, gen, lead=0, tail=0, sms=0):
    """Experts' rows ``[lead, lead + sum(counts))`` of ``lead + sum(counts) + tail`` rows; the rows outside hold NaN in x
    and must stay untouched in the output."""
    E, n = len(counts), sum(counts)
    rows = lead + n + tail
    x = torch.full((rows, Kd), NAN, dtype=BF16, device="cuda")
    x[lead:lead + n] = exact_grid(n, Kd, gen)[0]
    x = poisoned(x)
    w = torch.stack([exact_grid(N, Kd, gen)[0] for _ in range(E)])
    off = torch.tensor([lead] + [lead + int(s) for s in torch.tensor(counts).cumsum(0)], dtype=torch.int32, device="cuda")
    assert K.supports_grouped(x, w, off)
    out = Guarded(rows, N)
    K.grouped_matmul_nt(x, w, off, out=out.view, sms=sms)
    what = f"grouped E={E} N={N} K={Kd} lead={lead} tail={tail}"
    s = lead
    for e, c in enumerate(counts):
        if c:
            assert_gemm_exact(out.view[s:s + c], x[s:s + c], w[e], what=f"{what} expert {e}")
        s += c
    out.view[lead:lead + n] = out.before[out.rs, out.cs][lead:lead + n]
    out.check_untouched(f"{what}: rows outside the experts, or the guard band,")


@pytest.mark.parametrize("counts", [[300, 0, 17, 128, 1, 513], [0, 0, 5, 0], [256, 256]])
@pytest.mark.parametrize("N,K", [(512, 256), (328, 192), (136, 72)])
def test_grouped_gemm_matches_per_expert_loop(counts, N, K):
    """Device-driven grouped GEMM: ragged expert extents incl. empty experts, N not a tile multiple, a K tail."""
    run_grouped(counts, N, K, _gen("grouped", tuple(counts), N, K))


def test_grouped_gemm_offsets_inside_rows():
    """offsets[0] > 0 and offsets[E] < rows: the rows before and after the experts stay untouched."""
    gen = _gen("grouped-inside")
    run_grouped([130, 0, 7, 260], 328, 136, gen, lead=37, tail=90)
    run_grouped([5, 300], 136, 64, gen, lead=128, tail=1, sms=3)


def test_grouped_gemm_256_experts():
    """E at its limit of 256, most experts empty, on a few CTAs."""
    gen = _gen("grouped-256")
    counts = [0] * 256
    for e, c in ((0, 3), (17, 129), (128, 1), (200, 256), (255, 77)):
        counts[e] = c
    run_grouped(counts, 136, 64, gen, lead=8, tail=8, sms=5)


# ---------------------------------------------------------------------------------------------------------------------
# the training step's shapes (every key of gemm_table.json, on the in-tree kernel whatever the table chooses)
# ---------------------------------------------------------------------------------------------------------------------
def _free():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("key", STEP_KEYS)
def test_step_shapes(key):
    form, dims = key.split(":")
    M, N, Kd = (int(v) for v in dims.split("x"))
    gen = _gen("step", key)
    if form == "nt_swiglu":
        run_swiglu(M, Kd, N, gen, pad=False)
        _free()
        run_swiglu(M, Kd, N, gen, exact=False, pad=False)
    elif form == "nn_dswiglu":
        run_dswiglu(M, Kd, N, 1, gen, pad=False)
        _free()
        run_dswiglu(M, Kd, N, 1, gen, exact=False, pad=False)
    else:
        a_mn, b_mn = {"nt": (0, 0), "nn": (0, 1), "tn": (1, 1), "tn_acc": (1, 1)}[form]
        epi = ACCUM if form == "tn_acc" else STORE
        a, b, A, B, ea, eb = operands(M, N, Kd, a_mn, b_mn, gen, pad=False)
        c_old = exact_addend(ea, eb, gen) if epi == ACCUM else None
        out = Guarded(M, N, fill=c_old)
        K.matmul_2cta(a, b, bool(a_mn), bool(b_mn), out=out.view, epi=epi)
        assert_gemm_exact(out.view, A, B, c_old, what=key)
        out.check_guards(key)
        if epi == STORE:
            assert_cublas_exact(A, B, key)
        del a, b, A, B, out, c_old
        _free()
        a, b, A, B, _, _ = operands(M, N, Kd, a_mn, b_mn, gen, exact=False, pad=False)
        c_old = _randn(M, N, gen, 4.0) if epi == ACCUM else None
        c = c_old.clone() if epi == ACCUM else None
        c = K.matmul_2cta(a, b, bool(a_mn), bool(b_mn), out=c, epi=epi)
        assert_gemm_bounded(c, A, B, c_old, what=f"{key} random")
    _free()


# ---------------------------------------------------------------------------------------------------------------------
# 3. refused arguments: NativeOpError, nothing written
# ---------------------------------------------------------------------------------------------------------------------
def _in(rows, cols, width=None, col0=0):
    """A ``[rows, cols]`` random view at column ``col0`` of a ``[rows, width]`` buffer."""
    width = width or cols
    return torch.randn(rows, width, device="cuda").to(BF16)[:, col0:col0 + cols]


def _refusal(case):
    """-> (call(out, out2), out, out2 | None); each output is ``(rows, cols, width, col0)``: a view at column ``col0``
    of a ``[rows, width]`` buffer."""
    M, N, Kd = 256, 256, 128
    a, b, bm = _in(M, Kd), _in(N, Kd), _in(Kd, N)
    c, c2 = (M, N, N, 0), (M, 2 * N, 2 * N, 0)
    x2 = lambda *args, **kw: (lambda o, o2: K.matmul_2cta(*args, out=o, out2=o2, **kw))
    grouped = lambda x, w, off: (lambda o, o2: K.grouped_matmul_nt(x, w, off, out=o))
    w3 = lambda n, k: torch.randn(3, n, k, device="cuda").to(BF16)
    off = torch.tensor([0, 100, 200, 256], dtype=torch.int32, device="cuda")
    cases = {
        "a_misaligned": lambda: (x2(_in(M, Kd, Kd + 8, 1), b, False, False), c),
        "b_misaligned": lambda: (x2(a, _in(N, Kd, Kd + 8, 1), False, False), c),
        "c_misaligned": lambda: (x2(a, b, False, False), (M, N, N + 8, 1)),
        "lda": lambda: (x2(_in(M, Kd, Kd + 4), b, False, False), c),
        "ldb": lambda: (x2(a, _in(Kd, N, N + 4), False, True), c),
        "ldc": lambda: (x2(a, b, False, False), (M, N, N + 4, 0)),
        "n_mod8": lambda: (x2(a, _in(124, Kd), False, False), (M, 124, 128, 0)),
        "k_mod8": lambda: (x2(_in(M, 100, 104), _in(N, 100, 104), False, False), c),
        "m_mod8_mn_a": lambda: (x2(_in(Kd, 129, 136), b, True, False), (129, N, N, 0)),
        "swiglu_inter": lambda: (x2(a, _in(272, Kd), False, False, epi=SWIGLU, inter=136), (M, 136, 136, 0),
                                 (M, 272, 272, 0)),
        "swiglu_mn_a": lambda: (x2(_in(Kd, M), _in(2 * N, Kd), True, False, epi=SWIGLU, inter=N), c, c2),
        "swiglu_mn_b": lambda: (x2(a, _in(Kd, 2 * N), False, True, epi=SWIGLU, inter=N), c, c2),
        "dswiglu_no_aux": lambda: (x2(a, bm, False, True, epi=DSWIGLU, inter=N), c, c2),
        "nt_misaligned": lambda: ((lambda o, o2: K.matmul_nt(_in(M, Kd, Kd + 8, 1), b, out=o)), c),
        "nt_n_mod8": lambda: ((lambda o, o2: K.matmul_nt(a, _in(124, Kd), out=o)), (M, 124, 128, 0)),
        "nt_2cta_lda": lambda: ((lambda o, o2: K.matmul_nt_2cta(_in(M, Kd, Kd + 4), b, out=o)), c),
        "grouped_k_mod8": lambda: (grouped(_in(M, 100, 104), w3(N, 100), off), c),
        "grouped_e257": lambda: (grouped(a, torch.randn(257, 8, Kd, device="cuda").to(BF16),
                                         torch.zeros(258, dtype=torch.int32, device="cuda")), (M, 8, 8, 0)),
        "grouped_n_mod8": lambda: (grouped(a, w3(124, Kd), off), (M, 124, 128, 0)),
        "grouped_misaligned": lambda: (grouped(_in(M, Kd, Kd + 8, 1), w3(N, Kd), off), c),
        "grouped_lda": lambda: (grouped(_in(M, Kd, Kd + 4), w3(N, Kd), off), c),
    }
    return cases[case]()


_REFUSALS = ["a_misaligned", "b_misaligned", "c_misaligned", "lda", "ldb", "ldc", "n_mod8", "k_mod8", "m_mod8_mn_a",
             "swiglu_inter", "swiglu_mn_a", "swiglu_mn_b", "dswiglu_no_aux", "nt_misaligned", "nt_n_mod8", "nt_2cta_lda",
             "grouped_k_mod8", "grouped_e257", "grouped_n_mod8", "grouped_misaligned", "grouped_lda"]


@pytest.mark.parametrize("case", _REFUSALS)
def test_refused_arguments_raise_and_write_nothing(case):
    """Every -2 / -3 condition of ``dsb_gemm_bf16_2cta_ex``, ``dsb_gemm_nt_bf16`` and ``dsb_gemm_grouped_nt_bf16``."""
    torch.manual_seed(0)
    call, *specs = _refusal(case)
    bufs = [torch.full((rows, width), NAN, dtype=BF16, device="cuda") for rows, _, width, _ in specs]
    before = [t.clone() for t in bufs]
    views = [t[:, col0:col0 + cols] for t, (_, cols, _, col0) in zip(bufs, specs)]
    with pytest.raises(NativeOpError):
        call(views[0], views[1] if len(views) > 1 else None)
    torch.cuda.synchronize()
    for t, t0, what in zip(bufs, before, ("out", "out2")):
        assert_bits_equal(t, t0, f"{case}: {what} written by a refused call")


# ---------------------------------------------------------------------------------------------------------------------
# 4. front door (ops/gemm.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def backend(request, monkeypatch):
    """Select a backend for one test without leaving backend or choice state behind."""
    monkeypatch.setattr(gemm, "_backend", request.param)
    monkeypatch.setattr(gemm, "_used", {})
    monkeypatch.setattr(gemm, "_measured", {})
    return request.param


@pytest.mark.parametrize("backend", ["own", "lib"], indirect=True)
def test_front_door_exact(backend):
    """matmul_nt / nn / tn (with and without accumulate): own, lib and the exact reference are bit-equal, except that
    the library's accumulate (``addmm_`` into a bf16 C) rounds the product to bf16 before adding it, so it is bounded
    by that extra rounding; the fused ACCUM epilogue adds to the fp32 accumulator and rounds once."""
    M, N, Kd = 512, 384, 256
    gen = _gen("front", backend)
    for form, (a_mn, b_mn) in (("nt", (0, 0)), ("nn", (0, 1)), ("tn", (1, 1)), ("tn_acc", (1, 1))):
        a, b, A, B, ea, eb = operands(M, N, Kd, a_mn, b_mn, gen, pad=False)
        if form == "nt":
            c = gemm.matmul_nt(a, b)
        elif form == "nn":
            c = gemm.matmul_nn(a, b)
        elif form == "tn":
            c = gemm.matmul_tn(a, b)
        c_old = exact_addend(ea, eb, gen) if form == "tn_acc" else None
        if form == "tn_acc":
            c = c_old.clone()
            gemm.matmul_tn(a, b, out=c, accumulate=True)
        if form == "tn_acc" and backend == "lib":
            (_, _, p, _), = gemm_reference(A, B)
            ref = p + c_old.double()
            assert_within(c, ref, ulp(p, BF16) / 2 + ulp(ref.abs() + ulp(p, BF16), BF16), "lib tn_acc")
        else:
            assert_gemm_exact(c, A, B, c_old, what=f"{backend} {form}")
        key = f"{form}:{M}x{N}x{Kd}"
        assert gemm.tuning_table().get(key) == ("own" if backend == "own" else None), (key, gemm.tuning_table())


@pytest.mark.parametrize("save", [True, False])
@pytest.mark.parametrize("backend", ["own", "lib"], indirect=True)
def test_front_door_swiglu(backend, save):
    """gate_up_swiglu and down_dx_dswiglu.  gate|up is exact either way.  The fused epilogue applies silu to the fp32
    accumulators (exact here); the library path applies it to the bf16 gate|up it stored, and its dSwiGLU to the bf16
    dY W_down -- each is bounded from what it read."""
    T, H, I = 512, 256, 384
    gen = _gen("front-swiglu", backend, save)
    x, _ = exact_grid(T, H, gen)
    w_gu, _ = exact_grid(2 * I, H, gen)
    act, gu = gemm.gate_up_swiglu(x, w_gu, save_gate_up=save)
    if save:
        assert_gemm_exact(gu, x, w_gu, what=f"{backend} gate|up")
    else:
        assert gu is None
    (_, _, g, _), = gemm_reference(x, w_gu[:I])
    (_, _, u, _), = gemm_reference(x, w_gu[I:])
    if backend == "lib":
        g, u = g.to(BF16), u.to(BF16)
    ref, bound = swiglu_reference(g, u)
    assert_within(act, ref, bound, f"{backend} act")

    dy, _ = exact_grid(T, H, gen)
    wd_t, _ = exact_grid(I, H, gen)  # W_down^T: the [I, H] logical B of dY @ W_down
    w_down = wd_t.t().contiguous()
    aux = _randn(T, 2 * I, gen, 2.0)
    dgu = gemm.down_dx_dswiglu(dy, w_down, aux)
    (_, _, d, _), = gemm_reference(dy, wd_t)
    fused = backend == "own"
    dgate, dgate_bound, dup, dup_bound = dswiglu_reference(d if fused else d.to(BF16), aux[:, :I], aux[:, I:], d_fp32=fused)
    assert_within(dgu[:, :I], dgate, dgate_bound, f"{backend} dgate")
    assert_within(dgu[:, I:], dup, dup_bound, f"{backend} dup")
    used = gemm.tuning_table()
    assert used.get(f"nt_swiglu:{T}x{I}x{H}") == ("own" if fused else None), used
    assert used.get(f"nn_dswiglu:{T}x{I}x{H}") == ("own" if fused else None), used


def _ineligible(case, gen):
    """-> (front-door call, torch.mm of the same inputs)."""
    e = lambda r, c: exact_grid(r, c, gen)[0]
    if case == "nt_n50257":
        a, b = e(256, 64), e(50257, 64)
    elif case == "nt_m128":
        a, b = e(128, 256), e(384, 256)
    elif case == "nt_k32":
        a, b = e(512, 32), e(384, 32)
    elif case == "nt_k100":
        a, b = e(512, 100), e(384, 100)
    elif case == "nt_offset_view":
        a, b = e(512, 264)[:, 1:257], e(384, 256)
    elif case in ("nt_fp16", "nt_fp32"):
        dt = torch.float16 if case == "nt_fp16" else torch.float32
        a, b = e(512, 256).to(dt), e(384, 256).to(dt)
    elif case == "nt_stride0":
        a, b = e(1, 256).expand(512, 256), e(384, 256)
    if case.startswith("nt_"):
        return (lambda: gemm.matmul_nt(a, b)), torch.mm(a, b.t())
    if case == "nn_n50257":
        a, b = e(256, 64), e(50257, 64).t().contiguous()
        return (lambda: gemm.matmul_nn(a, b)), torch.mm(a, b)
    if case == "nn_stride0":  # dX of a 2-D flat_linear under y.mean(0): dY is expanded, row stride 0
        a, b = e(1, 384).expand(512, 384), e(256, 384).t().contiguous()
        return (lambda: gemm.matmul_nn(a, b)), torch.mm(a, b)
    if case == "tn_stride0":  # its dW = dY^T X
        a, b = e(1, 384).expand(512, 384), e(256, 512).t().contiguous()
        return (lambda: gemm.matmul_tn(a, b)), torch.mm(a.t(), b)
    if case == "tn_m_mod8":
        a, b = e(260, 256).t().contiguous(), e(384, 256).t().contiguous()
        return (lambda: gemm.matmul_tn(a, b)), torch.mm(a.t(), b)
    raise KeyError(case)


@pytest.mark.parametrize("case", ["nt_n50257", "nt_m128", "nt_k32", "nt_k100", "nt_offset_view", "nt_fp16", "nt_fp32",
                                  "nt_stride0", "nn_n50257", "nn_stride0", "tn_stride0", "tn_m_mod8"])
@pytest.mark.parametrize("backend", ["own", "lib", "auto"], indirect=True)
def test_front_door_ineligible_inputs(backend, case):
    """Inputs the in-tree kernel cannot take return what torch.mm returns, and never raise, under every backend."""
    call, want = _ineligible(case, _gen("inelig", case))
    got = call()
    assert_bits_equal(got, want, f"{backend} {case}")


def test_flat_linear_backward_uses_native_gemm_and_matches_autograd(monkeypatch):
    """flat_linear forward and backward on small integers (exact in fp32): bit-equal to autograd."""
    from deepspeed_b200.ops.linear import flat_linear
    monkeypatch.setattr(gemm, "_used", {})
    monkeypatch.setattr(gemm, "_measured", {})
    gen = _gen("flat")
    e = lambda r, c: exact_grid(r, c, gen, emin=0, emax=0)[0]
    x = e(2048, 1024).view(4, 512, 1024).requires_grad_(True)
    w = e(2048, 1024).requires_grad_(True)
    y = flat_linear(x, w)
    g = e(2048, 2048).view(4, 512, 2048)
    y.backward(g)
    xr, wr = x.detach().clone().requires_grad_(True), w.detach().clone().requires_grad_(True)
    yr = torch.nn.functional.linear(xr, wr)
    yr.backward(g)
    for got, ref, what in ((y, yr, "y"), (x.grad, xr.grad, "dx"), (w.grad, wr.grad, "dw")):
        assert_bits_equal(got, ref, what)
    assert any(k.split(":")[0] in ("nn", "tn") for k in gemm.tuning_table())


@pytest.mark.parametrize("backend", ["own", "lib"], indirect=True)
def test_swiglu_mlp_matches_autograd(backend):
    """Fused SwiGLU MLP node (3 GEMM launches per direction, activation in the epilogues) vs plain autograd."""
    from deepspeed_b200.ops.linear import swiglu_mlp
    torch.manual_seed(0)
    T, H, I = 1024, 512, 1280
    x = (torch.randn(2, T // 2, H, device="cuda") * 0.5).bfloat16().requires_grad_(True)
    wg = (torch.randn(2 * I, H, device="cuda") / H**0.5).bfloat16().requires_grad_(True)
    wd = (torch.randn(H, I, device="cuda") / I**0.5).bfloat16().requires_grad_(True)
    y = swiglu_mlp(x, wg, wd)
    gy = torch.randn_like(y)
    y.backward(gy)
    xr, wgr, wdr = (t.detach().float().requires_grad_(True) for t in (x, wg, wd))
    gu = xr @ wgr.t()
    yr = (torch.nn.functional.silu(gu[..., :I]) * gu[..., I:]) @ wdr.t()
    yr.backward(gy.float())
    for got, ref in ((y, yr), (x.grad, xr.grad), (wg.grad, wgr.grad), (wd.grad, wdr.grad)):
        s = ref.float().abs().max().item()
        assert (got.float() - ref.float()).abs().max().item() < 3e-2 * s + 1e-2


def test_grouped_swiglu_experts_match_bmm_reference():
    """MoE training experts: wgmma per-expert fused path vs the batched-GEMM autograd reference."""
    from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
    torch.manual_seed(0)
    E, C, H, I = 2, 512, 256, 384
    ex = GroupedSwiGLUExperts(E, H, I).cuda().bfloat16()
    x = (torch.randn(E, C, H, device="cuda") * 0.5).bfloat16().requires_grad_(True)
    y = ex(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    xr = x.detach().float().requires_grad_(True)
    w13, w2 = ex.w13.detach().float().requires_grad_(True), ex.w2.detach().float().requires_grad_(True)
    gu = torch.bmm(xr, w13.transpose(1, 2))
    yr = torch.bmm(torch.nn.functional.silu(gu[..., :I]) * gu[..., I:], w2.transpose(1, 2))
    yr.backward(gy.float())
    for got, ref in ((y, yr), (x.grad, xr.grad), (ex.w13.grad, w13.grad), (ex.w2.grad, w2.grad)):
        s = ref.abs().max().item()
        assert (got.float() - ref).abs().max().item() < 3e-2 * s + 1e-2
