"""GPU tier: dropless MoE training on the ragged forms of the wgmma GEMM (``dsb_gemm_ragged_bf16``,
``dsb_gemm_ragged_wgrad_bf16``), the autograd node over them (``ops/linear.py`` ``_RaggedSwiGLUFn``) and the dropless
``MOELayer`` / Mixtral path.

Kernel checks use the exact oracle of ``test_gemm_gpu.py``: exact-grid operands, so a correct result is bit-equal to the
float64 product rounded once.  Row operands hold NaN outside the experts' segments (a read there reaches the result) and
sit in NaN-padded buffers; outputs sit inside NaN guard bands, and rows outside the segments must keep their bits.
"""
import math

import pytest
import torch

from deepspeed_b200.ops import gemm
from deepspeed_b200.ops.kernels import gemm_sm100 as K
from deepspeed_b200.ops.native import NativeOpError
from tests.gpu.test_gemm_gpu import Guarded, _check_dswiglu, _check_swiglu, _gen, poisoned
from tests.numerics import assert_bits_equal, assert_gemm_exact, assert_within, exact_addend, exact_grid

pytestmark = pytest.mark.gpu

NAN = float("nan")
BF16 = torch.bfloat16
SMS = (0, 1, 3, 7)


def layout(counts, lead=0, tail=0):
    """Offsets of 64-row aligned segments after ``lead`` rows (a multiple of 64), and the row count with ``tail``."""
    off = [lead]
    for c in counts:
        off.append(off[-1] + -(-c // 64) * 64)
    return off, off[-1] + tail


def dev_offsets(off):
    return torch.tensor(off, dtype=torch.int32, device="cuda")


def segment_rows(counts, off, R, cols, make):
    """``[R, cols]`` row operand: expert e's ``counts[e]`` rows from ``make(c)``, zeros on its padding, NaN elsewhere;
    in a NaN-padded buffer."""
    x = torch.full((R, cols), NAN, dtype=BF16, device="cuda")
    for e, c in enumerate(counts):
        x[off[e]:off[e + 1]] = 0
        if c:
            x[off[e]:off[e] + c] = make(c)
    return poisoned(x)


def check_rows_untouched(out, counts, off, what):
    """Rows outside the segments and the guard bands keep their bits; every padding row is exact zero."""
    for e, c in enumerate(counts):
        pad = out.view[off[e] + c:off[e + 1]]
        assert not pad.numel() or bool((pad == 0).all()), f"{what}: padding rows of expert {e} are not zero"
    out.view[off[0]:off[-1]] = out.before[out.rs, out.cs][off[0]:off[-1]]
    out.check_untouched(f"{what}: rows outside the experts, or the guard band,")


# counts with every edge of the 64-row granule and the 128-row m-tile, empty experts and a few hundred rows
COUNTS = {
    "edges": [0, 1, 63, 64, 65, 127, 128, 129, 300, 0, 517],
    "e1": [200],
    "e8": [64, 0, 129, 1, 0, 383, 65, 127],
    "e256": [0] * 256,
}
for _e, _c in ((0, 3), (17, 129), (128, 1), (200, 256), (255, 77)):
    COUNTS["e256"][_e] = _c


# ---------------------------------------------------------------------------------------------------------------------
# 1. exact oracle per form
# ---------------------------------------------------------------------------------------------------------------------
def run_ragged_store(counts, N, Kd, b_mn, gen, lead=0, tail=0, sms=0):
    """out[r] = x[r] w[e]^T (b_mn=0, w [E, N, K]) or x[r] w[e] (b_mn=1, w [E, K, N])."""
    E = len(counts)
    off, R = layout(counts, lead, tail)
    x = segment_rows(counts, off, R, Kd, lambda c: exact_grid(c, Kd, gen)[0])
    wl = [exact_grid(N, Kd, gen)[0] for _ in range(E)]  # logical B_e [N, K]
    w = torch.stack([t.t() if b_mn else t for t in wl]).contiguous()
    offs = dev_offsets(off)
    assert K.supports_ragged(x, w, offs)
    out = Guarded(R, N)
    K.ragged_matmul(x, w, offs, bool(b_mn), out=out.view, sms=sms)
    what = f"ragged store b_mn={b_mn} E={E} N={N} K={Kd} lead={lead} tail={tail} sms={sms}"
    for e, c in enumerate(counts):
        if c:
            assert_gemm_exact(out.view[off[e]:off[e] + c], x[off[e]:off[e] + c], wl[e], what=f"{what} expert {e}")
    res = out.view.clone()
    check_rows_untouched(out, counts, off, what)
    return res


@pytest.mark.parametrize("case", sorted(COUNTS))
@pytest.mark.parametrize("b_mn", [0, 1])
def test_ragged_store_exact(case, b_mn):
    """NT (inference-style K-major w) and NN (dX of gate|up: MN-major w, expert offset on K) over ragged segments."""
    N, Kd = (328, 192) if b_mn == 0 else (200, 256)
    run_ragged_store(COUNTS[case], N, Kd, b_mn, _gen("ragged-store", case, b_mn), lead=64, tail=37)


def run_ragged_swiglu(counts, H, I, gen, lead=0, tail=0, sms=0, save=True):
    E = len(counts)
    off, R = layout(counts, lead, tail)
    x = segment_rows(counts, off, R, H, lambda c: exact_grid(c, H, gen, -6, 0)[0])
    w13 = torch.stack([exact_grid(2 * I, H, gen, -6, 0)[0] for _ in range(E)])
    offs = dev_offsets(off)
    act, gu = Guarded(R, I), (Guarded(R, 2 * I) if save else None)
    K.ragged_matmul(x, w13, offs, False, out=act.view, epi=K.EPI_SWIGLU, out2=gu.view if save else None, sms=sms)
    what = f"ragged swiglu E={E} H={H} I={I} sms={sms}"
    for e, c in enumerate(counts):
        if c:
            s = slice(off[e], off[e] + c)
            _check_swiglu(act.view[s], gu.view[s] if save else None, x[s], w13[e], I, True, f"{what} expert {e}")
    res = (act.view.clone(), gu.view.clone() if save else None)
    check_rows_untouched(act, counts, off, what + " act")
    if save:
        check_rows_untouched(gu, counts, off, what + " gate|up")
    return res


@pytest.mark.parametrize("case", sorted(COUNTS))
def test_ragged_swiglu_exact(case):
    """gate|up (+) SwiGLU: each expert's gate rows at e*2I + col0 and up rows at e*2I + I + col0 of w13 [E, 2I, H]."""
    run_ragged_swiglu(COUNTS[case], 192, 256, _gen("ragged-swiglu", case), lead=128, tail=5)


def run_ragged_dswiglu(counts, H, I, gen, lead=0, tail=0, sms=0):
    E = len(counts)
    off, R = layout(counts, lead, tail)
    dy = segment_rows(counts, off, R, H, lambda c: exact_grid(c, H, gen)[0])
    aux = segment_rows(counts, off, R, 2 * I, lambda c: (torch.randn(c, 2 * I, generator=gen, device="cuda") * 2).to(BF16))
    wl = [exact_grid(I, H, gen)[0] for _ in range(E)]  # logical [I, H]; stored w2 [E, H, I]
    w2 = torch.stack([t.t() for t in wl]).contiguous()
    offs = dev_offsets(off)
    dgu = Guarded(R, 2 * I)
    K.ragged_matmul(dy, w2, offs, True, out=dgu.view[:, :I], epi=K.EPI_DSWIGLU, aux=aux, out2=dgu.view, sms=sms)
    what = f"ragged dswiglu E={E} H={H} I={I} sms={sms}"
    for e, c in enumerate(counts):
        if c:
            s = slice(off[e], off[e] + c)
            _check_dswiglu(dgu.view[s], dy[s], wl[e], aux[s], I, True, f"{what} expert {e}")
    res = dgu.view.clone()
    check_rows_untouched(dgu, counts, off, what)
    return res


@pytest.mark.parametrize("case", sorted(COUNTS))
def test_ragged_dswiglu_exact(case):
    """down dX (+) dSwiGLU: w2 [E, H, I] MN-major, the expert's slab at K coordinate e*H."""
    run_ragged_dswiglu(COUNTS[case], 192, 256, _gen("ragged-dswiglu", case), lead=64, tail=64)


class GuardedStack:
    """A contiguous ``[E, M, N]`` output inside NaN guard bands before and after it."""

    def __init__(self, E, M, N, fill=None, guard=4096):
        self.buf = torch.full((E * M * N + 2 * guard, ), NAN, dtype=BF16, device="cuda")
        self.g = guard
        self.view = self.buf[guard:guard + E * M * N].view(E, M, N)
        if fill is not None:
            self.view.copy_(fill)
        self.before = self.buf.clone()

    def check_guards(self, what):
        n = self.view.numel()
        assert_bits_equal(self.buf[:self.g], self.before[:self.g], f"{what}: guard before")
        assert_bits_equal(self.buf[self.g + n:], self.before[self.g + n:], f"{what}: guard after")


def run_wgrad(counts, M, N, accumulate, gen, lead=0, tail=0, sms=0):
    """out[e] (+)= a_e^T b_e over expert e's rows only (variable K)."""
    E = len(counts)
    off, R = layout(counts, lead, tail)
    A, B, ea, eb = [], [], [], []
    for c in counts:  # logical A_e [M, c], B_e [N, c]: the rows of expert e transposed
        a_, ea_ = exact_grid(M, max(c, 1), gen)
        b_, eb_ = exact_grid(N, max(c, 1), gen)
        A.append(a_[:, :c])
        B.append(b_[:, :c])
        ea.append(ea_)
        eb.append(eb_)
    it_a, it_b = (iter([t for t, c in zip(L, counts) if c]) for L in (A, B))  # segment_rows asks for non-empty ones
    a = segment_rows(counts, off, R, M, lambda c: next(it_a).t())
    b = segment_rows(counts, off, R, N, lambda c: next(it_b).t())
    c_old = None
    if accumulate:
        c_old = torch.stack([exact_addend(ea[e], eb[e], gen) for e in range(E)])
    out = GuardedStack(E, M, N, fill=c_old)
    K.ragged_wgrad(a, b, dev_offsets(off), E, out=out.view, accumulate=accumulate, sms=sms)
    what = f"ragged wgrad acc={accumulate} E={E} M={M} N={N} sms={sms}"
    for e, c in enumerate(counts):
        if c:
            # the segment's zero padding rows add +0 products, and -0 + +0 = +0: an exact -0 comes out as +0
            ref = torch.mm(A[e].double(), B[e].double().t())
            if accumulate:
                ref = ref + c_old[e].double()
            assert_bits_equal(out.view[e] + 0.0, ref.to(BF16) + 0.0, f"{what} expert {e}")
        elif accumulate:
            assert_bits_equal(out.view[e], c_old[e], f"{what}: empty expert {e} under ACCUM")
        else:
            assert bool((out.view[e] == 0).all()), f"{what}: empty expert {e} under STORE is not zero"
    out.check_guards(what)
    return out.view.clone()


@pytest.mark.parametrize("case", sorted(COUNTS))
@pytest.mark.parametrize("accumulate", [False, True])
def test_ragged_wgrad_exact(case, accumulate):
    """Variable-K dW: each tile sums only its expert's k-blocks; empty experts store zeros or keep C; M and N tails."""
    M, N = (200, 328) if case != "e256" else (136, 264)
    run_wgrad(COUNTS[case], M, N, accumulate, _gen("ragged-wgrad", case, accumulate), lead=64, tail=21)


def test_ragged_forms_grid_independent():
    """Each tile's K loop runs in one CTA in a fixed order: every form is bit-identical over CTA counts and relaunches
    (the ring's stage and phase wrap across tiles, and across empty experts in the variable-K form)."""
    counts = COUNTS["edges"]
    for name, fn in (("store-nt", lambda g, s: run_ragged_store(counts, 328, 192, 0, g, 64, 9, s)),
                     ("store-nn", lambda g, s: run_ragged_store(counts, 200, 256, 1, g, 0, 0, s)),
                     ("swiglu", lambda g, s: run_ragged_swiglu(counts, 192, 256, g, 0, 3, s)[0]),
                     ("dswiglu", lambda g, s: run_ragged_dswiglu(counts, 192, 256, g, 64, 0, s)),
                     ("wgrad", lambda g, s: run_wgrad(counts, 200, 328, False, g, 0, 0, s)),
                     ("wgrad-acc", lambda g, s: run_wgrad(counts, 200, 328, True, g, 0, 0, s))):
        first = None
        for sms in SMS:
            for _ in range(2 if sms == 0 else 1):
                got = fn(_gen("grid", name), sms)
                if first is None:
                    first = got
                else:
                    assert_bits_equal(got, first, f"{name} sms={sms}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. refused arguments: NativeOpError, nothing written
# ---------------------------------------------------------------------------------------------------------------------
def _r(rows, cols, width=None, col0=0):
    width = width or cols
    return torch.randn(rows, width, device="cuda").to(BF16)[:, col0:col0 + cols]


def _w(E, n, k):
    return torch.randn(E, n, k, device="cuda").to(BF16)


def _refusal(case):
    """-> (call(out, out2), out spec, out2 spec | None), each spec ``(rows, cols, width, col0)``."""
    R, H, I, E = 256, 128, 128, 3
    off = dev_offsets([0, 64, 128, 256])
    x = _r(R, H)
    c, c2 = (R, H, H, 0), (R, 2 * I, 2 * I, 0)
    mm = lambda *args, **kw: (lambda o, o2: K.ragged_matmul(*args, out=o, out2=o2, **kw))
    cases = {
        "k_mod64": lambda: (mm(_r(R, 72, 72), _w(E, H, 72), off, False), c),
        "n_mod8": lambda: (mm(x, _w(E, 124, H), off, False), (R, 124, 128, 0)),
        "e257": lambda: (mm(x, _w(257, 8, H), dev_offsets([0] * 258), False), (R, 8, 8, 0)),
        "misaligned": lambda: (mm(_r(R, H, H + 8, 1), _w(E, H, H), off, False), c),
        "lda": lambda: (mm(_r(R, H, H + 4), _w(E, H, H), off, False), c),
        "ldc": lambda: (mm(x, _w(E, H, H), off, False), (R, H, H + 4, 0)),
        "accum": lambda: (mm(x, _w(E, H, H), off, False, epi=K.EPI_ACCUM), c),
        "swiglu_inter": lambda: (mm(x, _w(E, 2 * 192, H), off, False, epi=K.EPI_SWIGLU), (R, 192, 192, 0),
                                 (R, 384, 384, 0)),
        "swiglu_mn_b": lambda: (mm(x, _w(E, H, 2 * I), off, True, epi=K.EPI_SWIGLU), (R, 2 * I, 2 * I, 0), c2),
        "dswiglu_k_major_b": lambda: (mm(x, _w(E, I, H), off, False, epi=K.EPI_DSWIGLU, aux=_r(R, 2 * I)), (R, I, I, 0),
                                      c2),
        "dswiglu_no_aux": lambda: (mm(x, _w(E, H, I), off, True, epi=K.EPI_DSWIGLU), (R, I, I, 0), c2),
        "wgrad_m_mod8": lambda: ((lambda o, o2: K.ragged_wgrad(_r(R, 132, 136), x, off, E, out=o.reshape(E, 132, H))),
                                 (E * 132, H, H, 0)),
        "wgrad_n_mod8": lambda: ((lambda o, o2: K.ragged_wgrad(x, _r(R, 124, 128), off, E, out=o.reshape(E, H, 124))),
                                 (E * H, 124, 124, 0)),
        "wgrad_e257": lambda: ((lambda o, o2: K.ragged_wgrad(x, x, dev_offsets([0] * 258), 257, out=o.reshape(257, H, H))),
                               (257 * H, H, H, 0)),
        "wgrad_misaligned": lambda: ((lambda o, o2: K.ragged_wgrad(_r(R, H, H + 8, 1), x, off, E, out=o.reshape(E, H, H))),
                                     (E * H, H, H, 0)),
        "wgrad_lda": lambda: ((lambda o, o2: K.ragged_wgrad(_r(R, H, H + 4), x, off, E, out=o.reshape(E, H, H))),
                              (E * H, H, H, 0)),
    }
    return cases[case]()


_REFUSALS = ["k_mod64", "n_mod8", "e257", "misaligned", "lda", "ldc", "accum", "swiglu_inter", "swiglu_mn_b",
             "dswiglu_k_major_b", "dswiglu_no_aux", "wgrad_m_mod8", "wgrad_n_mod8", "wgrad_e257", "wgrad_misaligned",
             "wgrad_lda"]


@pytest.mark.parametrize("case", _REFUSALS)
def test_ragged_refused_arguments_raise_and_write_nothing(case):
    """Every host-side refusal of ``dsb_gemm_ragged_bf16`` / ``dsb_gemm_ragged_wgrad_bf16``.  (Malformed *device*
    offsets are refused by the kernel itself; that guard is not exercised on the GPU.)"""
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
# 3. against the capacity-padded path it replaces
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def own_backend(monkeypatch):
    """The front door on the in-tree kernel for every shape (the table could send a shape to cuBLAS)."""
    monkeypatch.setattr(gemm, "_backend", "own")
    monkeypatch.setattr(gemm, "_used", {})
    monkeypatch.setattr(gemm, "_measured", {})


def test_ragged_fn_bit_equal_to_padded_fn(own_backend):
    """The ragged node against ``_GroupedSwiGLUFn`` on the same tokens padded to ``[E, max_count, H]``: the same kernel
    body, the same k order per output, and only all-zero extra k-blocks, so y, the saved gate|up, dx, dW13 and dW2 are
    bit-equal."""
    from deepspeed_b200.ops.linear import _RaggedSwiGLUFn, grouped_swiglu_mlp
    counts = [300, 0, 17, 256, 1, 290, 64, 129]
    E, H, I = len(counts), 256, 384
    mx = max(counts)
    g = _gen("vs-padded")
    tok = [(torch.randn(c, H, generator=g, device="cuda") * 0.5).to(BF16) for c in counts]
    gy = [torch.randn(c, H, generator=g, device="cuda").to(BF16) for c in counts]
    w13 = (torch.randn(E, 2 * I, H, generator=g, device="cuda") * H**-0.5).to(BF16)
    w2 = (torch.randn(E, H, I, generator=g, device="cuda") * I**-0.5).to(BF16)

    xp = torch.zeros(E, mx, H, dtype=BF16, device="cuda")
    gp = torch.zeros(E, mx, H, dtype=BF16, device="cuda")
    for e, c in enumerate(counts):
        xp[e, :c], gp[e, :c] = tok[e], gy[e]
    xp.requires_grad_(True)
    w13p, w2p = w13.clone().requires_grad_(True), w2.clone().requires_grad_(True)
    yp = grouped_swiglu_mlp(xp, w13p, w2p)
    _, gus_p, _ = yp.grad_fn.saved
    gus_p = [t.clone() for t in gus_p]
    yp.backward(gp)

    off, R = layout(counts)
    xr = torch.zeros(R, H, dtype=BF16, device="cuda")
    gr = torch.zeros(R, H, dtype=BF16, device="cuda")
    for e, c in enumerate(counts):
        xr[off[e]:off[e] + c], gr[off[e]:off[e] + c] = tok[e], gy[e]
    xr.requires_grad_(True)
    w13r, w2r = w13.clone().requires_grad_(True), w2.clone().requires_grad_(True)
    yr = _RaggedSwiGLUFn.apply(xr, dev_offsets(off), w13r, w2r)
    gu_r = yr.grad_fn.saved_tensors[2].clone()
    yr.backward(gr)

    for e, c in enumerate(counts):
        s = slice(off[e], off[e] + c)
        assert_bits_equal(yr[s], yp[e, :c], f"y expert {e}")
        assert_bits_equal(gu_r[s], gus_p[e][:c], f"gate|up expert {e}")
        assert_bits_equal(xr.grad[s], xp.grad[e, :c], f"dx expert {e}")
    assert_bits_equal(w13r.grad, w13p.grad, "dW13")
    assert_bits_equal(w2r.grad, w2p.grad, "dW2")


# ---------------------------------------------------------------------------------------------------------------------
# 4. the dropless layer
# ---------------------------------------------------------------------------------------------------------------------
def _loop_reference(x, wg, w13, w2, ids, k, gy):
    """Float64 per-expert loop with the layer's routing decision ``ids``; returns y and the gradients of (y * gy).sum()
    with respect to x, the gate weight, w13 and w2."""
    xd, wgd, w13d, w2d = (t.detach().double().requires_grad_(True) for t in (x, wg, w13, w2))
    probs = torch.softmax(xd @ wgd.t(), dim=1)
    w = probs.gather(1, ids.long())
    w = w / w.sum(1, keepdim=True)
    y = torch.zeros_like(xd)
    I = w2.shape[2]
    for e in range(w13.shape[0]):
        tk = (ids == e).nonzero()
        if not tk.numel():
            continue
        t, j = tk[:, 0], tk[:, 1]
        gu = xd[t] @ w13d[e].t()
        o = (torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]) @ w2d[e].t()
        y = y.index_add(0, t, o * w[t, j][:, None])
    (y * gy.double()).sum().backward()
    return y, xd.grad, wgd.grad, w13d.grad, w2d.grad


def test_dropless_layer_no_sync_and_matches_float64_loop():
    """A dropless top-2 MoE layer with grouped experts (bf16, skewed routing, an empty expert) runs forward and backward
    with no host synchronisation, and its output and gradients (x, gate weight, w13, w2) match the float64 per-expert
    loop element by element."""
    from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
    from deepspeed_b200.moe.layer import MoE
    torch.manual_seed(0)
    E, H, I, T = 8, 256, 512, 384
    layer = MoE(H, GroupedSwiGLUExperts(E, H, I), num_experts=E, k=2, min_capacity=4, drop_tokens=False,
                use_rts=False).cuda().to(BF16)
    x = torch.randn(T, H, device="cuda").to(BF16)
    x[:, 0] = x[:, 0].abs() + 1
    with torch.no_grad():  # skew: expert 0 favoured, expert 7 never chosen (x[:, 0] >= 1)
        wg = layer.deepspeed_moe.gate.wg.weight
        wg.normal_(0, 0.05)
        wg[0, 0] = 1.0
        wg[7] = 0.0
        wg[7, 0] = -5.0
    x.requires_grad_(True)
    gy = torch.randn(T, H, device="cuda").to(BF16)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y, _, _ = layer(x)
        (y.float() * gy.float()).sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    gate = layer.deepspeed_moe.gate
    ids = gate(x.detach()).expert_ids
    counts = torch.bincount(ids.reshape(-1).long(), minlength=E)
    assert counts[7].item() == 0 and counts.max().item() > 2 * T * 2 / E, counts
    ex = layer.deepspeed_moe.experts
    ref = _loop_reference(x, gate.wg.weight, ex.w13, ex.w2, ids, 2, gy)
    for got, r, what in zip((y, x.grad, gate.wg.weight.grad, ex.w13.grad, ex.w2.grad), ref,
                            ("y", "dx", "d gate weight", "dW13", "dW2")):
        r = r.detach()
        bound = 2**-6 * r.abs() + 2e-2 * r.abs().max()
        assert_within(got.double(), r, bound, what)
    assert not bool(ex.w13.grad[7].any()) and not bool(ex.w2.grad[7].any())


def _first_backward_on_autograd_thread(which):
    """In a fresh process, the experts' backward is the first CUDA work of the autograd worker thread."""
    from deepspeed_b200.ops.linear import _RaggedSwiGLUFn, grouped_swiglu_mlp
    g = torch.Generator(device="cuda").manual_seed(0)
    E, H, I, C = 2, 256, 384, 256
    w13 = (torch.randn(E, 2 * I, H, generator=g, device="cuda") * H**-0.5).to(BF16).requires_grad_(True)
    w2 = (torch.randn(E, H, I, generator=g, device="cuda") * I**-0.5).to(BF16).requires_grad_(True)
    x = (torch.randn(E * C, H, generator=g, device="cuda") * 0.5).to(BF16).requires_grad_(True)
    gy = torch.randn(E * C, H, generator=g, device="cuda").to(BF16)
    torch.cuda.synchronize()
    if which == "ragged":
        y = _RaggedSwiGLUFn.apply(x, dev_offsets([0, C, 2 * C]), w13, w2)
    else:
        y = grouped_swiglu_mlp(x.view(E, C, H), w13, w2).view(E * C, H)
    y.backward(gy)
    for t in (x.grad, w13.grad, w2.grad):
        assert t is not None and bool(torch.isfinite(t).all()) and bool(t.any())


@pytest.mark.parametrize("which", ["ragged", "padded"])
def test_experts_backward_first_on_autograd_thread(which):
    """The tensor maps are encoded through the driver API, which needs a current context: the autograd worker thread has
    none before its first CUDA call, and the encode must bind one rather than fail."""
    from tests.common import run_distributed
    run_distributed(_first_backward_on_autograd_thread, 1, (which, ))


# ---------------------------------------------------------------------------------------------------------------------
# 5. engine
# ---------------------------------------------------------------------------------------------------------------------
def _mixtral_cfg():
    from deepspeed_b200.models.mixtral import mixtral_config
    return mixtral_config("tiny-moe", hidden_size=256, intermediate_size=384, num_attention_heads=4, num_key_value_heads=2,
                          vocab_size=1024, num_hidden_layers=2, num_local_experts=4, max_position_embeddings=512,
                          drop_tokens=False)


def _is_expert(n):
    return n.endswith(("experts.w13", "experts.w2"))


def _engine_dropless(stage, experts_only, read_grads, steps=5):
    """``experts_only``: every other parameter frozen, so w13 / w2 are their unit's last gradients (marking w13 ready
    reduces the unit: ZeRO-3 releases its weights, and a step fused into backward rewrites them).  ``read_grads``: a
    clip that never bites keeps the step out of backward, so the step-1 expert gradients can be read and compared with
    the same model in fp32 on the torch loop; without it the step runs inside backward."""
    import deepspeed_b200 as ds
    from deepspeed_b200.models.mixtral import MixtralForCausalLM
    from deepspeed_b200.utils import safe_get_full_grad
    cfg = _mixtral_cfg()
    torch.manual_seed(0)
    ref = MixtralForCausalLM(cfg)  # fp32 on the CPU: the torch per-expert loop
    model = MixtralForCausalLM(cfg)
    model.load_state_dict(ref.state_dict())
    model = model.cuda().to(BF16)
    if experts_only:
        for n, p in model.named_parameters():
            p.requires_grad_(_is_expert(n))
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (2, 256), generator=g)
    loss_ref = ref(ids, labels=ids)
    loss_ref.backward()
    config = {
        "train_micro_batch_size_per_gpu": 2,
        "bf16": {"enabled": True},
        "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
        "zero_optimization": {"stage": stage},
    }
    if read_grads:
        config["gradient_clipping"] = 1e6
    engine, _, _, _ = ds.initialize(model=model, config=config)
    experts = [(n, p) for n, p in model.named_parameters() if _is_expert(n)]
    assert len(experts) == 2 * cfg.num_hidden_layers
    ids_d = ids.cuda()
    losses = []
    for step in range(steps):
        loss = engine(ids_d, labels=ids_d)
        engine.backward(loss)
        if step == 0 and read_grads:
            ref_params = dict(ref.named_parameters())
            for n, p in experts:
                got = safe_get_full_grad(p)
                assert got is not None, n
                r = ref_params[n].grad.double()
                # a bf16 model against an fp32 one: activations rounded to bf16 through two layers, per-element slack.
                # A token whose top-2 is a near tie can pick another expert in bf16 than in fp32, which moves a handful
                # of elements by more: at most 1e-5 of them may leave the bound, and the whole tensor stays close
                d = got.double().cpu()
                bound = 0.1 * r.abs() + 0.1 * r.abs().max()
                outside = int(((d - r).abs() > bound).sum())
                assert outside <= 1e-5 * r.numel(), (f"ZeRO-{stage} {n}", outside)
                assert (d - r).norm() <= 0.1 * r.norm(), (f"ZeRO-{stage} {n}", float((d - r).norm() / r.norm()))
        engine.step()
        losses.append(float(loss.detach()))
    assert abs(losses[0] - float(loss_ref)) < 2e-2 * abs(float(loss_ref)), (losses[0], float(loss_ref))
    assert all(math.isfinite(v) for v in losses) and losses[-1] < losses[0], losses
    return losses


def _engine_dropless_fused_vs_two_phase(stage):
    """Experts only, the step fused into backward against the two-phase step: the same losses."""
    fused = _engine_dropless(stage, True, False)
    two_phase = _engine_dropless(stage, True, True)
    for a, b in zip(fused, two_phase):
        assert abs(a - b) <= 2e-3 * abs(b), (fused, two_phase)


@pytest.mark.parametrize("stage", [2, 3])
def test_mixtral_dropless_engine_trains(stage):
    """A small dropless Mixtral (H 256, I 384, 4 experts) in bf16 under ZeRO-2 / ZeRO-3, in a fresh process: step-1 loss
    and expert gradients against the same model and weights in fp32 on the torch loop; the loss decreases."""
    from tests.common import run_distributed
    run_distributed(_engine_dropless, 1, (stage, False, True))


@pytest.mark.parametrize("stage", [2, 3])
def test_mixtral_dropless_engine_experts_only(stage):
    """Only the experts train, so w13 / w2 are the last gradients of their unit: the expert gradients still match the
    fp32 loop (ZeRO-3 releases the unit's weights once they are reduced, after every read), and the step fused into
    backward gives the losses of the two-phase step."""
    from tests.common import run_distributed
    run_distributed(_engine_dropless_fused_vs_two_phase, 1, (stage, ), timeout=400)
