"""The optimizer step per element (``csrc/cuda/optim.cu``): fused Adam/AdamW (flat and multi-tensor), Lion, LAMB,
Adagrad and SGD against their float64 forms, the gradient norm / clip / skip kernels and the casts, and the ZeRO step
that composes them.  References and bounds are in ``tests/numerics.py``; each step is checked from the state the
kernel started from, so errors do not compound."""
import math

import pytest
import torch

from tests.numerics import (U, _rel, adagrad_reference, adam_hyper, adam_reference, assert_bits_equal, assert_within,
                            clip_coeff_reference, f32, lion_reference, round_bf16_truncate, sgd_reference, sumsq_bound,
                            ulp)

pytestmark = pytest.mark.gpu

F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
GUARD = 16  # elements of guard band on each side of every buffer (keeps 16-byte alignment for every dtype)
CAP = 132 * 8 * 256 * 8  # elements one grid-stride pass of adam_flat covers: 132 SMs x 8 blocks x 256 threads x 8


def _dev():
    return torch.device("cuda", 0)


def _flat():
    from deepspeed_b200.ops.kernels import flat_ops
    return flat_ops


class Guarded:
    """``n`` elements of ``dtype`` with ``GUARD`` sentinel elements on each side; ``off`` shifts the view by that many
    elements (a misaligned view when the element offset is not a multiple of 16 bytes)."""

    def __init__(self, values, dtype, off=0, sentinel=-12345.0):
        n = values.numel()
        self.base = torch.full((n + 2 * GUARD + 8, ), sentinel, dtype=dtype, device=_dev())
        self.lo = GUARD + off
        self.t = self.base[self.lo:self.lo + n]
        self.t.copy_(values)
        self.snap = self.base.clone()

    def check_guards(self, what):
        n = self.t.numel()
        assert_bits_equal(self.base[:self.lo], self.snap[:self.lo], f"{what}: guard before")
        assert_bits_equal(self.base[self.lo + n:], self.snap[self.lo + n:], f"{what}: guard after")


def _families(n, gdt, gen, sdt=F32):
    """``(p, g, m, v)`` in fp32 for one Adam step, cycling the data families element by element:
    randn; gradients spread over 2**-40..2**20 (over fp16's range for fp16 gradients, and up to 2**7 for fp16 states,
    whose second moment would overflow); g = m = v = 0 (only the decay moves p); v small enough that eps dominates;
    signed zeros; fp16 gradients near 65504 (fp32 states only)."""
    dev = gen.device
    rn = lambda: torch.randn(n, generator=gen, device=dev)  # noqa: E731
    p, g, m, v = rn(), rn() * 0.1, rn() * 0.01, rn().abs() * 1e-3
    fam = torch.arange(n, device=dev) % 6
    lo, hi = (-24, 7) if sdt == F16 else (-24, 15) if gdt == F16 else (-40, 20)
    spread = torch.ldexp(torch.sign(rn()), torch.randint(lo, hi + 1, (n, ), generator=gen, device=dev))
    g = torch.where(fam == 1, spread, g)
    m = torch.where(fam == 1, spread * 0.1, m)
    v = torch.where(fam == 1, spread * spread * 0.5, v)
    zero = fam == 2
    g, m, v = (torch.where(zero, 0.0, x) for x in (g, m, v))
    tiny = fam == 3
    g = torch.where(tiny, rn() * 1e-12, g)
    m = torch.where(tiny, rn() * 1e-13, m)
    v = torch.where(tiny, 1e-26, v)
    sz = fam == 4
    g = torch.where(sz, -0.0, g)
    m = torch.where(sz, -0.0, m)
    v = torch.where(sz, 0.0, v)
    if gdt == F16 and sdt != F16:
        big = fam == 5
        g = torch.where(big, torch.sign(rn()) * (65504.0 - torch.rand(n, generator=gen, device=dev) * 64), g)
    return p, g.to(gdt), m, v


def _adam_call(P, G, M, V, O, h, step, d_gscale=None, d_skip=None, grad_scale=1.0):
    _flat().adam_flat(P.t, G.t, M.t, V.t, O.t if O is not None else None, lr=h["lr"], beta1=h["b1"], beta2=h["b2"],
                      eps=h["eps"], weight_decay=h["wd"], step=step, adamw=h["adamw"], grad_scale=grad_scale,
                      d_gscale=d_gscale, d_skip=d_skip)


def _adam_run(n, pdt, gdt, sdt, odt, adamw, bc, steps, seed, off=(0, 0, 0, 0, 0)):
    """Run ``adam_flat`` for the given steps on guarded buffers and check every step per element."""
    gen = torch.Generator(device=_dev()).manual_seed(seed)
    p, g, m, v = _families(n, gdt, gen, sdt)
    P, G, M, V = (Guarded(x, dt, o) for x, dt, o in zip((p, g, m, v), (pdt, gdt, sdt, sdt), off))
    O = Guarded(torch.zeros(n), odt, off[4]) if odt is not None else None
    d_gscale = torch.tensor([0.375], device=_dev())
    for step in steps:
        h = adam_hyper(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=step, bias_correction=bc,
                       grad_scale=2.0, d_gscale=0.375, adamw=adamw)
        p0, m0, v0 = P.t.clone(), M.t.clone(), V.t.clone()
        _flat().adam_flat(P.t, G.t, M.t, V.t, O.t if O is not None else None, lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8,
                          weight_decay=0.1, step=step, adamw=adamw, bias_correction=bc, grad_scale=2.0,
                          d_gscale=d_gscale)
        rp, rm, rv, bp, bm, bv = adam_reference(p0, G.t, m0, v0, h, (pdt, sdt))
        what = f"n={n} {pdt}/{gdt}/{sdt}/{odt} adamw={adamw} bc={bc} step={step}"
        assert_within(P.t, rp, bp, f"p {what}")
        assert_within(M.t, rm, bm, f"m {what}")
        assert_within(V.t, rv, bv, f"v {what}")
        if O is not None:
            if pdt == F32 or pdt == odt:  # the copy is RNE of the kernel's own fp32 master
                assert_bits_equal(O.t, P.t.to(odt), f"out {what}")
            else:
                assert_within(O.t, rp, ulp(rp.abs() + bp, odt) + bp, f"out {what}")
        for X, name in ((P, "p"), (G, "g"), (M, "m"), (V, "v")) + (((O, "out"), ) if O is not None else ()):
            X.check_guards(f"{name} {what}")


ADAM_SIZES = [1, 7, 8, 9, 4095, 65535, 65537, CAP - 8, CAP - 1, CAP, CAP + 1, CAP + 8, 3_000_001]
# (master, gradient, state, out, adamw, bias correction)
ADAM_CONFIGS = [
    (F32, F32, F32, BF16, True, True),
    (F32, BF16, F32, BF16, False, True),
    (F32, F16, F32, F16, True, False),
    (F32, F32, F32, None, False, False),
    (BF16, BF16, BF16, None, True, True),
    (BF16, F32, F32, F16, False, True),
    (F16, F16, F32, BF16, True, True),
    (F16, F16, F16, F16, False, True),
]


def _cfg_id(c):
    name = lambda d: "none" if d is None else str(d).replace("torch.", "")  # noqa: E731
    return "-".join(name(d) for d in c[:4]) + f"-adamw{int(c[4])}-bc{int(c[5])}"


@pytest.mark.parametrize("cfg", ADAM_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("n", ADAM_SIZES)
def test_adam_flat_per_element(n, cfg):
    _adam_run(n, *cfg, steps=(1, 2, 10, 1000), seed=n)


@pytest.mark.parametrize("off", [1, 2, 3, 4, 5, 6, 7])
@pytest.mark.parametrize("which", ["all", "p", "g", "m", "v", "out"])
def test_adam_flat_misaligned(off, which):
    """Views that are not 16-byte aligned take the scalar path (one pointer or all of them)."""
    names = ["p", "g", "m", "v", "out"]
    offs = tuple(off if which in ("all", nm) else 0 for nm in names)
    _adam_run(65537 + off, F32, BF16, F32, BF16, True, True, steps=(1, 2), seed=off, off=offs)
    _adam_run(4099, BF16, BF16, BF16, F16, False, True, steps=(3, ), seed=off, off=offs)


@pytest.mark.parametrize("n", [9, 65537])
def test_adam_flat_skip_leaves_everything(n):
    gen = torch.Generator(device=_dev()).manual_seed(1)
    p, g, m, v = _families(n, BF16, gen)
    P, G, M, V = Guarded(p, F32), Guarded(g, BF16), Guarded(m, F32), Guarded(v, F32)
    O = Guarded(torch.zeros(n), BF16, sentinel=777.0)
    O.t.fill_(777.0)
    O.snap = O.base.clone()
    skip = torch.ones(1, dtype=torch.int32, device=_dev())
    h = adam_hyper(1e-2, 0.9, 0.95, 1e-8, 0.1, 1)
    _adam_call(P, G, M, V, O, h, 1, d_gscale=torch.tensor([0.5], device=_dev()), d_skip=skip)
    for X in (P, G, M, V, O):
        assert_bits_equal(X.base, X.snap, "d_skip = 1")
    skip.zero_()  # and 0 means step
    _adam_call(P, G, M, V, O, h, 1, d_skip=skip)
    assert not torch.equal(P.t, P.snap[GUARD:GUARD + n])


MUTATIONS = ["bias_correction_t-1", "eps_inside_sqrt", "adamw_as_l2", "lr_wd_dropped", "gscale_ignored",
             "tail_not_updated", "truncating_bf16_cast"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_adam_bound_rejects_mutations(mutation):
    """The bound has teeth: for each plausible kernel bug, the real kernel's output falls outside the bound of a
    reference that carries that bug."""
    n, step = 4099, 3
    gen = torch.Generator(device=_dev()).manual_seed(5)
    p = torch.randn(n, generator=gen, device=_dev())
    g = (torch.randn(n, generator=gen, device=_dev()) * 1e-4).bfloat16()  # v ~ eps**2: eps and sqrt interact
    m = torch.randn(n, generator=gen, device=_dev()) * 1e-5
    v = torch.rand(n, generator=gen, device=_dev()) * 1e-9
    out = torch.empty(n, dtype=BF16, device=_dev())
    p0, m0, v0 = p.clone(), m.clone(), v.clone()
    d_gscale = torch.tensor([0.5], device=_dev())
    kw = dict(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1)
    _flat().adam_flat(p, g, m, v, out, step=step, d_gscale=d_gscale, **kw)
    h = adam_hyper(step=step, d_gscale=0.5, **kw)
    rp, _, _, bp, _, _ = adam_reference(p0, g, m0, v0, h)
    assert_within(p, rp, bp, "unmutated")
    assert_bits_equal(out, p.bfloat16(), "unmutated out")
    if mutation == "truncating_bf16_cast":
        assert not torch.equal(out, round_bf16_truncate(p)), "a truncating cast would pass"
        return
    if mutation == "bias_correction_t-1":
        h = adam_hyper(step=step - 1, d_gscale=0.5, **kw)
    elif mutation == "adamw_as_l2":
        h = adam_hyper(step=step, d_gscale=0.5, adamw=False, **kw)
    elif mutation == "lr_wd_dropped":
        h = adam_hyper(step=step, d_gscale=0.5, **dict(kw, weight_decay=0.0))
    elif mutation == "gscale_ignored":
        h = adam_hyper(step=step, **kw)
    mp, _, _, mb, _, _ = adam_reference(p0, g, m0, v0, h)
    if mutation == "eps_inside_sqrt":  # u = mh / sqrt(vh + eps)
        m1 = h["b1"] * m0.double() + h["b1m"] * g.double() * h["gs"]
        v1 = h["b2"] * v0.double() + h["b2m"] * (g.double() * h["gs"])**2
        u = (m1 / h["bc1"]) / (v1 / h["bc2"] + h["eps"]).sqrt() + h["wd"] * p0.double()
        mp = p0.double() - h["lr"] * u
    elif mutation == "tail_not_updated":
        mp = mp.clone()
        mp[-1] = p0[-1]
    with pytest.raises(AssertionError):
        assert_within(p, mp, mb, f"mutation {mutation}")


# ---------------------------------------------------------------------------------------------------------------------
# multi-tensor Adam
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pdt,gdt,sdt,odt", [(F32, BF16, F32, BF16), (BF16, BF16, BF16, None), (F32, F32, F32, F16)],
                         ids=["f32-bf16-out_bf16", "bf16", "f32-out_f16"])
@pytest.mark.parametrize("misalign", [False, True])
def test_adam_multi_per_tensor(pdt, gdt, sdt, odt, misalign):
    """``dsb_adam_multi`` over tensors that straddle the 65 536-element chunk, as views into one buffer with guard bands
    between them; misaligned views take the scalar path."""
    from deepspeed_b200.ops.adam.fused_adam import _launch
    sizes = [65536 + 3, 1, 131072 - 1, 63, 65536, 200_001]
    gen = torch.Generator(device=_dev()).manual_seed(9)
    bufs, views = {}, {k: [] for k in "pgmvo"}
    total = sum(s + 2 * GUARD for s in sizes) + 8
    dts = dict(p=pdt, g=gdt, m=sdt, v=sdt, o=odt)
    for k, dt in dts.items():
        if dt is not None:
            bufs[k] = torch.full((total, ), -999.0, dtype=dt, device=_dev())
    pos = GUARD
    for i, s in enumerate(sizes):
        o = pos + ((i % 7) + 1 if misalign else 0)
        p, g, m, v = _families(s, gdt, gen, sdt)
        for k, x in zip("pgmv", (p, g, m, v)):
            views[k].append(bufs[k][o:o + s])
            views[k][-1].copy_(x)
        if odt is not None:
            views["o"].append(bufs["o"][o:o + s])
        pos += s + 2 * GUARD
    snaps = {k: b.clone() for k, b in bufs.items()}
    p0 = [x.clone() for x in views["p"]]
    m0 = [x.clone() for x in views["m"]]
    v0 = [x.clone() for x in views["v"]]
    _launch(views["p"], views["g"], views["m"], views["v"], views["o"] if odt is not None else None, 1e-3, 0.9, 0.999,
            1e-8, 4, 1, 1, 0.01, grad_scale=0.5, d_gscale=torch.tensor([2.0], device=_dev()))
    h = adam_hyper(1e-3, 0.9, 0.999, 1e-8, 0.01, 4, grad_scale=0.5, d_gscale=2.0)
    inside = torch.zeros(total, dtype=torch.bool, device=_dev())
    for i, s in enumerate(sizes):
        rp, rm, rv, bp, bm, bv = adam_reference(p0[i], views["g"][i], m0[i], v0[i], h, (pdt, sdt))
        assert_within(views["p"][i], rp, bp, f"tensor {i} p")
        assert_within(views["m"][i], rm, bm, f"tensor {i} m")
        assert_within(views["v"][i], rv, bv, f"tensor {i} v")
        if odt is not None:
            assert_bits_equal(views["o"][i], views["p"][i].to(odt), f"tensor {i} out")
        o = views["p"][i].data_ptr() // views["p"][i].element_size() - bufs["p"].data_ptr() // bufs["p"].element_size()
        inside[o:o + s] = True
    for k, b in bufs.items():
        if k != "g":
            assert_bits_equal(b[~inside], snaps[k][~inside], f"{k}: guard bands between tensors")
        else:
            assert_bits_equal(b, snaps[k], "gradients are read only")


# ---------------------------------------------------------------------------------------------------------------------
# Lion, LAMB, Adagrad, SGD
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pdt,gdt,sdt", [(F32, F32, F32), (F32, BF16, F32), (BF16, BF16, BF16), (F16, F16, F32)], ids=str)
@pytest.mark.parametrize("n", [1, 4097, 2_000_003])
@pytest.mark.parametrize("wd", [0.0, 0.1])
def test_lion_per_element(pdt, gdt, sdt, n, wd):
    gen = torch.Generator(device=_dev()).manual_seed(n)
    p, g, m, _ = _families(n, gdt, gen)
    # exact ties c = b1 m + (1 - b1) g = 0: m = 0.5, g = -0.5 with b1 = 0.5 in the first elements
    k = min(n, 5)
    m[:k], g[:k] = 0.5, -0.5
    P, G, M = Guarded(p, pdt), Guarded(g.to(gdt), gdt), Guarded(m, sdt)
    O = Guarded(torch.zeros(n), BF16)
    p0, m0 = P.t.clone(), M.t.clone()
    _flat().lion_flat(P.t, G.t, M.t, O.t, lr=1e-2, beta1=0.5, beta2=0.99, weight_decay=wd, grad_scale=2.0,
                      d_gscale=torch.tensor([0.5], device=_dev()))
    gs = f32(2.0 * 0.5)
    rp, rm, sign, bp, bm = lion_reference(p0, G.t, m0, 1e-2, 0.5, 0.99, wd, gs, (pdt, sdt))
    assert bool((sign[:k] == 0).all())
    if wd == 0.0 and pdt == F32:  # p' = fp32(p - lr sign): one rounding of an exact difference, so bit-exact
        want = (p0.double() - f32(1e-2) * sign).float()
        assert_bits_equal(P.t, want, "lion p (sign exact)")
    else:
        assert_within(P.t, rp, bp, "lion p")
    assert_within(M.t, rm, bm, "lion m")
    if pdt in (F32, BF16):
        assert_bits_equal(O.t, P.t.to(BF16), "lion out")
    for X in (P, G, M, O):
        X.check_guards("lion")


def test_lion_skip_and_gscale():
    n = 1000
    gen = torch.Generator(device=_dev()).manual_seed(3)
    p, g, m, _ = _families(n, F32, gen)
    q, mq = p.clone(), m.clone()
    skip = torch.ones(1, dtype=torch.int32, device=_dev())
    _flat().lion_flat(q, g, mq, None, lr=1e-2, beta1=0.9, beta2=0.99, weight_decay=0.1, d_skip=skip)
    assert_bits_equal(q, p, "lion d_skip p")
    assert_bits_equal(mq, m, "lion d_skip m")
    _flat().lion_flat(q, g, mq, None, lr=1e-2, beta1=0.9, beta2=0.99, weight_decay=0.0,
                      d_gscale=torch.tensor([-1.0], device=_dev()))  # a negative scale flips every sign
    rp, rm, _, bp, bm = lion_reference(p, g, m, 1e-2, 0.9, 0.99, 0.0, -1.0)
    assert_within(q, rp, bp, "lion gscale p")
    assert_within(mq, rm, bm, "lion gscale m")


def _lamb_check(p, g, m, v, coeff, p1, m1, v1, kw, step, min_c, max_c):
    """Per-element LAMB check: the trust ratio from float64 norms, then p against the Adam-style reference at
    ``lr * coeff`` with the kernel's coeff."""
    n = p.numel()
    h = adam_hyper(kw["lr"], kw["beta1"], kw["beta2"], kw["eps"], kw["weight_decay"], step)
    rp, rm, rv, bp, bm, bv, u, eu = adam_reference(p, g, m, v, h, update=True)
    assert_within(m1, rm, bm, "lamb m")
    assert_within(v1, rv, bv, "lamb v")
    pn, un = p.double().norm(), u.norm()
    c = float(coeff)
    if pn == 0 or un == 0:
        assert c == 1.0
    else:
        ratio = float(pn / un)
        grid = min(-(-n // 256), 132 * 4)
        depth = -(-n // (grid * 256)) + 10 + -(-grid // 256) + 10
        rel_u = float((2 * u.abs() * eu + eu * eu).sum() / (un * un))
        rel = (_rel(depth) + rel_u) / 2 + _rel(depth) / 2 + 3 * U
        want = min(max(ratio, min_c), max_c)
        if f32(min_c) < ratio * (1 - rel) and ratio * (1 + rel) < f32(max_c):
            assert abs(c - ratio) <= rel * ratio + 1e-30, (c, ratio, rel)
        elif ratio < min_c:
            assert c == f32(min_c), (c, min_c)
        elif ratio > max_c:
            assert c == f32(max_c), (c, max_c)
        else:
            assert abs(c - want) <= rel * ratio
    hs = adam_hyper(f32(kw["lr"]) * c, kw["beta1"], kw["beta2"], kw["eps"], kw["weight_decay"], step)
    rp, _, _, bp, _, _ = adam_reference(p, g, m, v, hs, (p1.dtype, F32))
    assert_within(p1, rp, bp, "lamb p")
    return c


@pytest.mark.parametrize("n", [1000, 300_001, 3_000_001])
@pytest.mark.parametrize("clamp", ["none", "min", "max"])
def test_lamb_per_element_and_trust_ratio(n, clamp):
    """Sizes span one to the full 528 blocks of the partials reduction; the clamps are exact fp32 values."""
    gen = torch.Generator(device=_dev()).manual_seed(n)
    p, g, m, v = _families(n, F32, gen)
    kw = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.01)
    min_c, max_c = {"none": (1e-6, 1e6), "min": (1e4, 1e6), "max": (1e-6, 1e-3)}[clamp]
    q, mq, vq = p.clone(), m.clone(), v.clone()
    out = torch.empty(n, dtype=BF16, device=_dev())
    coeff = _flat().lamb_flat(q, g, mq, vq, out, step=3, max_coeff=max_c, min_coeff=min_c, **kw)
    _lamb_check(p, g, m, v, coeff, q, mq, vq, kw, 3, min_c, max_c)
    assert_bits_equal(out, q.bfloat16(), "lamb out")


def test_lamb_zero_norms_give_coefficient_one():
    n = 70_001
    kw = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.01)
    z = torch.zeros(n, device=_dev())
    g = torch.randn(n, device=_dev())
    # |p| = 0
    c = _flat().lamb_flat(z.clone(), g, z.clone(), z.clone(), None, step=1, **kw)
    assert float(c) == 1.0
    # |u| = 0: no gradient, no moments, no decay
    p = torch.randn(n, device=_dev())
    q = p.clone()
    c = _flat().lamb_flat(q, z, z.clone(), z.clone(), None, step=1, **dict(kw, weight_decay=0.0))
    assert float(c) == 1.0
    assert_bits_equal(q, p, "lamb with u = 0")


@pytest.mark.parametrize("pdt,gdt", [(F32, F32), (F32, BF16), (BF16, F16)], ids=str)
@pytest.mark.parametrize("n", [1, 4097, 1_000_003])
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_adagrad_per_element(pdt, gdt, n, wd):
    gen = torch.Generator(device=_dev()).manual_seed(n)
    p, g, _, v = _families(n, gdt, gen)
    P, G, Hs = Guarded(p, pdt), Guarded(g, gdt), Guarded(v, F32)
    O = Guarded(torch.zeros(n), F16)
    p0, h0 = P.t.clone(), Hs.t.clone()
    for step in range(2):
        _flat().adagrad_flat(P.t, G.t, Hs.t, O.t, lr=1e-2, eps=1e-10, weight_decay=wd, grad_scale=0.5)
        rp, rh, bp, bh = adagrad_reference(p0, G.t, h0, 1e-2, 1e-10, wd, 0.5, pdt)
        assert_within(P.t, rp, bp, f"adagrad p step {step}")
        assert_within(Hs.t, rh, bh, f"adagrad h step {step}")
        if pdt == F32:
            assert_bits_equal(O.t, P.t.half(), "adagrad out")
        p0, h0 = P.t.clone(), Hs.t.clone()
    for X in (P, G, Hs, O):
        X.check_guards("adagrad")


@pytest.mark.parametrize("momentum,dampening,nesterov,wd", [(0.0, 0.0, False, 0.0), (0.9, 0.0, False, 0.01),
                                                            (0.9, 0.1, False, 0.0), (0.9, 0.0, True, 0.01)])
@pytest.mark.parametrize("n", [1, 4097, 1_000_003])
def test_sgd_per_element(momentum, dampening, nesterov, wd, n):
    gen = torch.Generator(device=_dev()).manual_seed(n)
    p, g, m, _ = _families(n, BF16, gen)
    P, G, B = Guarded(p, F32), Guarded(g, BF16), Guarded(m, F32)
    O = Guarded(torch.zeros(n), BF16)
    for first in (True, False, False):
        p0, b0 = P.t.clone(), B.t.clone()
        _flat().sgd_flat(P.t, G.t, B.t, O.t, lr=1e-2, momentum=momentum, dampening=dampening, weight_decay=wd,
                         nesterov=nesterov, first=first, grad_scale=0.5)
        rp, rb, bp, bb = sgd_reference(p0, G.t, b0, 1e-2, momentum, dampening, wd, nesterov, first, 0.5)
        assert_within(P.t, rp, bp, f"sgd p first={first}")
        assert_within(B.t, rb, bb, f"sgd buf first={first}")
        assert_bits_equal(O.t, P.t.bfloat16(), "sgd out")
    for X in (P, G, B, O):
        X.check_guards("sgd")


# ---------------------------------------------------------------------------------------------------------------------
# gradient norm, overflow flag, clip coefficient
# ---------------------------------------------------------------------------------------------------------------------
SUMSQ_N = 1_000_003


def _spike_positions(n, dtype):
    per = 4 if dtype == F32 else 8
    nv = n // per
    return {"first": 0, "last_vector": nv * per - 1, "tail": n - 1, "block_end": 512 * per - 1,
            "block_start": 512 * per}


@pytest.mark.parametrize("dtype", [F32, BF16, F16], ids=str)
@pytest.mark.parametrize("off", [0, 1, 3])
@pytest.mark.parametrize("where", ["first", "last_vector", "tail", "block_end", "block_start"])
def test_sumsq_spike_exact(dtype, off, where):
    """Ones and one spike of 64: every partial sum is an integer below 2**24, so the fp32 sum is exact in any order and a
    dropped or doubled element (1 or 4096) shows."""
    from deepspeed_b200.ops.kernels.flat_ops import GradStats
    n = SUMSQ_N
    X = Guarded(torch.ones(n), dtype, off, sentinel=1000.0)
    i = _spike_positions(n, dtype)[where]
    X.t[i] = 64.0
    st = GradStats(_dev())
    st.accumulate(X.t)
    assert float(st.sumsq) == n - 1 + 4096.0 and int(st.found_inf) == 0
    st.accumulate(X.t[:1001])  # accumulate across calls
    assert float(st.sumsq) == n - 1 + 4096.0 + 1001 + (4095.0 if i < 1001 else 0.0)
    for bad in (math.inf, -math.inf, math.nan):
        st.reset()
        assert float(st.sumsq) == 0.0 and int(st.found_inf) == 0
        X.t[i] = bad
        st.accumulate(X.t)
        assert int(st.found_inf) == 1, (where, bad)
        X.t[i] = 64.0


@pytest.mark.parametrize("dtype", [F32, BF16, F16], ids=str)
@pytest.mark.parametrize("n", [1, 9, 65537, 4_000_037])
@pytest.mark.parametrize("off", [0, 5])
def test_sumsq_randn_within_bound(dtype, n, off):
    from deepspeed_b200.ops.kernels.flat_ops import GradStats
    gen = torch.Generator(device=_dev()).manual_seed(n + off)
    X = Guarded(torch.randn(n, generator=gen, device=_dev()) * 3, dtype, off)
    st = GradStats(_dev())
    st.accumulate(X.t)
    ref = float((X.t.double()**2).sum())
    assert abs(float(st.sumsq) - ref) <= sumsq_bound(ref, n, dtype), (float(st.sumsq), ref)
    assert int(st.found_inf) == 0


def test_sumsq_fp16_max_is_finite_and_n_zero():
    from deepspeed_b200.ops import native as N
    from deepspeed_b200.ops.kernels.flat_ops import GradStats
    x = torch.full((4099, ), 65504.0, dtype=F16, device=_dev())
    st = GradStats(_dev())
    st.accumulate(x)
    assert int(st.found_inf) == 0
    ref = 4099 * 65504.0**2
    assert abs(float(st.sumsq) - ref) <= sumsq_bound(ref, 4099, F16)
    st.accumulate(x[:0])  # n = 0 adds nothing
    assert abs(float(st.sumsq) - ref) <= sumsq_bound(ref, 4099, F16)
    out = torch.full((1, ), 5.0, device=_dev())
    N.check(N.cuda().dsb_sumsq(N.ptr(x), N.c_i64(0), N.dt(x), N.ptr(st.partials(1)), N.ptr(out), N.ptr(st.found_inf),
                               0, N.stream()), "sumsq")
    assert float(out) == 0.0  # n = 0 without accumulate writes 0


@pytest.mark.parametrize("dtype", [BF16, F32], ids=str)
def test_sumsq_large_arena_past_int32(dtype):
    """``GradStats.accumulate`` over a whole ZeRO gradient arena: more than 2**31 elements, a spike and then a NaN past
    2**31.  The reference comes from the fill value and the spike."""
    from deepspeed_b200.ops.kernels.flat_ops import GradStats
    n = 2**31 + 9
    need = n * torch.tensor([], dtype=dtype).element_size()
    free, _ = torch.cuda.mem_get_info()
    if free < need + 2 * 2**30:
        pytest.skip(f"needs {(need + 2**31) / 2**30:.1f} GiB free on the device, {free / 2**30:.1f} GiB are")
    fill, spike, at = 2.0**-6, 2.0**10, 2**31 + 3
    x = torch.full((n, ), fill, dtype=dtype, device=_dev())
    x[at] = spike
    st = GradStats(_dev())
    st.accumulate(x)
    ref = (n - 1) * fill**2 + spike**2
    bound = sumsq_bound(ref, n, dtype)
    assert bound < 0.01 * spike**2
    assert abs(float(st.sumsq) - ref) <= bound, (float(st.sumsq), ref, bound)
    assert int(st.found_inf) == 0
    x[2**31 + 7] = math.nan
    st.reset()
    st.accumulate(x)
    assert int(st.found_inf) == 1
    del x
    torch.cuda.empty_cache()


@pytest.mark.parametrize("case", ["no_clip", "below", "above", "zero", "clip_big", "loss_scale"])
def test_clip_coeff(case):
    from deepspeed_b200.ops.kernels.flat_ops import GradStats
    st = GradStats(_dev())
    inv, mx, ss = 1.0, 1.0, 0.25
    if case == "no_clip":
        mx = 0.0
    elif case == "below":  # norm just under max_norm - 1e-6: no clipping
        ss = f32((1.0 - 3e-6)**2)
    elif case == "above":
        ss = f32((1.0 + 3e-6)**2)
    elif case == "zero":
        ss = 0.0
    elif case == "clip_big":
        ss = 1.5e6
    elif case == "loss_scale":
        inv, ss = 2.0**-12, 1e9
    st.sumsq.fill_(ss)
    st.finalize(inv_loss_scale=inv, max_norm=mx)
    c, norm, rel_c, rel_n = clip_coeff_reference(f32(ss), inv, mx)
    assert abs(float(st.norm) - norm) <= rel_n * norm, (float(st.norm), norm)
    assert abs(float(st.gscale) - c) <= rel_c * c + 2 * U * c, (float(st.gscale), c)
    assert int(st.skip) == 0
    if case in ("no_clip", "zero", "below"):
        assert float(st.gscale) == f32(inv)


def test_clip_coeff_overflowing_sum_skips():
    """Finite gradients whose squares overflow fp32: found_inf stays 0, the sum is inf, and the step is skipped."""
    from deepspeed_b200.ops.kernels.flat_ops import GradStats
    st = GradStats(_dev())
    st.accumulate(torch.full((1000, ), 1e20, device=_dev()))
    assert int(st.found_inf) == 0 and float(st.sumsq) == math.inf
    st.finalize(inv_loss_scale=1.0, max_norm=1.0)
    assert int(st.skip) == 1 and float(st.gscale) == 0.0 and float(st.norm) == math.inf
    st.reset()
    st.found_inf.fill_(1)
    st.finalize(inv_loss_scale=1.0, max_norm=0.0)
    assert int(st.skip) == 1 and float(st.gscale) == 0.0 and float(st.norm) == math.inf


# ---------------------------------------------------------------------------------------------------------------------
# scale_cast
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tin", [F32, BF16, F16], ids=str)
@pytest.mark.parametrize("tout", [F32, BF16, F16], ids=str)
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("d_scale", [None, 0.75])
@pytest.mark.parametrize("off", [0, 3])
def test_scale_cast(tin, tout, accumulate, d_scale, off):
    n = 70_001
    gen = torch.Generator(device=_dev()).manual_seed(n + off)
    X = Guarded(torch.randn(n, generator=gen, device=_dev()) * 8, tin, off)
    Y = Guarded(torch.randn(n, generator=gen, device=_dev()), tout, 0 if off == 0 else 1)
    y0 = Y.t.clone()
    a = 0.3
    _flat().scale_cast(X.t, Y.t, scale=a, accumulate=accumulate,
                       d_scale=torch.tensor([d_scale], device=_dev()) if d_scale is not None else None)
    s = f32(a) if d_scale is None else f32(f32(a) * f32(d_scale))
    st = torch.tensor(s, dtype=F32, device=_dev())
    if not accumulate:
        assert_bits_equal(Y.t, (X.t.float() * st).to(tout), "scale_cast")
    else:
        prod = X.t.double() * s
        ref = prod + y0.double()
        err = U * prod.abs() + U * (ref.abs() + U * prod.abs())  # product and sum round (or one fma)
        if tout == F32:
            err = U * prod.abs()
        assert_within(Y.t, ref, ulp(ref.abs() + err, tout) + err, "scale_cast accumulate")
    X.check_guards("scale_cast x")
    Y.check_guards("scale_cast y")


@pytest.mark.parametrize("dtype", [F32, BF16, F16], ids=str)
def test_scale_cast_in_place(dtype):
    n = 65_541
    x = torch.randn(n, device=_dev()).to(dtype)
    x[::97] = math.nan
    x0 = x.clone()
    _flat().scale_cast(x, x, scale=0.5, d_scale=torch.tensor([2.0], device=_dev()))  # s == 1: a bit-identical no-op
    assert_bits_equal(x, x0, "in place, s == 1")
    _flat().scale_cast(x, x, scale=0.25)
    nan = x0.isnan()
    assert bool(x[nan].isnan().all())  # (NaN payloads of the two casts differ)
    assert_bits_equal(x[~nan], (x0[~nan].float() * 0.25).to(dtype), "in place, s = 0.25")


# ---------------------------------------------------------------------------------------------------------------------
# the ZeRO step
# ---------------------------------------------------------------------------------------------------------------------
def _zero_engine(stage, clip):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=1024, num_hidden_layers=2)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(BF16)
    decay = [p for p in model.parameters() if p.ndim >= 2]
    norms = [p for p in model.parameters() if p.ndim < 2]
    groups = [{"params": decay, "lr": 2e-3, "weight_decay": 0.1}, {"params": norms, "lr": 5e-4, "weight_decay": 0.0}]
    eng, *_ = ds.initialize(model=model, model_parameters=groups, config={
        "train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True}, "gradient_clipping": clip,
        "optimizer": {"type": "AdamW", "params": {"lr": 1e-3, "betas": [0.9, 0.95], "eps": 1e-8}},
        "zero_optimization": {"stage": stage}})
    return eng, model, cfg


def _lp_and_master(zo):
    return [(zo._piece_lp(rt, s, e).clone(), zo._piece_master(rt, s, e).clone()) for rt, gi, s, e in zo.pieces
            if gi >= 0]


@pytest.mark.parametrize("stage", [1, 2, 3])
@pytest.mark.parametrize("clip", [0.0, 0.05])
def test_zero_step_per_segment(stage, clip, monkeypatch):
    """Every ``FlatAdam.step_segment`` of a ZeRO step on the tiny Llama, with two parameter groups, checked per element
    against the float64 step of its own group and step count; the low-precision weights against their masters."""
    from deepspeed_b200.runtime.zero.flat_optimizers import FlatAdam
    calls = []
    orig = FlatAdam.step_segment

    def record(self, s, e, p, g, out, group, step, grad_scale=1.0, d_gscale=None, d_skip=None):
        m, v = self.state["exp_avg"][s:e], self.state["exp_avg_sq"][s:e]
        rec = dict(s=s, e=e, p0=p.clone(), g=g.clone(), m0=m.clone(), v0=v.clone(), lr=group["lr"],
                   wd=group.get("weight_decay", 0.0), betas=tuple(group.get("betas", self.defaults["betas"])),
                   eps=group.get("eps", self.defaults["eps"]), step=step, grad_scale=grad_scale, adamw=self.adamw,
                   d_gscale=d_gscale.clone() if d_gscale is not None else None,
                   d_skip=d_skip.clone() if d_skip is not None else None,
                   ptrs=[t.data_ptr() for t in (p, g, m, v) + ((out, ) if out is not None else ())])
        orig(self, s, e, p, g, out, group, step, grad_scale=grad_scale, d_gscale=d_gscale, d_skip=d_skip)
        rec.update(p1=p.clone(), m1=m.clone(), v1=v.clone(), out=out.clone() if out is not None else None)
        calls.append(rec)

    monkeypatch.setattr(FlatAdam, "step_segment", record)
    eng, model, cfg = _zero_engine(stage, clip)
    zo = eng.optimizer
    assert isinstance(zo.flat_opt, FlatAdam)
    assert zo.fused_in_backward == (clip == 0.0)
    ids = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    pieces = sorted((s, e) for _, gi, s, e in zo.pieces if gi >= 0)
    group_of = {(s, e): gi for _, gi, s, e in zo.pieces if gi >= 0}
    ntrain = sum(p.numel() for p in model.parameters() if p.requires_grad)
    for it in range(3):
        calls.clear()
        steps_before = list(zo.group_steps)
        loss = eng(ids, labels=ids)
        eng.backward(loss)
        garena = zo.grad_arena.clone() if zo.grad_arena is not None else None
        eng.step()
        torch.cuda.synchronize()
        assert list(zo.group_steps) == [s + 1 for s in steps_before]
        # the segments cover every trainable element once
        ranges = sorted((c["s"], c["e"]) for c in calls)
        assert ranges == pieces, (ranges[:4], pieces[:4])
        assert sum(e - s for s, e in ranges) >= ntrain
        if clip > 0:
            norm = float(garena.double().norm())
            want = min(1.0, f32(clip) / (norm + 1e-6))
            rel = _rel(sumsq_depth_arena(garena)) + 8 * U
        for c in calls:
            gi = group_of[(c["s"], c["e"])]
            assert c["lr"] == zo.param_groups[gi]["lr"] and c["step"] == steps_before[gi] + 1
            assert all(ptr % 16 == 0 for ptr in c["ptrs"]), "arena segments must be 16-byte aligned"
            gs = c["grad_scale"]
            dg = None
            if c["d_gscale"] is not None:
                dg = float(c["d_gscale"])
                assert int(c["d_skip"]) == 0
                if clip > 0:
                    assert abs(dg - want) <= rel * want + 1e-12, (dg, want)
            h = adam_hyper(c["lr"], c["betas"][0], c["betas"][1], c["eps"], c["wd"], c["step"], grad_scale=gs,
                           d_gscale=dg, adamw=c["adamw"])
            rp, rm, rv, bp, bm, bv = adam_reference(c["p0"], c["g"], c["m0"], c["v0"], h)
            what = f"stage {stage} clip {clip} step {it + 1} segment [{c['s']}, {c['e']})"
            assert_within(c["p1"], rp, bp, f"p {what}")
            assert_within(c["m1"], rm, bm, f"m {what}")
            assert_within(c["v1"], rv, bv, f"v {what}")
            if c["out"] is not None:
                assert_bits_equal(c["out"], c["p1"].to(c["out"].dtype), f"out {what}")
        for lp, master in _lp_and_master(zo):
            assert_bits_equal(lp, master.to(lp.dtype), "bf16 weight = RNE(master) after engine.step()")


def sumsq_depth_arena(garena):
    from tests.numerics import sumsq_depth
    return sumsq_depth(garena.numel(), garena.dtype) + 2


@pytest.mark.parametrize("stage", [1, 2, 3])
def test_zero_bf16_clip_skips_nonfinite_step_on_device(stage):
    """bf16 with clipping: an inf gradient at step 3 leaves every master, moment and bf16 weight bit-identical; the step
    is skipped on the device without a host synchronisation, so, as DESIGN.md documents, the step counters still
    advance, ``overflow`` stays False, ``skipped_steps`` does not count it, and ``get_global_grad_norm()`` is inf."""
    eng, model, cfg = _zero_engine(stage, 0.05)
    zo = eng.optimizer
    assert not zo.fused_in_backward
    ids = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    inject = {"on": False}

    def hook(grad):
        if inject["on"]:
            grad = grad.clone()
            grad.view(-1)[0] = math.inf
        return grad

    layer0 = model.model.layers[0]
    handle = layer0.register_forward_hook(lambda mod, inp, out: (out[0].register_hook(hook), out)[1])
    for it in range(4):
        inject["on"] = it == 2
        loss = eng(ids, labels=ids)
        eng.backward(loss)
        if it == 2:
            torch.cuda.synchronize()
            before = _lp_and_master(zo)
            st = zo.flat_opt.state
            m0, v0 = st["exp_avg"].clone(), st["exp_avg_sq"].clone()
            steps0, skipped0 = list(zo.group_steps), zo.skipped_steps
        eng.step()
        if it == 2:
            torch.cuda.synchronize()
            for (lp0, ma0), (lp1, ma1) in zip(before, _lp_and_master(zo)):
                assert_bits_equal(lp1, lp0, "bf16 weights after a skipped step")
                assert_bits_equal(ma1, ma0, "masters after a skipped step")
            assert_bits_equal(st["exp_avg"], m0, "exp_avg after a skipped step")
            assert_bits_equal(st["exp_avg_sq"], v0, "exp_avg_sq after a skipped step")
            assert list(zo.group_steps) == [s + 1 for s in steps0]
            assert zo.overflow is False and zo.skipped_steps == skipped0
            assert eng.get_global_grad_norm() == math.inf
        elif it == 3:
            n = eng.get_global_grad_norm()
            assert n is not None and math.isfinite(n) and n > 0
    handle.remove()
