"""Host-tier optimizer kernels (``csrc/cpu/cpu_optim.cpp``) per element against the float64 references in
``tests/numerics.py``, and those references against hand-computed steps and torch's own optimizers."""
import ctypes
import math

import pytest
import torch

from tests.numerics import (U, adagrad_reference, adam_hyper, adam_reference, assert_bits_equal, assert_within,
                            clip_coeff_reference, f32, lion_reference, sgd_reference, sumsq_bound, sumsq_depth)

F, I64 = ctypes.c_float, ctypes.c_int64
DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _lib():
    from deepspeed_b200.ops import native
    return native.cpu()


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


LEVEL = _lib().dsb_cpu_simd_level()
WIDTH = {2: 16, 1: 8, 0: 1}[LEVEL]
SIMD = {2: "avx512", 1: "avx2", 0: "scalar"}[LEVEL]
# tails of 1..15 elements past a whole number of SIMD vectors, and a size spanning several 64 Ki-element OpenMP tiles
SIZES = [3 * WIDTH + t for t in range(1, 16)] + [2 * 65536 + 16 * 5 + 13]


@pytest.fixture
def threads():
    lib = _lib()
    before = lib.dsb_cpu_get_threads()
    yield lib
    lib.dsb_cpu_set_threads(before)


def _data(n, seed, gdt):
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=gen)
    g = (torch.randn(n, generator=gen) * 0.3).to(gdt)
    m = torch.randn(n, generator=gen) * 0.05
    v = torch.rand(n, generator=gen) * 0.01
    return p, g, m, v


# ---------------------------------------------------------------------------------------------------------------------
# the references themselves
# ---------------------------------------------------------------------------------------------------------------------
def test_references_hand_computed():
    one = lambda x: torch.tensor([x], dtype=torch.float32)  # noqa: E731
    # Adam, step 1, powers of two: g1 = 0.5, m = 0.25, v = 0.0625, mh = 0.5, vh = 0.25, u = 0.5 / 0.5 = 1
    h = adam_hyper(lr=0.125, beta1=0.5, beta2=0.75, eps=0.0, weight_decay=0.0, step=1)
    p, m, v, bp, bm, bv = adam_reference(one(1.0), one(0.5), one(0.0), one(0.0), h)
    assert (float(p), float(m), float(v)) == (0.875, 0.25, 0.0625)
    # a few fp32 ulps: 2**-24 at 0.875, 2**-25 at 0.25, 2**-28 at 0.0625
    assert 0 < float(bp) < 4 * 2.0**-24 and 0 < float(bm) < 4 * 2.0**-25 and 0 < float(bv) < 8 * 2.0**-28
    # AdamW adds wd * p to u (1 + 0.5 * 1), L2 adds it to the gradient (g = 1: m = 0.5, v = 0.25, u = 1)
    h = adam_hyper(lr=0.125, beta1=0.5, beta2=0.75, eps=0.0, weight_decay=0.5, step=1)
    assert float(adam_reference(one(1.0), one(0.5), one(0.0), one(0.0), h)[0]) == 1 - 0.125 * 1.5
    h = adam_hyper(lr=0.125, beta1=0.5, beta2=0.75, eps=0.0, weight_decay=0.5, step=1, adamw=False)
    p, m, v = adam_reference(one(1.0), one(0.5), one(0.0), one(0.0), h)[:3]
    assert (float(p), float(m), float(v)) == (0.875, 0.5, 0.25)
    # the hyperparameters are the kernel's fp32 values: 1 - fp32(0.9), not 1 - 0.9
    h = adam_hyper(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0, step=3, grad_scale=0.1, d_gscale=3.0)
    assert h["b1m"] == 1.0 - f32(0.9) != 1.0 - 0.9 and h["bc2"] == f32(1 - 0.999**3)
    assert h["gs"] == f32(f32(0.1) * 3.0)
    # Lion: c = 0.5 * 0.5 + 0.5 * (-0.5) = 0 exactly, so the sign is 0 and only the decay moves p
    p, m, s, _, _ = lion_reference(one(2.0), one(-0.5), one(0.5), lr=0.25, beta1=0.5, beta2=0.5, weight_decay=0.5,
                                   gs=1.0)
    assert (float(s), float(p), float(m)) == (0.0, 2.0 * (1 - 0.125), 0.0)
    # Adagrad: h = 4, p = 1 - 0.5 * 2 / 2
    p, hs, _, _ = adagrad_reference(one(1.0), one(2.0), one(0.0), lr=0.5, eps=0.0, weight_decay=0.0, gs=1.0)
    assert (float(p), float(hs)) == (0.5, 4.0)
    # SGD, nesterov, first step: buf = d = 1, direction d + 0.5 buf
    p, b, _, _ = sgd_reference(one(1.0), one(1.0), one(7.0), lr=0.25, momentum=0.5, dampening=0.5, weight_decay=0.0,
                               nesterov=True, first=True, gs=1.0)
    assert (float(p), float(b)) == (1 - 0.25 * 1.5, 1.0)
    # second step: buf = 0.5 * 1 + (1 - 0.5) * 1 = 1 (dampening applies after the first step only)
    p, b, _, _ = sgd_reference(one(1.0), one(1.0), one(1.0), lr=0.25, momentum=0.5, dampening=0.5, weight_decay=0.0,
                               nesterov=False, first=False, gs=1.0)
    assert (float(p), float(b)) == (0.75, 1.0)
    # clip: ss = 4, inv_ls = 0.5 -> norm = 1; max_norm 0.5 clips, 2.0 does not, 0 disables
    c, norm, rel_c, _ = clip_coeff_reference(4.0, 0.5, 0.5)
    assert norm == 1.0 and c == 0.5 * 0.5 / (1 + 1e-6) and 0 < rel_c < 1e-6
    assert clip_coeff_reference(4.0, 0.5, 2.0)[0] == 0.5 and clip_coeff_reference(4.0, 0.5, 0.0)[0] == 0.5
    # sum of squares: 1 element is a scalar-tail chain of 1, then two block trees, the partials sum and the accumulate
    assert sumsq_depth(1, torch.float32) == 1 + 10 + 1 + 10 + 1
    assert sumsq_depth(10**8, torch.float32) > 10**8 // (528 * 512)
    assert 23 * U * 100 < sumsq_bound(100.0, 1, torch.bfloat16) < 24 * U * 100


@pytest.mark.parametrize("adamw", [True, False])
def test_references_match_torch_optimizers_in_float64(adamw):
    """The float64 references follow torch.optim's semantics: run torch's optimizers on float64 parameters and compare
    over several steps, feeding the same state into the reference each step."""
    gen = torch.Generator().manual_seed(7)
    n = 257
    p0 = torch.randn(n, generator=gen, dtype=torch.float64)
    grads = [torch.randn(n, generator=gen, dtype=torch.float64) for _ in range(4)]
    lr, b1, b2, eps, wd = 2.0**-7, 0.5, 0.75, 2.0**-20, 0.25  # fp32-exact, so the fp32 rounding of the reference is moot
    # Adam / AdamW
    q = torch.nn.Parameter(p0.clone())
    opt = (torch.optim.AdamW if adamw else torch.optim.Adam)([q], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    p, m, v = p0.clone(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    for t, g in enumerate(grads, 1):
        q.grad = g.clone()
        opt.step()  # AdamW decays p by (1 - lr wd) first; the kernels add wd p to the update: the same p'
        p, m, v = adam_reference(p, g, m, v, adam_hyper(lr, b1, b2, eps, wd, t, adamw=adamw))[:3]
        torch.testing.assert_close(q.detach(), p, rtol=1e-12, atol=1e-14)
        torch.testing.assert_close(opt.state[q]["exp_avg_sq"], v, rtol=1e-12, atol=1e-16)
    # Adagrad
    q = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adagrad([q], lr=lr, eps=eps, weight_decay=wd)
    p, hs = p0.clone(), torch.zeros(n, dtype=torch.float64)
    for g in grads:
        q.grad = g.clone()
        opt.step()
        p, hs = adagrad_reference(p, g, hs, lr, eps, wd, 1.0)[:2]
        torch.testing.assert_close(q.detach(), p, rtol=1e-12, atol=1e-14)
    # SGD with momentum, dampening, nesterov off and on
    for nesterov, damp in ((False, 0.25), (True, 0.0)):
        q = torch.nn.Parameter(p0.clone())
        opt = torch.optim.SGD([q], lr=lr, momentum=0.5, dampening=damp, weight_decay=wd, nesterov=nesterov)
        p, buf = p0.clone(), torch.zeros(n, dtype=torch.float64)
        for t, g in enumerate(grads):
            q.grad = g.clone()
            opt.step()
            p, buf = sgd_reference(p, g, buf, lr, 0.5, damp, wd, nesterov, t == 0, 1.0)[:2]
            torch.testing.assert_close(q.detach(), p, rtol=1e-12, atol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------
# host kernels
# ---------------------------------------------------------------------------------------------------------------------
def _cpu_adam(p, g, m, v, out, h, odt=torch.bfloat16):
    rc = _lib().dsb_cpu_adam(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(out), I64(p.numel()), DT[g.dtype],
                             DT[out.dtype] if out is not None else DT[odt], F(h["lr"]), F(h["b1"]), F(h["b2"]),
                             F(h["eps"]), F(h["wd"]), F(h["bc1"]), F(h["bc2"]), int(h["adamw"]), F(h["gs"]))
    assert rc == 0


@pytest.mark.parametrize("n", SIZES, ids=lambda n: f"{SIMD}-n{n}")
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16, torch.float16], ids=str)
def test_cpu_adam_per_element(n, gdt):
    p, g, m, v = _data(n, n, gdt)
    for step, (adamw, odt) in enumerate(((True, torch.bfloat16), (False, torch.float16), (True, None)), 1):
        h = adam_hyper(lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=step, adamw=adamw,
                       grad_scale=0.75)
        p0, m0, v0 = p.clone(), m.clone(), v.clone()
        out = torch.full((n, ), 7.0, dtype=odt) if odt is not None else None
        _cpu_adam(p, g, m, v, out, h)
        rp, rm, rv, bp, bm, bv = adam_reference(p0, g, m0, v0, h)
        what = f"{SIMD} n={n} step={step}"
        assert_within(p, rp, bp, f"p {what}")
        assert_within(m, rm, bm, f"m {what}")
        assert_within(v, rv, bv, f"v {what}")
        if out is not None:
            assert_bits_equal(out, p.to(odt), f"out {what}")


@pytest.mark.parametrize("n", SIZES[::4] + SIZES[-1:], ids=lambda n: f"{SIMD}-n{n}")
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16, torch.float16], ids=str)
def test_cpu_lion_per_element(n, gdt):
    p, g, m, _ = _data(n, n + 1, gdt)
    m[:3] = 0.0
    g[:3] = 0.0  # c == 0 ties: sign 0, only the decay moves p
    out = torch.empty(n, dtype=torch.bfloat16)
    p0, m0 = p.clone(), m.clone()
    rc = _lib().dsb_cpu_lion(_ptr(p), _ptr(g), _ptr(m), _ptr(out), I64(n), DT[gdt], DT[torch.bfloat16], F(1e-2),
                             F(0.9), F(0.99), F(0.1), F(0.5))
    assert rc == 0
    rp, rm, _, bp, bm = lion_reference(p0, g, m0, 1e-2, 0.9, 0.99, 0.1, 0.5, fused=False)
    assert_within(p, rp, bp, "lion p")
    assert_within(m, rm, bm, "lion m")
    assert_bits_equal(out, p.bfloat16(), "lion out")
    assert_within(p[:3], p0[:3].double() * (1 - f32(1e-2) * f32(0.1)), 2 * U * p0[:3].double().abs(), "lion tie")


@pytest.mark.parametrize("n", SIZES[::4] + SIZES[-1:], ids=lambda n: f"{SIMD}-n{n}")
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16, torch.float16], ids=str)
def test_cpu_adagrad_per_element(n, gdt):
    p, g, _, v = _data(n, n + 2, gdt)
    hs = v.clone()
    out = torch.empty(n, dtype=torch.float16)
    p0, h0 = p.clone(), hs.clone()
    rc = _lib().dsb_cpu_adagrad(_ptr(p), _ptr(g), _ptr(hs), _ptr(out), I64(n), DT[gdt], DT[torch.float16], F(1e-2),
                                F(1e-10), F(0.01), F(2.0))
    assert rc == 0
    rp, rh, bp, bh = adagrad_reference(p0, g, h0, 1e-2, 1e-10, 0.01, 2.0)
    assert_within(p, rp, bp, "adagrad p")
    assert_within(hs, rh, bh, "adagrad h")
    assert_bits_equal(out, p.half(), "adagrad out")


def _special_fp32(n, seed):
    """fp32 values that exercise a 16-bit cast: ties at both formats' rounding points, subnormals of fp16 and fp32,
    overflow past 65504, signed zeros and infinities."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=gen) * torch.exp2(torch.randint(-30, 30, (n, ), generator=gen).float())
    bits = x.view(torch.int32)
    x[0::7] = (bits[0::7] & ~0xFFFF | 0x8000).view(torch.float32)  # bf16 ties
    x[1::7] = (bits[1::7] & ~0x1FFF | 0x1000).view(torch.float32)  # fp16 ties
    x[2::11] = torch.randn(x[2::11].shape, generator=gen) * 2.0**-20  # fp16 subnormals
    x[3::13] = torch.randn(x[3::13].shape, generator=gen) * 2.0**-135  # fp32 subnormals
    x[4::17] = 65520.0  # rounds to inf in fp16 (the tie at 65520 goes up)
    x[5::17] = 65519.0  # rounds to 65504
    x[:4] = torch.tensor([0.0, -0.0, math.inf, -math.inf])
    return x


@pytest.mark.parametrize("odt", [torch.bfloat16, torch.float16], ids=str)
def test_cpu_cast_is_round_to_nearest_even(odt):
    n = 65536 + 37
    x = _special_fp32(n, 11)
    y = torch.empty(n, dtype=odt)
    assert _lib().dsb_cpu_cast(_ptr(x), _ptr(y), I64(n), DT[odt]) == 0
    assert_bits_equal(y, x.to(odt), f"cast to {odt}")
    x[6] = math.nan
    assert _lib().dsb_cpu_cast(_ptr(x), _ptr(y), I64(n), DT[odt]) == 0
    assert math.isnan(float(y[6]))
    assert _lib().dsb_cpu_cast(_ptr(x), _ptr(y), I64(n), 0) == -1  # only 16-bit targets


def test_cpu_adam_out_is_round_to_nearest_even_at_ties():
    """The SIMD paths' own bf16 rounding, on masters that sit exactly at bf16 ties after a zero-gradient step."""
    n = 3 * WIDTH + 7
    p = _special_fp32(n, 5).clamp(-1e30, 1e30).nan_to_num(0.0)
    g = torch.zeros(n)
    m, v = torch.zeros(n), torch.zeros(n)
    for odt in (torch.bfloat16, torch.float16):
        out = torch.empty(n, dtype=odt)
        h = adam_hyper(lr=1e-3, beta1=0.9, beta2=0.99, eps=1e-8, weight_decay=0.0, step=1)
        q = p.clone()
        _cpu_adam(q, g, m, v, out, h)
        assert_bits_equal(q, p, "zero gradient, no decay: p unchanged")
        assert_bits_equal(out, p.to(odt), f"out {odt}")


@pytest.mark.parametrize("kernel", ["adam", "lion", "adagrad", "cast"])
def test_cpu_threaded_equals_single_thread(kernel, threads):
    n = 5 * 65536 + 29
    p, g, m, v = _data(n, 3, torch.bfloat16)
    res = []
    for nt in (1, max(2, threads.dsb_cpu_get_threads())):
        threads.dsb_cpu_set_threads(nt)
        q, mq, vq = p.clone(), m.clone(), v.clone()
        out = torch.empty(n, dtype=torch.bfloat16)
        if kernel == "adam":
            _cpu_adam(q, g, mq, vq, out, adam_hyper(1e-2, 0.9, 0.95, 1e-8, 0.1, 2))
        elif kernel == "lion":
            threads.dsb_cpu_lion(_ptr(q), _ptr(g), _ptr(mq), _ptr(out), I64(n), 2, 2, F(1e-2), F(0.9), F(0.99),
                                 F(0.1), F(1.0))
        elif kernel == "adagrad":
            threads.dsb_cpu_adagrad(_ptr(q), _ptr(g), _ptr(vq), _ptr(out), I64(n), 2, 2, F(1e-2), F(1e-10), F(0.0),
                                    F(1.0))
        else:
            threads.dsb_cpu_cast(_ptr(q), _ptr(out), I64(n), 2)
        res.append((q, mq, vq, out))
    for a, b in zip(*res):
        assert_bits_equal(a, b, f"{kernel}: threaded vs single-thread")
