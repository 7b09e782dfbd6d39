"""GPU tier: every sm_90a kernel against a plain PyTorch fp32 reference of the same op."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda", 0)


def _tol(dtype):
    return {torch.float32: 1e-5, torch.bfloat16: 2e-2, torch.float16: 2e-3}[dtype]


# ----------------------------------------------------------------------------------------------------
# optimizers
# ----------------------------------------------------------------------------------------------------
def _adam_ref(p, g, m, v, lr, b1, b2, eps, wd, step, adamw, gs=1.0):
    g = g.float() * gs
    if not adamw:
        g = g + wd * p
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    upd = (m / (1 - b1**step)) / ((v / (1 - b2**step)).sqrt() + eps)
    if adamw:
        upd = upd + wd * p
    return p - lr * upd, m, v


@pytest.mark.parametrize("n", [1, 7, 1024, 65536 + 5, 3_000_001])
@pytest.mark.parametrize("gdt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("adamw", [True, False])
def test_adam_flat_matches_reference(n, gdt, adamw):
    from deepspeed_b200.ops.kernels import flat_ops
    torch.manual_seed(n)
    d = _dev()
    p = torch.randn(n, device=d)
    g = (torch.randn(n, device=d) * 0.1).to(gdt)
    m = torch.zeros(n, device=d)
    v = torch.zeros(n, device=d)
    out = torch.empty(n, device=d, dtype=torch.bfloat16)
    rp, rm, rv = p.clone(), m.clone(), v.clone()
    gscale = torch.tensor([0.5], device=d)
    for step in (1, 2, 3):
        flat_ops.adam_flat(p, g, m, v, out, lr=1e-2, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.1, step=step,
                           adamw=adamw, grad_scale=2.0, d_gscale=gscale)
        rp, rm, rv = _adam_ref(rp, g, rm, rv, 1e-2, 0.9, 0.95, 1e-8, 0.1, step, adamw, gs=1.0)
    # fp32 math in a different association order (fma) than the torch reference: elements whose second
    # moment is ~0 amplify 1-ulp differences through m/sqrt(v), hence the absolute bound
    assert (p - rp).abs().max() < 2e-4 and (p - rp).abs().mean() < 1e-6
    # (in L2 mode p feeds back into the moments, so the same amplification reaches m)
    assert torch.allclose(m, rm, atol=1e-5, rtol=1e-4) and torch.allclose(v, rv, atol=1e-6, rtol=1e-4)
    assert torch.equal(out, rp.to(torch.bfloat16)) or (out.float() - rp).abs().max() <= rp.abs().max() * 2**-7


def test_adam_flat_skip_flag_and_16bit_master():
    from deepspeed_b200.ops.kernels import flat_ops
    d = _dev()
    n = 4099
    p = torch.randn(n, device=d)
    p0 = p.clone()
    g = torch.randn(n, device=d)
    m, v = torch.zeros(n, device=d), torch.zeros(n, device=d)
    skip = torch.ones(1, dtype=torch.int32, device=d)
    flat_ops.adam_flat(p, g, m, v, None, lr=1e-2, beta1=0.9, beta2=0.99, eps=1e-8, weight_decay=0, step=1, d_skip=skip)
    assert torch.equal(p, p0) and m.abs().sum() == 0
    # same-dtype (bf16 p/m/v) variant used by FusedAdam on 16-bit params
    pb = torch.randn(n, device=d).bfloat16()
    gb = torch.randn(n, device=d).bfloat16()
    mb, vb = torch.zeros_like(pb), torch.zeros_like(pb)
    ref, _, _ = _adam_ref(pb.float(), gb, mb.float(), vb.float(), 1e-2, 0.9, 0.99, 1e-8, 0.0, 1, True)
    flat_ops.adam_flat(pb, gb, mb, vb, None, lr=1e-2, beta1=0.9, beta2=0.99, eps=1e-8, weight_decay=0, step=1)
    assert (pb.float() - ref).abs().max() < 2e-2


def test_fused_adam_multi_tensor_vs_torch_adamw():
    from deepspeed_b200.ops.adam import FusedAdam
    torch.manual_seed(0)
    d = _dev()
    shapes = [(22, ), (64, 33), (128, 128), (1024, 17), (1048576, ), (3, 5, 7)]
    ps = [torch.nn.Parameter(torch.randn(*s, device=d)) for s in shapes]
    qs = [torch.nn.Parameter(p.detach().clone()) for p in ps]
    a = FusedAdam(ps, lr=1e-3, weight_decay=0.01)
    b = torch.optim.AdamW(qs, lr=1e-3, weight_decay=0.01)
    for _ in range(3):
        for p, q in zip(ps, qs):
            gr = torch.randn_like(p)
            p.grad, q.grad = gr.clone(), gr.clone()
        a.step()
        b.step()
    for p, q in zip(ps, qs):
        assert torch.allclose(p, q, atol=1e-5, rtol=1e-5)


def test_lion_lamb_adagrad_sgd_flat():
    from deepspeed_b200.ops.kernels import flat_ops
    torch.manual_seed(0)
    d = _dev()
    n = 100_003
    p = torch.randn(n, device=d)
    g = torch.randn(n, device=d)
    # lion
    m = torch.zeros(n, device=d)
    q, mq = p.clone().cpu(), m.clone().cpu()
    flat_ops.lion_flat(p, g, m, None, lr=1e-3, beta1=0.9, beta2=0.99, weight_decay=0.1)
    flat_ops.lion_flat(q, g.cpu(), mq, None, lr=1e-3, beta1=0.9, beta2=0.99, weight_decay=0.1)
    assert torch.allclose(p.cpu(), q, atol=1e-6) and torch.allclose(m.cpu(), mq, atol=1e-6)
    # adagrad
    h = torch.zeros(n, device=d)
    q, hq = p.clone().cpu(), h.clone().cpu()
    flat_ops.adagrad_flat(p, g, h, None, lr=1e-2, eps=1e-10, weight_decay=0.0)
    flat_ops.adagrad_flat(q, g.cpu(), hq, None, lr=1e-2, eps=1e-10, weight_decay=0.0)
    assert torch.allclose(p.cpu(), q, atol=1e-5)
    # sgd momentum
    b = torch.zeros(n, device=d)
    q, bq = p.clone().cpu(), b.clone().cpu()
    for first in (True, False):
        flat_ops.sgd_flat(p, g, b, None, lr=1e-2, momentum=0.9, first=first, nesterov=True)
        flat_ops.sgd_flat(q, g.cpu(), bq, None, lr=1e-2, momentum=0.9, first=first, nesterov=True)
    assert torch.allclose(p.cpu(), q, atol=1e-5)
    # lamb
    m, v = torch.zeros(n, device=d), torch.zeros(n, device=d)
    q, mq, vq = p.clone().cpu(), m.clone().cpu(), v.clone().cpu()
    c1 = flat_ops.lamb_flat(p, g, m, v, None, lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=1)
    c2 = flat_ops.lamb_flat(q, g.cpu(), mq, vq, None, lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, step=1)
    assert abs(float(c1) - float(c2)) < 1e-3 * abs(float(c2))
    assert torch.allclose(p.cpu(), q, atol=1e-4)


def test_grad_stats_norm_clip_overflow():
    from deepspeed_b200.ops.kernels import flat_ops
    d = _dev()
    for dt in (torch.float32, torch.bfloat16, torch.float16):
        x = torch.randn(1_000_003, device=d).to(dt)
        st = flat_ops.GradStats(d)
        st.accumulate(x)
        st.accumulate(x[:1001])
        ref = (x.float()**2).sum() + (x[:1001].float()**2).sum()
        assert abs(st.sumsq.item() - ref.item()) / ref.item() < 1e-4
        st.finalize(inv_loss_scale=0.5, max_norm=1.0)
        norm = math.sqrt(ref.item()) * 0.5
        assert abs(st.norm.item() - norm) / norm < 1e-4
        assert abs(st.gscale.item() - 0.5 * min(1.0, 1.0 / (norm + 1e-6))) < 1e-6 and st.skip.item() == 0
    x[12345] = float("inf")
    st.reset()
    st.accumulate(x)
    st.finalize(1.0, 0.0)
    assert st.skip.item() == 1 and st.gscale.item() == 0.0


def test_scale_cast_variants():
    from deepspeed_b200.ops.kernels import flat_ops
    d = _dev()
    x = torch.randn(70001, device=d).bfloat16()
    y = torch.ones(70001, device=d)
    flat_ops.scale_cast(x, y, scale=0.25, accumulate=True)
    assert torch.allclose(y, 1 + x.float() * 0.25, atol=1e-6)
    z = torch.empty(70001, device=d, dtype=torch.bfloat16)
    flat_ops.scale_cast(y, z, scale=2.0)
    assert torch.equal(z, (y * 2).bfloat16())


# ----------------------------------------------------------------------------------------------------
# transformer ops
# ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("hidden", [128, 1024, 4096, 8192])
@pytest.mark.parametrize("with_res", [False, True])
def test_rms_norm_fwd_bwd(dtype, hidden, with_res):
    from deepspeed_b200.ops.kernels import transformer_ops as T
    torch.manual_seed(0)
    d = _dev()
    rows = 257
    x = torch.randn(rows, hidden, device=d, dtype=dtype, requires_grad=True)
    r = torch.randn(rows, hidden, device=d, dtype=dtype, requires_grad=True) if with_res else None
    w = (1 + 0.1 * torch.randn(hidden, device=d)).to(dtype).requires_grad_(True)
    if with_res:
        y, s = T.rms_norm(x, w, 1e-5, residual=r)
        (y.float().sum() * 0.5 + (s.float() * 0.1).sum()).backward()
    else:
        y = T.rms_norm(x, w, 1e-5)
        (y.float().sum() * 0.5).backward()
    xf = x.detach().float().requires_grad_(True)
    rf = r.detach().float().requires_grad_(True) if with_res else None
    wf = w.detach().float().requires_grad_(True)
    xin = (xf + rf).to(dtype).float() if with_res else xf
    if with_res:
        xin = xf + rf  # for grads; value uses rounded sum below
    yr = xin * torch.rsqrt(xin.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    loss = yr.sum() * 0.5 + ((xin * 0.1).sum() if with_res else 0)
    loss.backward()
    tol = _tol(dtype)
    assert (y.float() - yr).abs().max() < tol * max(1.0, yr.abs().max().item())
    assert (x.grad.float() - xf.grad).abs().max() < tol * max(1.0, xf.grad.abs().max().item())
    assert (w.grad.float() - wf.grad).abs().max() < 4 * tol * max(1.0, wf.grad.abs().max().item())
    if with_res:
        assert (r.grad.float() - rf.grad).abs().max() < tol * max(1.0, rf.grad.abs().max().item())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_layer_norm_fwd_bwd(dtype):
    from deepspeed_b200.ops.kernels import transformer_ops as T
    torch.manual_seed(0)
    d = _dev()
    rows, hidden = 300, 1024
    x = torch.randn(rows, hidden, device=d, dtype=dtype, requires_grad=True)
    w = torch.randn(hidden, device=d).to(dtype).requires_grad_(True)
    b = torch.randn(hidden, device=d).to(dtype).requires_grad_(True)
    y = T.layer_norm(x, w, b, 1e-5)
    y.float().pow(2).sum().backward()
    xf, wf, bf = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    yr = torch.nn.functional.layer_norm(xf, (hidden, ), wf, bf, 1e-5)
    yr.pow(2).sum().backward()
    tol = _tol(dtype)
    assert (y.float() - yr).abs().max() < tol * yr.abs().max()
    assert (x.grad.float() - xf.grad).abs().max() < tol * xf.grad.abs().max()
    assert (w.grad.float() - wf.grad).abs().max() < 4 * tol * wf.grad.abs().max()
    assert (b.grad.float() - bf.grad).abs().max() < 4 * tol * bf.grad.abs().max()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_rope_packed_qk_fwd_bwd(dtype):
    from deepspeed_b200.ops.kernels import transformer_ops as T
    torch.manual_seed(0)
    d = _dev()
    B, S, hq, hkv, hd = 2, 64, 8, 2, 128
    table = T.RotaryTable(hd, 256, 500000.0, d)
    qkv = torch.randn(B * S, (hq + 2 * hkv) * hd, device=d, dtype=dtype)
    ref = qkv.clone().cpu().float()
    T.rope_qk_inplace(qkv, hq, hkv, hd, table, None, S)
    tc = T.RotaryTable(hd, 256, 500000.0, "cpu")
    T.rope_qk_inplace(ref, hq, hkv, hd, tc, None, S)
    assert (qkv.float().cpu() - ref).abs().max() < _tol(dtype) * 4
    # backward rotation is the inverse
    T.rope_qk_inplace(qkv, hq, hkv, hd, table, None, S, backward=True)
    T.rope_qk_inplace(ref, hq, hkv, hd, tc, None, S, backward=True)
    assert (qkv.float().cpu() - ref).abs().max() < _tol(dtype) * 4
    # explicit positions
    pos = torch.randint(0, 256, (B * S, ), device=d, dtype=torch.int32)
    q2 = torch.randn(B * S, (hq + 2 * hkv) * hd, device=d, dtype=dtype)
    r2 = q2.clone().cpu().float()
    T.rope_qk_inplace(q2, hq, hkv, hd, table, pos, S)
    T.rope_qk_inplace(r2, hq, hkv, hd, tc, pos.cpu(), S)
    assert (q2.float().cpu() - r2).abs().max() < _tol(dtype) * 4


@pytest.mark.parametrize("act", ["silu", "gelu_tanh", "relu", "gelu"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_gated_act_fwd_bwd(act, dtype):
    from deepspeed_b200.ops.kernels import transformer_ops as T
    torch.manual_seed(0)
    d = _dev()
    gu = torch.randn(130, 2 * 1024, device=d, dtype=dtype, requires_grad=True)
    out = T.gated_act(gu, act)
    out.float().pow(2).sum().backward()
    gf = gu.detach().float().requires_grad_(True)
    g, u = gf[:, :1024], gf[:, 1024:]
    a = T._act_torch(g, T.act_code(act))
    (a * u).pow(2).sum().backward()
    tol = _tol(dtype)
    assert (out.float() - (a * u)).abs().max() < tol * 8
    assert (gu.grad.float() - gf.grad).abs().max() < tol * max(1.0, gf.grad.abs().max().item())


@pytest.mark.parametrize("tokens,inter", [(8192, 8192)])  # the Llama-3.2-3B training step: 2 x 4096 tokens, I = 8192
def test_swiglu_raw_at_step_shape(tokens, inter):
    """``gated_act_fwd_raw`` / ``gated_act_bwd`` (the kernels behind the library SwiGLU GEMMs) against float64, per element."""
    from deepspeed_b200.ops.kernels import transformer_ops as T
    from tests.numerics import assert_within, dswiglu_reference, swiglu_reference
    g = torch.Generator(device="cuda").manual_seed(0)
    gu = (torch.randn(tokens, 2 * inter, generator=g, device="cuda") * 2).bfloat16()
    dout = torch.randn(tokens, inter, generator=g, device="cuda").bfloat16()
    out = T.gated_act_fwd_raw(gu)
    dgu = T.gated_act_bwd(dout, gu)
    ref, bound = swiglu_reference(gu[:, :inter], gu[:, inter:])
    assert_within(out, ref, bound, "silu(gate) * up")
    del ref, bound
    # dout is bf16, so dout * up is exact in fp32
    dgate, dgate_bound, dup, dup_bound = dswiglu_reference(dout, gu[:, :inter], gu[:, inter:])
    assert_within(dgu[:, :inter], dgate, dgate_bound, "d(gate)")
    assert_within(dgu[:, inter:], dup, dup_bound, "d(up)")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("vocab", [1000, 32064, 128256])
def test_softmax_xent_and_grad(dtype, vocab):
    from deepspeed_b200.ops.kernels import transformer_ops as T
    torch.manual_seed(0)
    d = _dev()
    rows = 37
    logits = (torch.randn(rows, vocab, device=d) * 3).to(dtype)
    labels = torch.randint(0, vocab, (rows, ), device=d)
    labels[5] = -100
    lf = logits.float().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lf, labels, ignore_index=-100, reduction="sum")
    ref.backward()
    work = logits.clone()
    loss, grad = T.softmax_xent_fwd_bwd(work, labels, gscale=1.0)
    assert abs(loss.sum().item() - ref.item()) < 2e-3 * abs(ref.item())
    assert loss[5].item() == 0.0 and grad[5].abs().sum() == 0
    assert (grad.float() - lf.grad).abs().max() < (1e-2 if dtype == torch.bfloat16 else 1e-5)
    lg = logits.clone().requires_grad_(True)
    l2 = T.cross_entropy(lg, labels)
    l2.backward()
    assert abs(l2.item() - ref.item() / (rows - 1)) < 2e-3 * abs(l2.item())


def test_bias_act_and_fused_add():
    from deepspeed_b200.ops.kernels import transformer_ops as T
    torch.manual_seed(0)
    d = _dev()
    x = torch.randn(64, 512, device=d, dtype=torch.bfloat16, requires_grad=True)
    b = torch.randn(512, device=d, dtype=torch.bfloat16, requires_grad=True)
    r = torch.randn(64, 512, device=d, dtype=torch.bfloat16)
    y = T.bias_act(x, b, "gelu", residual=r)
    ref = torch.nn.functional.gelu(x.float() + b.float()) + r.float()
    assert (y.float() - ref).abs().max() < 3e-2
    y.float().sum().backward()
    xf = x.detach().float().requires_grad_(True)
    (torch.nn.functional.gelu(xf + b.detach().float())).sum().backward()
    assert (x.grad.float() - xf.grad).abs().max() < 2e-2
    s = T.fused_add(x.detach(), r, r, None, scale=0.5)
    assert (s.float() - (x.detach().float() + 2 * r.float()) * 0.5).abs().max() < 3e-2
