"""The fused softmax cross-entropy kernel against float64 ``log_softmax``: per-row loss and the in-place gradient.

Vocabulary sizes pick the kernel's load paths: 128256 (the Llama 3 LM head) is all 16-byte vectors, 50257 and 32001 have
rows that are not 16-byte aligned and take the scalar loop, and 1003 stored with a row stride of 1008 takes vectors plus a
3-element tail.  Bounds are per element, from ``tests/numerics.py``.
"""
import pytest
import torch

from tests.numerics import assert_within, xent_bounds, xent_reference

pytestmark = pytest.mark.gpu

IGNORE = -100
VOCABS = [(128256, 128256), (50257, 50257), (32001, 32001), (1003, 1008)]  # (vocab, row stride)
PATTERNS = ["normal", "large", "label_at_max", "label_at_min", "neg_inf", "only_label"]


def _case(rows, vocab, stride, dtype, pattern, seed):
    """Logits viewed from a ``[rows, stride]`` buffer whose padding holds a sentinel, and int64 labels."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(rows, vocab, generator=g, device="cuda") * 3
    if pattern == "large":
        z = 80 + z * 1.5  # exp() of these overflows fp32 unless the row maximum is subtracted first
    z = z.to(dtype)
    labels = torch.randint(0, vocab, (rows, ), generator=g, device="cuda")
    if pattern == "label_at_max":
        labels = z.float().argmax(-1)
    elif pattern == "label_at_min":
        labels = z.float().argmin(-1)
    elif pattern == "neg_inf":
        drop = torch.rand(rows, vocab, generator=g, device="cuda") < 0.1
        drop.scatter_(1, labels[:, None], False)
        z = z.masked_fill(drop, float("-inf"))
    elif pattern == "only_label":
        keep = z.gather(1, labels[:, None])
        z = torch.full_like(z, float("-inf")).scatter_(1, labels[:, None], keep)
    if rows >= 8:
        labels[3] = IGNORE
        labels[5] = vocab  # out of range: ignored like IGNORE
        labels[7] = -1
    buf = torch.full((rows, stride), 7.0, device="cuda", dtype=dtype)
    buf[:, :vocab] = z
    return buf, labels


def _run_and_check(buf, vocab, labels, dtype, gscale=1.0, d_gscale=None):
    from deepspeed_b200.ops.kernels import transformer_ops as T
    logits = buf[:, :vocab]
    gs = gscale * (float(d_gscale) if d_gscale is not None else 1.0)
    loss_ref, grad_ref, lse, p, valid = xent_reference(logits, labels, IGNORE, gs)
    loss_bound, grad_bound = xent_bounds(logits, loss_ref, grad_ref, lse, p, gs, dtype)
    pad = buf[:, vocab:].clone()
    loss, grad = T.softmax_xent_fwd_bwd(logits, labels, gscale, d_gscale, IGNORE, True)
    assert grad.data_ptr() == logits.data_ptr()
    assert torch.equal(buf[:, vocab:], pad), "the gradient spilled into the row padding"
    assert_within(loss, loss_ref, loss_bound, "loss")
    assert_within(grad, grad_ref, grad_bound, "gradient")
    ignored = ~valid
    assert bool((loss[ignored] == 0).all()) and bool((grad[ignored] == 0).all())
    return loss, grad


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("rows", [1, 37, 2048])  # 2048: one LM-head chunk
@pytest.mark.parametrize("vocab,stride", VOCABS)
def test_xent_bf16(vocab, stride, rows, pattern):
    buf, labels = _case(rows, vocab, stride, torch.bfloat16, pattern, seed=vocab + rows)
    _run_and_check(buf, vocab, labels, torch.bfloat16)


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("rows", [1, 37, 2048])
@pytest.mark.parametrize("vocab,stride", [(128256, 128256), (32001, 32001), (1003, 1008)])  # 32001, 1003: not % 4
def test_xent_fp32(vocab, stride, rows, pattern):
    buf, labels = _case(rows, vocab, stride, torch.float32, pattern, seed=vocab + rows)
    _run_and_check(buf, vocab, labels, torch.float32)


@pytest.mark.parametrize("mode", ["host", "device", "both"])
@pytest.mark.parametrize("vocab,stride", VOCABS)
def test_xent_gradient_scale(vocab, stride, mode):
    """The gradient is scaled by the host ``gscale`` times the device scalar ``d_gscale`` (the LM head passes 1/n)."""
    buf, labels = _case(37, vocab, stride, torch.bfloat16, "normal", seed=vocab)
    gscale = {"host": 0.37, "device": 1.0, "both": 3.0}[mode]
    d_gscale = None if mode == "host" else torch.tensor([1 / 37], device="cuda")
    _run_and_check(buf, vocab, labels, torch.bfloat16, gscale, d_gscale)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("vocab,stride", [(50257, 50257), (1003, 1008)])
def test_xent_label_contract_matches_cpu(vocab, stride, dtype):
    """Labels that are ``ignore_index``, negative or ``>= vocab`` give zero loss and gradient on the GPU and the host."""
    from deepspeed_b200.ops.kernels import transformer_ops as T
    buf, labels = _case(37, vocab, stride, dtype, "normal", seed=stride)
    labels[0], labels[1], labels[2], labels[4] = -5, vocab + 7, vocab - 1, 0
    host = buf[:, :vocab].cpu()
    loss, _ = _run_and_check(buf, vocab, labels, dtype)
    loss_cpu, grad_cpu = T.softmax_xent_fwd_bwd(host.clone(), labels.cpu(), 1.0, None, IGNORE, True)
    valid = T.xent_valid(labels, vocab, IGNORE)
    assert torch.equal(valid.cpu(), loss_cpu != 0)
    assert bool((grad_cpu[~valid.cpu()] == 0).all())
    # both sides hold the same float64 reference to the kernel's bound (the host computes exp and log exactly rounded)
    loss_ref, grad_ref, lse, p, _ = xent_reference(host, labels.cpu(), IGNORE, 1.0)
    loss_bound, grad_bound = xent_bounds(host, loss_ref, grad_ref, lse, p, 1.0, dtype)
    assert_within(loss_cpu, loss_ref, loss_bound, "host loss")
    assert_within(grad_cpu, grad_ref, grad_bound, "host gradient")
    assert_within(loss.cpu(), loss_cpu, 2 * loss_bound, "GPU vs host loss")
