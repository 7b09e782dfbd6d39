"""``chunked_linear_xent`` and the host softmax cross entropy against float64, without a GPU.

The host path runs the same chunk loop, gradient scaling and ``dW`` accumulation as the GPU path; here at H 64, V 1003,
300 tokens in chunks of 128 (a ragged last chunk).  Bounds are per element, from ``tests/numerics.py``.
"""
import pytest
import torch

from tests.numerics import assert_within, chunked_xent_reference, xent_bounds, xent_reference

H, V, T, CHUNK, IGNORE = 64, 1003, 300, 128, -100


def _inputs(dtype, all_ignored_chunk=False):
    g = torch.Generator().manual_seed(0)
    h = torch.randn(T, H, generator=g).to(dtype)
    w = (torch.randn(V, H, generator=g) * 0.3).to(dtype)
    labels = torch.randint(0, V, (T, ), generator=g)
    labels[torch.rand(T, generator=g) < 0.1] = IGNORE
    if all_ignored_chunk:
        labels[CHUNK:2 * CHUNK] = IGNORE
    return h, w, labels


@pytest.mark.parametrize("all_ignored_chunk", [False, True])
@pytest.mark.parametrize("scale", [1.0, 1024.0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_chunked_linear_xent_cpu(dtype, scale, all_ignored_chunk):
    from deepspeed_b200.ops.linear import chunked_linear_xent
    h, w, labels = _inputs(dtype, all_ignored_chunk)
    loss_ref, dh_ref, dw_ref, loss_bound, dh_bound, dw_bound = chunked_xent_reference(h, w, labels, CHUNK, IGNORE)
    with torch.no_grad():
        loss_ng = chunked_linear_xent(h, w, labels, chunk=CHUNK, ignore_index=IGNORE)
    hp = h.clone().requires_grad_(True)
    wp = w.clone().requires_grad_(True)
    loss = chunked_linear_xent(hp, wp, labels, chunk=CHUNK, ignore_index=IGNORE, assumed_scale=scale)
    (loss * (0.5 * scale)).backward()  # dloss / assumed_scale = 0.5, a power of two
    assert torch.equal(loss_ng, loss.detach())
    assert_within(loss.detach().reshape(1), torch.tensor([loss_ref]), loss_bound, "loss")
    f = 0.5 * scale
    assert_within(hp.grad, dh_ref * f, dh_bound * f, "dh")
    assert bool((hp.grad[labels == IGNORE] == 0).all())
    assert_within(wp.grad, dw_ref * f, dw_bound * f, "dW")


def test_chunked_linear_xent_counts_only_labels_in_range():
    """Labels outside [0, V) are ignored like ``ignore_index``: no loss, no gradient, not in the mean's count."""
    from deepspeed_b200.ops.linear import chunked_linear_xent
    h, w, labels = _inputs(torch.float32)
    odd = labels.clone()
    odd[labels == IGNORE] = V + 5
    odd[:3] = -7
    ref = labels.clone()
    ref[:3] = IGNORE
    for lab in (odd, ref):
        with torch.no_grad():
            assert chunked_linear_xent(h, w, lab, chunk=CHUNK, ignore_index=IGNORE).item() == pytest.approx(
                chunked_linear_xent(h, w, ref, chunk=CHUNK, ignore_index=IGNORE).item(), rel=1e-6)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_softmax_xent_host_label_contract(dtype):
    """The host fallback follows the kernel's label contract: only labels in [0, vocab) other than ``ignore_index``
    count; a negative label is not clamped to class 0 and a label >= vocab does not raise."""
    from deepspeed_b200.ops.kernels import transformer_ops as T
    g = torch.Generator().manual_seed(1)
    logits = (torch.randn(9, V, generator=g) * 3).to(dtype)
    labels = torch.tensor([0, V - 1, IGNORE, -1, -5, V, V + 100, 17, 500])
    work = logits.clone()
    loss, grad = T.softmax_xent_fwd_bwd(work, labels, 0.25, torch.tensor([2.0]), IGNORE, True)
    assert grad is work
    loss_ref, grad_ref, lse, p, valid = xent_reference(logits, labels, IGNORE, 0.5)
    assert valid.tolist() == [True, True, False, False, False, False, False, True, True]
    loss_bound, grad_bound = xent_bounds(logits, loss_ref, grad_ref, lse, p, 0.5, dtype)
    assert_within(loss, loss_ref, loss_bound, "loss")
    assert_within(grad, grad_ref, grad_bound, "gradient")
    assert bool((loss[~valid] == 0).all()) and bool((grad[~valid] == 0).all())
