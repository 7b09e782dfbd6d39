"""Dropless MoE layer on the host: the ragged layout (64-row aligned, zero-padded expert segments, experts called with
``(rows, offsets)``) computes what the capacity path computes when the capacity is large enough that nothing drops."""
import pytest
import torch

from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
from deepspeed_b200.moe.layer import MoE


def _layer(drop_tokens, E, H, I, k):
    torch.manual_seed(0)
    return MoE(H, GroupedSwiGLUExperts(E, H, I), num_experts=E, k=k, capacity_factor=float(E), eval_capacity_factor=float(E),
               min_capacity=4, drop_tokens=drop_tokens, use_rts=False)


@pytest.mark.parametrize("E,k", [(4, 2), (8, 2), (3, 1)])
def test_dropless_equals_capacity_path_without_drops(E, k):
    H, I, T = 64, 128, 70
    dropless, capacity = _layer(False, E, H, I, k), _layer(True, E, H, I, k)
    capacity.load_state_dict(dropless.state_dict())
    x = torch.randn(2, T // 2, H)
    gy = torch.randn(2, T // 2, H)
    outs = []
    for layer in (dropless, capacity):
        xi = x.clone().requires_grad_(True)
        y, l_aux, counts = layer(xi)
        (y * gy).sum().add(l_aux).backward()
        outs.append((y, xi.grad, counts, *(p.grad for p in layer.parameters())))
    for a, b in zip(*outs):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def test_ragged_experts_zero_outside_segments():
    """GroupedSwiGLUExperts on ``(rows, offsets)``: rows outside ``[offsets[0], offsets[E])`` give zeros, each segment is
    its own expert's SwiGLU MLP."""
    torch.manual_seed(0)
    E, H, I = 3, 64, 128
    ex = GroupedSwiGLUExperts(E, H, I)
    off = torch.tensor([64, 128, 128, 256], dtype=torch.int32)
    rows = torch.randn(300, H)
    y = ex((rows, off))
    assert y.shape == (300, H)
    assert bool((y[:64] == 0).all()) and bool((y[256:] == 0).all())
    for e, (s, t) in enumerate(zip(off[:-1].tolist(), off[1:].tolist())):
        gu = rows[s:t] @ ex.w13[e].t()
        ref = (torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]) @ ex.w2[e].t()
        torch.testing.assert_close(y[s:t], ref, rtol=1e-5, atol=1e-6)


def test_dropless_refuses_other_grouped_containers():
    """A grouped container other than GroupedSwiGLUExperts takes the capacity buffer, not the dropless layout: a clear
    TypeError instead of a failure inside the container."""

    class Stacked(torch.nn.Module):
        num_local_experts = 2

        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.randn(2, 64, 64))

        def forward(self, x):
            return torch.bmm(x, self.w)

    layer = MoE(64, Stacked(), num_experts=2, k=1, drop_tokens=False, use_rts=False)
    with pytest.raises(TypeError, match="GroupedSwiGLUExperts"):
        layer(torch.randn(8, 64))


def test_ragged_swiglu_mlp_refuses_mismatched_weights():
    from deepspeed_b200.ops.linear import ragged_swiglu_mlp
    off = torch.tensor([0, 64, 128], dtype=torch.int32)
    x = torch.randn(128, 64)
    with pytest.raises(ValueError):
        ragged_swiglu_mlp(x, off, torch.randn(2, 256, 72), torch.randn(2, 64, 128))
    with pytest.raises(ValueError):
        ragged_swiglu_mlp(x, off[:2], torch.randn(2, 256, 64), torch.randn(2, 64, 128))
