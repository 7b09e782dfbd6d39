"""Where the training nodes put their weight gradients under a ZeRO owner, on the host.

Each node runs two micro steps with a fake owner whose gradient views are bf16 (the product's dtype) or fp32 (fp32
accumulation), and once without an owner.  A gradient written into the owner's view is stored on the first micro step
and accumulated on the second, and its weight is marked ready once per backward; a gradient the node hands back to
autograd leaves the view alone and marks nothing.  Marking the last of a unit's weights reduces the unit, which under
ZeRO-3 releases the gathered weights and with the step fused into backward rewrites them: the fake owner overwrites the
node's weights with NaN at that point, so a weight read after it shows up as a non-finite gradient."""
import weakref

import pytest
import torch

from deepspeed_b200.ops import linear

BF16 = torch.bfloat16
NAN = float("nan")
NODES = ["flat_linear", "swiglu_mlp", "grouped_swiglu_mlp"] + [
    f"{n}-{r}" for n in ("fp8_linear", "fp8_swiglu_mlp", "fp8_ragged_swiglu_mlp") for r in ("tensorwise", "blockwise")
]


class _Owner:
    """Fake ZeRO owner of one node's weights: a gradient view per weight, NaN until written (the real flat buffer is
    not cleared between steps), fresh until its first mark, and the weights overwritten with NaN when the last of them
    is marked ready."""

    def __init__(self, weights, dtype):
        self.weights = weights
        self.views = {id(w): torch.full(w.shape, NAN, dtype=dtype) for w in weights}
        self.written = set()
        self.marks = []
        for w in weights:
            w._ds_zero = weakref.ref(self)

    def grad_view_for(self, w):
        return self.views[id(w)]

    def grad_is_fresh(self, w):
        return id(w) not in self.written

    def mark_grad_ready(self, w):
        self.marks.append(id(w))
        self.written.add(id(w))
        if {id(v) for v in self.weights} <= set(self.marks):
            with torch.no_grad():
                for v in self.weights:
                    v.fill_(NAN)


def _case(node):
    """-> (weights, inputs(step) -> (args, dy), forward(*args, *weights))."""
    name, _, recipe = node.partition("-")
    g = torch.Generator().manual_seed(0)

    def r(*shape, scale=1.0, gen=g):
        return (torch.randn(*shape, generator=gen) * scale).to(BF16)

    T, H, I, E = 256, 64, 64, 2
    if name == "flat_linear":
        weights, x_shape, y_shape = [r(96, H, scale=H**-0.5)], (2, T // 2, H), (2, T // 2, 96)
        fwd = linear.flat_linear
    elif name == "fp8_linear":
        weights, x_shape, y_shape = [r(96, H, scale=H**-0.5)], (T, H), (T, 96)
        fwd = lambda x, w: linear.fp8_linear(x, w, recipe=recipe)
    elif name in ("swiglu_mlp", "fp8_swiglu_mlp"):
        weights, x_shape, y_shape = [r(2 * I, H, scale=H**-0.5), r(H, I, scale=I**-0.5)], (T, H), (T, H)
        fwd = linear.swiglu_mlp if name == "swiglu_mlp" else (lambda x, a, b: linear.fp8_swiglu_mlp(x, a, b, recipe))
    elif name == "grouped_swiglu_mlp":
        weights = [r(E, 2 * I, H, scale=H**-0.5), r(E, H, I, scale=I**-0.5)]
        x_shape = y_shape = (E, T // E, H)
        fwd = linear.grouped_swiglu_mlp
    else:
        weights, x_shape, y_shape = [r(E, 2 * I, H, scale=H**-0.5), r(E, H, I, scale=I**-0.5)], (T, H), (T, H)
        offsets = torch.tensor([0, 128, T], dtype=torch.int32)
        fwd = lambda x, w13, w2: linear.fp8_ragged_swiglu_mlp(x, offsets, w13, w2, recipe)

    def inputs(step):
        gs = torch.Generator().manual_seed(1 + step)
        return [r(*x_shape, gen=gs).requires_grad_(True)], r(*y_shape, gen=gs)

    return weights, inputs, fwd


def _run(node, view_dtype):
    """Two micro steps of ``node``, under a fake owner with ``view_dtype`` views (None: no owner) -> per step the input
    gradients, the weight gradients handed to autograd, the owner's views and marks; and the weights."""
    weights0, inputs, fwd = _case(node)
    weights = [w.clone().requires_grad_(True) for w in weights0]
    owner = _Owner(weights, view_dtype) if view_dtype is not None else None
    steps = []
    for step in range(2):
        with torch.no_grad():
            for w, w0 in zip(weights, weights0):
                w.copy_(w0)
        args, dy = inputs(step)
        y = fwd(*args, *weights)
        if owner is not None:
            owner.marks = []
        y.backward(dy)
        steps.append({
            "dx": [a.grad for a in args],
            "dw": [w.grad for w in weights],
            "views": [owner.views[id(w)].clone() for w in weights] if owner else None,
            "marks": list(owner.marks) if owner else None,
        })
        for w in weights:
            w.grad = None
    return steps, weights


@pytest.mark.parametrize("view_dtype", [BF16, torch.float32], ids=["bf16_view", "fp32_view"])
@pytest.mark.parametrize("node", NODES)
def test_weight_grad_routes_and_mark_order(node, view_dtype):
    ref, _ = _run(node, None)
    got, weights = _run(node, view_dtype)
    # the stacked bf16 experts' GEMM epilogues write only views of the product's dtype; anything else is returned
    returned = node == "grouped_swiglu_mlp" and view_dtype != BF16
    for s in range(2):
        for dw in ref[s]["dw"]:
            assert dw is not None and bool(torch.isfinite(dw).all()), "no owner: the gradient goes to autograd"
        for dx, want in zip(got[s]["dx"], ref[s]["dx"]):
            assert bool(torch.isfinite(dx).all()), f"step {s}: a weight was read after the node's last mark"
            assert torch.equal(dx, want)
        if returned:
            assert got[s]["marks"] == []
            for dw, want, view in zip(got[s]["dw"], ref[s]["dw"], got[s]["views"]):
                assert torch.equal(dw, want)
                assert bool(view.isnan().all()), "a returned gradient leaves the view alone"
            continue
        assert sorted(got[s]["marks"]) == sorted(id(w) for w in weights), "one mark per weight per backward"
        for i, (dw, view) in enumerate(zip(got[s]["dw"], got[s]["views"])):
            assert dw is None, "a gradient written into the view is not handed to autograd too"
            want = sum(ref[k]["dw"][i].float() for k in range(s + 1))
            mag = sum(ref[k]["dw"][i].float().abs() for k in range(s + 1))
            err = (view.float() - want).abs()
            what = "the first product" if s == 0 else "the sum of both"
            assert bool((err <= 2**-7 * mag).all()), f"step {s}, weight {i}: the view holds {what}"
