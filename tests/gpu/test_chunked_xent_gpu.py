"""``chunked_linear_xent`` at the Llama-3.2-3B LM head (H 3072, V 128256) against float64 cross entropy of ``h @ W.T``.

The loss, ``dh`` and ``dW`` are produced chunk by chunk inside the forward: logits GEMM, fused softmax-xent kernel with the
device scalar 1/n as gradient scale, ``dh`` GEMM, and ``dW`` accumulated across chunks in the GEMM epilogue; the backward
rescales by ``dloss / assumed_scale``.  Both GEMM backends run: ``own`` forces the in-tree NN and TN kernels (with the
accumulate epilogue) at V = 128256.  Bounds are per element, from ``tests/numerics.py``.
"""
import functools

import pytest
import torch

from tests.numerics import assert_within, chunked_xent_reference

pytestmark = pytest.mark.gpu

H, V, CHUNK, IGNORE = 3072, 128256, 2048, -100


def _inputs(T):
    g = torch.Generator(device="cuda").manual_seed(T)
    h = torch.randn(T, H, generator=g, device="cuda").bfloat16()
    w = (torch.randn(V, H, generator=g, device="cuda") * 0.05).bfloat16()  # logits ~ N(0, 2.8^2)
    labels = torch.randint(0, V, (T, ), generator=g, device="cuda")
    labels[torch.rand(T, generator=g, device="cuda") < 0.1] = IGNORE
    if T >= 3 * CHUNK:
        labels[CHUNK:2 * CHUNK] = IGNORE  # a chunk without a single counted token
    return h, w, labels


@functools.lru_cache(maxsize=1)
def _reference(T):
    h, w, labels = _inputs(T)
    return chunked_xent_reference(h, w, labels, CHUNK, IGNORE)


@pytest.fixture(scope="module", autouse=True)
def _release_reference():
    yield
    _reference.cache_clear()  # ~6 GB of float64 dW reference and bound at T = 8192


@pytest.fixture
def gemm_backend():
    from deepspeed_b200.ops import gemm
    before, used = gemm.get_backend(), dict(gemm._used)
    yield gemm.set_backend
    gemm.set_backend(before)
    gemm._used.clear()  # forced choices must not stand in for the shipped table in later tests
    gemm._used.update(used)


# ordered by T so that each float64 reference is computed once
CASES = [(T, backend, scale) for T in (2048, 5000, 8192) for backend in ("own", "lib") for scale in (1.0, 1024.0)]


@pytest.mark.parametrize("T,backend,scale", CASES)
def test_chunked_linear_xent(T, backend, scale, gemm_backend):
    from deepspeed_b200.ops.linear import chunked_linear_xent
    gemm_backend(backend)
    h, w, labels = _inputs(T)
    loss_ref, dh_ref, dw_ref, loss_bound, dh_bound, dw_bound = _reference(T)
    with torch.no_grad():
        loss_ng = chunked_linear_xent(h, w, labels, chunk=CHUNK, ignore_index=IGNORE)
    hp = h.clone().requires_grad_(True)
    wp = w.clone().requires_grad_(True)
    loss = chunked_linear_xent(hp, wp, labels, chunk=CHUNK, ignore_index=IGNORE, assumed_scale=scale)
    # the engine's convention: the backward sees dloss = loss scale x the user's factor (0.5 here), and the gradients
    # come out at that scale; 0.5 * scale is a power of two, so the rescale adds no rounding
    (loss * (0.5 * scale)).backward()
    assert torch.equal(loss_ng, loss.detach()), "the no-grad loss differs from the grad-mode loss"
    assert_within(loss.detach().cpu().reshape(1), torch.tensor([loss_ref]), loss_bound, "loss")
    f = 0.5 * scale
    assert_within(hp.grad, dh_ref * f, dh_bound * f, "dh")
    if T >= 3 * CHUNK:
        assert bool((hp.grad[CHUNK:2 * CHUNK] == 0).all())
    assert_within(wp.grad, dw_ref * f, dw_bound * f, "dW")
