"""GPU tier: causal sliding-window wgmma attention (row i sees keys i - W < j <= i), dense and packed, and Llama training
with a window."""
import math

import numpy as np
import pytest
import torch

from tests.numerics import assert_attention_bounded

pytestmark = pytest.mark.gpu

d = 128
# offsets are not multiples of 128: the first document has 5 rows
RAGGED = [5, 1, 63, 64, 65, 0, 127, 128, 129, 200, 1000, 0]
# windows on both sides of the 64-key and 128-row tile edges
SHAPES = [(1, 256, 2, 1, 1), (1, 512, 4, 2, 64), (2, 512, 4, 2, 65), (1, 1024, 8, 2, 127), (1, 1024, 4, 4, 128),
          (1, 2048, 6, 2, 129), (1, 2048, 3, 1, 1000)]


def _cu(lens):
    return torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")


def _spans(lens):
    cu = np.concatenate([[0], np.cumsum(lens)]).tolist()
    return [(s, e) for s, e in zip(cu[:-1], cu[1:]) if e > s]


def _qkv(T, hq, hkv, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(T, (hq + 2 * hkv) * d, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _cols(x, hq, hkv):
    return x[:, :hq * d], x[:, hq * d:(hq + hkv) * d], x[:, (hq + hkv) * d:]


def _dense_fwd_bwd(qkv, d_o, B, S, hq, hkv, window):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    q, k, v = A.split_packed(qkv, hq, hkv)
    o, lse = A.fwd(q, k, v, B, S, hq, hkv, causal=True, window=window)
    dqkv = torch.full_like(qkv, float("nan"))
    dq, dk, dv = _cols(dqkv, hq, hkv)
    A.bwd(d_o, q, k, v, o, lse, B, S, hq, hkv, causal=True, dq=dq, dk=dk, dv=dv, window=window)
    return o, lse, dqkv


def _varlen_fwd_bwd(qkv, d_o, lens, hq, hkv, window):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    q, k, v = A.split_packed(qkv, hq, hkv)
    cu = _cu(lens)
    o, lse = A.fwd_varlen(q, k, v, cu, max(lens), hq, hkv, causal=True, window=window)
    dqkv = torch.full_like(qkv, float("nan"))
    dq, dk, dv = _cols(dqkv, hq, hkv)
    A.bwd_varlen(d_o, q, k, v, o, lse, cu, max(lens), hq, hkv, causal=True, dq=dq, dk=dk, dv=dv, window=window)
    return o, lse, dqkv


@pytest.mark.parametrize("B,S,hq,hkv,W", SHAPES)
def test_window_matches_float64_reference(B, S, hq, hkv, W):
    qkv = _qkv(B * S, hq, hkv, 31 + hq + W, 0.7)
    d_o = _qkv(B * S, hq, 0, 32 + W)
    o, lse, dqkv = _dense_fwd_bwd(qkv, d_o, B, S, hq, hkv, W)
    assert torch.isfinite(dqkv.float()).all()  # every gradient element written
    o2, lse2, dqkv2 = _dense_fwd_bwd(qkv, d_o, B, S, hq, hkv, W)
    assert torch.equal(o, o2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2)  # deterministic
    T = B * S
    heads = lambda x, n: x.view(T, n, d)  # noqa: E731
    q, k, v = (heads(c, n) for c, n in zip(_cols(qkv, hq, hkv), (hq, hkv, hkv)))
    dq, dk, dv = (heads(c, n) for c, n in zip(_cols(dqkv, hq, hkv), (hq, hkv, hkv)))
    assert_attention_bounded({"o": heads(o, hq), "lse": lse.permute(1, 0, 2).reshape(hq, T), "dq": dq, "dk": dk,
                              "dv": dv}, q, k, v, heads(d_o, hq), [b * S for b in range(B + 1)], True, W)


@pytest.mark.parametrize("B,S", [(1, 384), (2, 512)])
def test_window_covering_sequence_equals_unwindowed_kernel(B, S):
    hq, hkv = 4, 2
    qkv = _qkv(B * S, hq, hkv, 7, 0.7)
    d_o = _qkv(B * S, hq, 0, 8)
    base = _dense_fwd_bwd(qkv, d_o, B, S, hq, hkv, None)
    for W in (S, S + 1, 10 * S):
        got = _dense_fwd_bwd(qkv, d_o, B, S, hq, hkv, W)
        assert all(torch.equal(a, b) for a, b in zip(base, got)), W


@pytest.mark.parametrize("W", [1, 64, 65, 200])
def test_packed_fwd_equals_dense_windowed_launch_per_document(W):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    hq, hkv = 4, 2
    T = sum(RAGGED)
    qkv = _qkv(T, hq, hkv, W)
    q, k, v = A.split_packed(qkv, hq, hkv)
    out = torch.full((T + 3, hq * d), 7.0, device="cuda", dtype=torch.bfloat16)
    _, lse = A.fwd_varlen(q, k, v, _cu(RAGGED), max(RAGGED), hq, hkv, causal=True, out=out[:T], window=W)
    for s, e in _spans(RAGGED):
        doc = qkv[s:e].clone()
        o1, l1 = A.fwd(*A.split_packed(doc, hq, hkv), 1, e - s, hq, hkv, causal=True, window=W)
        assert torch.equal(out[s:e], o1), (s, e)
        assert torch.equal(lse[:, s:e], l1[0]), (s, e)
    assert float((out[T:].float() - 7.0).abs().max()) == 0.0  # rows past T are never written


@pytest.mark.parametrize("W", [1, 100, 129])
def test_packed_bwd_equals_dense_windowed_launch_per_document(W):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    hq, hkv = 4, 2
    lens = [5, 128, 256, 77, 384, 0, 128]
    T = sum(lens)
    qkv = _qkv(T, hq, hkv, 11 + W, 0.7)
    d_o = _qkv(T, hq, 0, 12 + W)
    o, _, dqkv = _varlen_fwd_bwd(qkv, d_o, lens, hq, hkv, W)
    assert torch.isfinite(dqkv.float()).all()
    for s, e in _spans(lens):
        if (e - s) % 128:
            continue
        o1, _, g1 = _dense_fwd_bwd(qkv[s:e].clone(), d_o[s:e].clone(), 1, e - s, hq, hkv, W)
        assert torch.equal(o[s:e], o1)
        assert torch.equal(dqkv[s:e], g1), (s, e)


@pytest.mark.parametrize("B,S,W,P", [(1, 1024, 64, 128), (2, 512, 129, 200), (1, 1024, 300, 77)])
def test_keys_before_the_window_are_masked(B, S, W, P):
    """K / V rows [0, P) of every sequence get large finite values: rows >= P + W - 1 of O, LSE, dQ, dK and dV do not
    change by a bit."""
    hq, hkv = 4, 2
    qkv = _qkv(B * S, hq, hkv, 61, 0.7)
    d_o = _qkv(B * S, hq, 0, 62)
    base = _dense_fwd_bwd(qkv, d_o, B, S, hq, hkv, W)
    pert = qkv.clone()
    for b in range(B):
        _, k, v = _cols(pert[b * S:b * S + P], hq, hkv)
        k.fill_(12.0)
        v.fill_(3000.0)
    got = _dense_fwd_bwd(pert, d_o, B, S, hq, hkv, W)
    keep = (torch.arange(B * S, device="cuda") % S) >= P + W - 1
    o, lse, g = base
    o2, lse2, g2 = got
    assert torch.equal(o[keep], o2[keep])
    assert torch.equal(lse.permute(1, 0, 2).reshape(hq, B * S)[:, keep], lse2.permute(1, 0, 2).reshape(hq, B * S)[:, keep])
    assert torch.equal(g[keep], g2[keep])
    assert not torch.equal(o[~keep], o2[~keep])  # the perturbation is visible where the window reaches it
    assert torch.isfinite(o2.float()).all() and torch.isfinite(g2.float()).all()


def _public_op(backend, packed, W, rope, base, gy, B, S, hq, hkv, cu):
    from deepspeed_b200.ops.attention import causal_attention
    qkv = base.clone().requires_grad_(True)
    kw = dict(cu_seqlens=cu) if packed else {}
    y = causal_attention(qkv * 1.0, B, S, hq, hkv, d, rope, None, backend=backend, sliding_window=W, **kw)
    y.backward(gy)
    return y.detach().float(), qkv.grad.float()


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("W", [1, 96, 200])
def test_public_op_native_matches_masked_sdpa(packed, W):
    """Through the public op with in-place RoPE: the native windowed kernel against the masked-SDPA fallback."""
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    hq, hkv = 4, 2
    B, S = 2, 256
    cu = torch.tensor(np.concatenate([[0], np.cumsum([100, 300, 28, 0, 84])]), dtype=torch.int32)
    rope = RotaryTable(d, 512, 10000.0, "cuda")
    base = _qkv(B * S, hq, hkv, 51 + W, 0.5)
    gy = _qkv(B * S, hq, 0, 52)
    ya, ga = _public_op("native", packed, W, rope, base, gy, B, S, hq, hkv, cu)
    yb, gb = _public_op("cudnn", packed, W, rope, base, gy, B, S, hq, hkv, cu)
    assert (ya - yb).abs().max().item() < 3e-2
    assert torch.isfinite(ga).all()
    assert torch.nn.functional.cosine_similarity(ga.flatten(), gb.flatten(), dim=0).item() > 0.999


def test_llama_receptive_field_native():
    """bf16 tiny Llama (head dim 128) on the native kernel: token 0 reaches positions up to L (W - 1) and no further."""
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    W = 4
    cfg = llama_config("tiny", hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=1024, num_hidden_layers=2, attention_backend="native", sliding_window=W)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    ids = torch.randint(1, cfg.vocab_size, (1, 256), device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    ids2 = ids.clone()
    ids2[0, 0] = 0
    with torch.no_grad():
        a, b = model(ids), model(ids2)
    edge = cfg.num_hidden_layers * (W - 1)
    assert torch.equal(a[:, edge + 1:], b[:, edge + 1:])
    assert not torch.equal(a[:, edge], b[:, edge])


def _train_windowed(backend, steps=4):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=1024, num_hidden_layers=2, checkpoint_layers=1, attention_backend=backend,
                       max_position_embeddings=1024, sliding_window=256)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    engine, _, _, _ = ds.initialize(model=model, config={
        "train_micro_batch_size_per_gpu": 2,
        "bf16": {"enabled": True},
        "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
        "zero_optimization": {"stage": 3},
    })
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (2, 1024), device="cuda", generator=g)
    losses = []
    for _ in range(steps):
        loss = engine(ids, labels=ids)
        engine.backward(loss)
        engine.step()
        losses.append(float(loss.detach()))
    return losses


def _native_vs_fallback_training():
    native = _train_windowed("native")
    sdpa = _train_windowed("cudnn")
    assert all(math.isfinite(x) for x in native), native
    assert native[-1] < native[0], native
    for a, b in zip(native, sdpa):
        assert abs(a - b) < 2e-2 * abs(b) + 2e-2, (native, sdpa)


def test_llama_zero3_trains_with_sliding_window():
    """Native windowed kernel against the masked-SDPA fallback under the ZeRO-3 bf16 engine, in a fresh process so no
    state left by earlier tests in the session reaches the engines."""
    from tests.common import run_distributed
    run_distributed(_native_vs_fallback_training, 1, ())
