"""GPU tier: document-masked (varlen) wgmma attention over packed sequences, and Llama training on packed batches."""
import math

import numpy as np
import pytest
import torch

from tests.numerics import assert_attention_bounded

pytestmark = pytest.mark.gpu

d = 128
# offsets are not multiples of 128: the first document has 5 rows
RAGGED = [5, 1, 63, 64, 65, 0, 127, 128, 129, 200, 1000, 0]


def _cu(lens):
    return torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")


def _cols(x, hq, hkv):
    return x[:, :hq * d], x[:, hq * d:(hq + hkv) * d], x[:, (hq + hkv) * d:]


def _spans(lens):
    cu = np.concatenate([[0], np.cumsum(lens)]).tolist()
    return [(s, e) for s, e in zip(cu[:-1], cu[1:]) if e > s]


def _qkv(T, hq, hkv, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(T, (hq + 2 * hkv) * d, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _packed_lengths(seed, rows=2, row_len=4096, lo=16, hi=4096):
    """Document lengths drawn from [lo, hi] and cut to fill `rows` rows of `row_len` tokens."""
    rng = np.random.default_rng(seed)
    lens = []
    for _ in range(rows):
        left = row_len
        while left:
            n = min(int(rng.integers(lo, hi + 1)), left)
            lens.append(n)
            left -= n
    return lens


def _fwd_per_doc_bit_exact(lens, hq, hkv, causal, seed):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    T = sum(lens)
    qkv = _qkv(T, hq, hkv, seed)
    q, k, v = A.split_packed(qkv, hq, hkv)
    assert A.supports_varlen(qkv, hq, hkv, d)
    out = torch.full((T + 3, hq * d), 7.0, device="cuda", dtype=torch.bfloat16)
    _, lse = A.fwd_varlen(q, k, v, _cu(lens), max(lens), hq, hkv, causal=causal, out=out[:T])
    for s, e in _spans(lens):
        doc = qkv[s:e].clone()
        o1, l1 = A.fwd(*A.split_packed(doc, hq, hkv), 1, e - s, hq, hkv, causal=causal)
        assert torch.equal(out[s:e], o1), (s, e)
        assert torch.equal(lse[:, s:e], l1[0]), (s, e)
    assert float((out[T:].float() - 7.0).abs().max()) == 0.0  # rows past T are never written


@pytest.mark.parametrize("hq,hkv,causal", [(4, 2, True), (4, 2, False), (3, 1, True)])
def test_varlen_fwd_equals_dense_launch_per_document(hq, hkv, causal):
    _fwd_per_doc_bit_exact(RAGGED, hq, hkv, causal, seed=hq + causal)


def test_varlen_fwd_bit_exact_at_benchmark_shape():
    _fwd_per_doc_bit_exact(_packed_lengths(0), 24, 8, True, seed=0)


def _varlen_fwd_bwd(qkv, d_o, lens, hq, hkv, causal, max_seqlen=None):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    q, k, v = A.split_packed(qkv, hq, hkv)
    cu = _cu(lens)
    ms = max_seqlen or max(lens)
    o, lse = A.fwd_varlen(q, k, v, cu, ms, hq, hkv, causal=causal)
    dqkv = torch.full_like(qkv, float("nan"))
    dq, dk, dv = A.split_packed(dqkv, hq, hkv)
    A.bwd_varlen(d_o, q, k, v, o, lse, cu, ms, hq, hkv, causal=causal, dq=dq, dk=dk, dv=dv)
    return o, lse, dqkv


@pytest.mark.parametrize("causal", [True, False])
def test_varlen_bwd_equals_dense_launch_per_document(causal):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    hq, hkv = 4, 2
    lens = [5, 128, 256, 77, 384, 0, 128]
    T = sum(lens)
    qkv = _qkv(T, hq, hkv, 11, 0.7)
    d_o = _qkv(T, hq, 0, 12)
    o, _, dqkv = _varlen_fwd_bwd(qkv, d_o, lens, hq, hkv, causal)
    assert torch.isfinite(dqkv.float()).all()  # every gradient element written
    for s, e in _spans(lens):
        if (e - s) % 128:
            continue
        doc, ddo = qkv[s:e].clone(), d_o[s:e].clone()
        q1, k1, v1 = A.split_packed(doc, hq, hkv)
        o1, l1 = A.fwd(q1, k1, v1, 1, e - s, hq, hkv, causal=causal)
        assert torch.equal(o[s:e], o1)
        g1 = torch.empty_like(doc)
        A.bwd(ddo, q1, k1, v1, o1, l1, 1, e - s, hq, hkv, causal=causal, dq=g1[:, :hq * d], dk=g1[:, hq * d:(hq + hkv) * d], dv=g1[:, (hq + hkv) * d:])
        assert torch.equal(dqkv[s:e], g1), (s, e)


def test_uniform_lengths_equal_dense_batch():
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    B, S, hq, hkv = 3, 256, 4, 2
    qkv = _qkv(B * S, hq, hkv, 21, 0.7)
    d_o = _qkv(B * S, hq, 0, 22)
    o, lse, dqkv = _varlen_fwd_bwd(qkv, d_o, [S] * B, hq, hkv, True)
    q, k, v = A.split_packed(qkv, hq, hkv)
    o1, l1 = A.fwd(q, k, v, B, S, hq, hkv, causal=True)
    g1 = torch.empty_like(qkv)
    A.bwd(d_o, q, k, v, o1, l1, B, S, hq, hkv, causal=True, dq=g1[:, :hq * d], dk=g1[:, hq * d:(hq + hkv) * d],
          dv=g1[:, (hq + hkv) * d:])
    assert torch.equal(o, o1)
    assert torch.equal(lse, l1.permute(1, 0, 2).reshape(hq, B * S))
    assert torch.equal(dqkv, g1)


@pytest.mark.parametrize("hq,hkv", [(2, 2), (6, 2), (8, 2)])
@pytest.mark.parametrize("causal", [True, False])
def test_varlen_matches_float64_reference(hq, hkv, causal):
    lens = RAGGED
    T = sum(lens)
    qkv = _qkv(T, hq, hkv, 31 + hq, 0.7)
    d_o = _qkv(T, hq, 0, 32)
    o, lse, dqkv = _varlen_fwd_bwd(qkv, d_o, lens, hq, hkv, causal)
    assert torch.isfinite(dqkv.float()).all()
    o2, lse2, dqkv2 = _varlen_fwd_bwd(qkv, d_o, lens, hq, hkv, causal)
    assert torch.equal(o, o2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2)  # deterministic
    heads = lambda x, n: x.view(T, n, d)  # noqa: E731
    q, k, v = (heads(c, n) for c, n in zip(_cols(qkv, hq, hkv), (hq, hkv, hkv)))
    dq, dk, dv = (heads(c, n) for c, n in zip(_cols(dqkv, hq, hkv), (hq, hkv, hkv)))
    assert_attention_bounded({"o": heads(o, hq), "lse": lse, "dq": dq, "dk": dk, "dv": dv}, q, k, v,
                             heads(d_o, hq), np.concatenate([[0], np.cumsum(lens)]).tolist(), causal)


def test_documents_are_isolated():
    hq, hkv = 4, 2
    lens = RAGGED
    T = sum(lens)
    qkv = _qkv(T, hq, hkv, 41, 0.7)
    d_o = _qkv(T, hq, 0, 42)
    o, lse, dqkv = _varlen_fwd_bwd(qkv, d_o, lens, hq, hkv, True)
    spans = _spans(lens)
    for j in (0, 5, len(spans) - 1):
        s, e = spans[j]
        qkv2, d_o2 = qkv.clone(), d_o.clone()
        qkv2[s:e] = _qkv(e - s, hq, hkv, 43 + j, 0.7)
        d_o2[s:e] = _qkv(e - s, hq, 0, 44 + j)
        o2, lse2, dqkv2 = _varlen_fwd_bwd(qkv2, d_o2, lens, hq, hkv, True)
        keep = torch.ones(T, dtype=torch.bool, device="cuda")
        keep[s:e] = False
        assert torch.equal(o[keep], o2[keep]) and torch.equal(lse[:, keep], lse2[:, keep])
        assert torch.equal(dqkv[keep], dqkv2[keep])
        assert not torch.equal(o[s:e], o2[s:e])


def test_causal_attention_native_matches_per_document_cudnn():
    """Through the public op with in-place RoPE and per-document positions: native varlen kernel vs the per-document
    cuDNN loop."""
    from deepspeed_b200.ops.attention import causal_attention
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    hq, hkv = 4, 2
    lens = [100, 300, 28, 0, 84]
    B, S = 2, 256
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32)
    rope = RotaryTable(d, 512, 10000.0, "cuda")
    base = _qkv(B * S, hq, hkv, 51, 0.5)
    gy = _qkv(B * S, hq, 0, 52)
    outs = {}
    for backend in ("native", "cudnn"):
        qkv = base.clone().requires_grad_(True)
        y = causal_attention(qkv * 1.0, B, S, hq, hkv, d, rope, None, backend=backend, cu_seqlens=cu)
        y.backward(gy)
        outs[backend] = (y.detach().float(), qkv.grad.float())
    assert (outs["native"][0] - outs["cudnn"][0]).abs().max().item() < 3e-2
    ga, gb = outs["native"][1], outs["cudnn"][1]
    assert torch.isfinite(ga).all()
    assert torch.nn.functional.cosine_similarity(ga.flatten(), gb.flatten(), dim=0).item() > 0.999


def _train_packed(backend, steps=4):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=1024, num_hidden_layers=2, checkpoint_layers=1, attention_backend=backend)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    engine, _, _, _ = ds.initialize(model=model, config={
        "train_micro_batch_size_per_gpu": 2,
        "bf16": {"enabled": True},
        "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
        "zero_optimization": {"stage": 3},
    })
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (2, 384), device="cuda", generator=g)
    cu = torch.tensor([0, 100, 300, 384, 400, 768], dtype=torch.int32)
    losses = []
    for _ in range(steps):
        loss = engine(ids, labels=ids, cu_seqlens=cu)
        engine.backward(loss)
        engine.step()
        losses.append(float(loss.detach()))
    return losses


def _native_vs_fallback_training():
    native = _train_packed("native")
    cudnn = _train_packed("cudnn")
    assert all(math.isfinite(x) for x in native), native
    assert native[-1] < native[0], native
    for a, b in zip(native, cudnn):
        assert abs(a - b) < 2e-2 * abs(b) + 2e-2, (native, cudnn)


def test_llama_zero3_trains_on_packed_batches():
    """Native varlen kernel vs the per-document cuDNN loop under the ZeRO-3 bf16 engine, in a fresh process so no state
    left by earlier tests in the session reaches the engines."""
    from tests.common import run_distributed
    run_distributed(_native_vs_fallback_training, 1, ())
