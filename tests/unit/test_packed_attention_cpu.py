"""Packed-sequence (document-masked) attention and Llama training on packed batches, CPU tier, fp32.

Every packed result is compared with the same documents run on their own."""
import math

import pytest
import torch

from tests.common import run_distributed

D = 16


def _rope_ref(x, rope, pos):
    """Differentiable rotation of x [L, H, D] at positions pos [L] (same half-split convention as the kernels)."""
    half = rope.rot_dim // 2
    c, s = rope.cos[pos][:, None, :].to(x.dtype), rope.sin[pos][:, None, :].to(x.dtype)
    a, b = x[..., :half], x[..., half:2 * half]
    return torch.cat([a * c - b * s, b * c + a * s, x[..., 2 * half:]], dim=-1)


def _doc_ref(qkv, hq, hkv, rope, causal):
    """One document on its own: [L, (hq + 2 hkv) * D] -> [L, hq * D], float64, autograd-friendly."""
    L = qkv.shape[0]
    x = qkv.double().view(L, hq + 2 * hkv, D)
    q, k, v = x[:, :hq], x[:, hq:hq + hkv], x[:, hq + hkv:]
    if rope is not None:
        pos = torch.arange(L)
        q, k = _rope_ref(q, rope, pos), _rope_ref(k, rope, pos)
    rep = hq // hkv
    k, v = k.repeat_interleave(rep, 1), v.repeat_interleave(rep, 1)
    s = torch.einsum("qhd,khd->hqk", q, k) / math.sqrt(D)
    if causal:
        s = s.masked_fill(torch.triu(torch.ones(L, L, dtype=torch.bool), 1), float("-inf"))
    return torch.einsum("hqk,khd->qhd", torch.softmax(s, -1), v).reshape(L, hq * D)


LENS = [7, 0, 1, 64, 20, 0]


@pytest.mark.parametrize("use_rope", [False, True])
@pytest.mark.parametrize("hq,hkv", [(2, 2), (4, 2)])
@pytest.mark.parametrize("causal", [True, False])
def test_packed_matches_documents_alone(use_rope, hq, hkv, causal):
    from deepspeed_b200.ops.attention import causal_attention, varlen_attention_sdpa
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    torch.manual_seed(hq + 2 * use_rope + 4 * causal)
    T = sum(LENS)
    cu = torch.tensor([0] + list(torch.tensor(LENS).cumsum(0)), dtype=torch.int32)
    rope = RotaryTable(D, 128, 10000.0) if use_rope else None
    base = torch.randn(T, (hq + 2 * hkv) * D)
    leaf = base.clone().requires_grad_(True)
    if causal:
        out = causal_attention(leaf * 1.0, 1, T, hq, hkv, D, rope, cu_seqlens=cu)
    else:
        out = varlen_attention_sdpa(leaf * 1.0, cu, hq, hkv, D, rope, causal=False)
    gy = torch.randn_like(out)
    out.backward(gy)
    for s, e in zip(cu[:-1].tolist(), cu[1:].tolist()):
        if e == s:
            continue
        doc = base[s:e].clone().requires_grad_(True)
        ref = _doc_ref(doc, hq, hkv, rope, causal)
        ref.backward(gy[s:e].double())
        torch.testing.assert_close(out[s:e].double(), ref, atol=2e-6, rtol=1e-5)
        torch.testing.assert_close(leaf.grad[s:e].double(), doc.grad.double(), atol=5e-6, rtol=1e-5)


def test_packed_no_grad_matches_grad_mode():
    from deepspeed_b200.ops.attention import causal_attention
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    torch.manual_seed(0)
    T, hq, hkv = sum(LENS), 4, 2
    cu = torch.tensor([0] + list(torch.tensor(LENS).cumsum(0)), dtype=torch.int32)
    rope = RotaryTable(D, 128, 10000.0)
    base = torch.randn(T, (hq + 2 * hkv) * D)
    with torch.no_grad():
        a = causal_attention(base.clone(), 1, T, hq, hkv, D, rope, cu_seqlens=cu)
    b = causal_attention(base.clone().requires_grad_(True) * 1.0, 1, T, hq, hkv, D, rope, cu_seqlens=cu)
    assert torch.equal(a, b.detach())


def test_document_positions_restart_at_zero():
    from deepspeed_b200.ops.attention import document_positions
    cu = torch.tensor([0, 3, 3, 4, 9], dtype=torch.int32)
    pos = document_positions(cu, 9)
    assert pos.dtype == torch.int32
    assert pos.tolist() == [0, 1, 2, 0, 0, 1, 2, 3, 4]


@pytest.mark.parametrize("cu,why", [
    (torch.tensor([0, 4, 8], dtype=torch.int64), "int32"),
    (torch.tensor([1, 4, 8], dtype=torch.int32), "start at 0"),
    (torch.tensor([0, 4, 7], dtype=torch.int32), "end at"),
    (torch.tensor([0, 5, 4, 8], dtype=torch.int32), "non-decreasing"),
    (torch.tensor([[0, 8]], dtype=torch.int32), "1-D"),
])
def test_malformed_cu_seqlens_raise(cu, why):
    from deepspeed_b200.ops.attention import causal_attention
    qkv = torch.randn(8, 4 * D)
    with pytest.raises(ValueError, match=why):
        causal_attention(qkv, 2, 4, 2, 1, D, cu_seqlens=cu)


def _tiny(**kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", vocab_size=97, hidden_size=64, intermediate_size=128, num_attention_heads=4,
                       num_key_value_heads=2, loss_chunk_tokens=8, **kw)
    return LlamaForCausalLM(cfg)


def test_model_rejects_document_crossing_rows():
    model = _tiny()
    ids = torch.randint(0, 97, (2, 8))
    with pytest.raises(ValueError, match="row start"):
        model(ids, labels=ids, cu_seqlens=torch.tensor([0, 5, 16], dtype=torch.int32))


def test_cross_document_target_is_ignored():
    """Shifted labels with packing equal the unshifted call with every document's last target set to -100."""
    model = _tiny()
    ids = torch.randint(0, 97, (2, 8), generator=torch.Generator().manual_seed(3))
    cu = torch.tensor([0, 5, 8, 16], dtype=torch.int32)
    got = model(ids, labels=ids, cu_seqlens=cu)
    labels = torch.cat([ids[:, 1:], torch.full_like(ids[:, :1], -100)], dim=1).reshape(-1).clone()
    labels[[4, 7, 15]] = -100
    want = model(ids, labels=labels.view(2, 8), shift_labels=False, cu_seqlens=cu)
    assert torch.equal(got, want)
    # without the document mask on the targets, the loss would differ
    unmasked = torch.cat([ids[:, 1:], torch.full_like(ids[:, :1], -100)], dim=1)
    assert not torch.equal(got, model(ids, labels=unmasked, shift_labels=False, cu_seqlens=cu))


@pytest.mark.parametrize("checkpoint_layers", [0, 1])
def test_llama_packed_batch_matches_documents_alone(checkpoint_layers):
    """3 documents in 2 rows: loss and every parameter gradient equal the documents run one at a time, their losses
    combined with their valid-token weights."""
    model = _tiny(checkpoint_layers=checkpoint_layers)
    model.train()
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 97, (2, 12), generator=g)
    cu = torch.tensor([0, 7, 12, 24], dtype=torch.int32)
    loss = model(ids, labels=ids, cu_seqlens=cu)
    loss.backward()
    packed = {n: p.grad.clone() for n, p in model.named_parameters()}
    model.zero_grad()
    flat = ids.reshape(-1)
    docs = [flat[s:e] for s, e in zip(cu[:-1].tolist(), cu[1:].tolist())]
    n_valid = [len(d) - 1 for d in docs]
    total = 0.0
    for d, n in zip(docs, n_valid):
        total = total + model(d[None], labels=d[None]) * (n / sum(n_valid))
    total.backward()
    torch.testing.assert_close(loss, total, atol=1e-6, rtol=1e-6)
    for n, p in model.named_parameters():
        torch.testing.assert_close(packed[n], p.grad, atol=1e-6, rtol=1e-4, msg=n)


def test_llama_default_positions_are_per_document(monkeypatch):
    """RoPE is shift-invariant inside a document, so the loss cannot tell; look at the positions the rotation gets."""
    import deepspeed_b200.ops.attention as A
    seen = []
    real = A.rope_qk_inplace

    def spy(qkv, hq, hkv, d, rope, positions, *a, **kw):
        seen.append(positions.clone())
        return real(qkv, hq, hkv, d, rope, positions, *a, **kw)

    monkeypatch.setattr(A, "rope_qk_inplace", spy)
    model = _tiny()
    ids = torch.randint(0, 97, (2, 12), generator=torch.Generator().manual_seed(2))
    cu = torch.tensor([0, 7, 12, 24], dtype=torch.int32)
    model(ids, labels=ids, cu_seqlens=cu)
    want = list(range(7)) + list(range(5)) + list(range(12))
    assert len(seen) == model.cfg.num_hidden_layers
    assert all(p.tolist() == want for p in seen)


def _engine_passes_packing():
    import deepspeed_b200 as ds
    model = _tiny()
    ids = torch.randint(0, 97, (2, 12), generator=torch.Generator().manual_seed(4))
    cu = torch.tensor([0, 7, 12, 24], dtype=torch.int32)
    with torch.no_grad():
        want = model(ids, labels=ids, cu_seqlens=cu)
        unpacked = model(ids, labels=ids)
    cfg = {"train_micro_batch_size_per_gpu": 2, "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
           "zero_optimization": {"stage": 0}}
    eng, _, _, _ = ds.initialize(model=model, config=cfg)
    got = eng(ids, labels=ids, cu_seqlens=cu)
    assert torch.equal(got.detach(), want) and not torch.equal(want, unpacked)
    eng.backward(got)
    eng.step()
    # fp16 input auto-casting touches floating tensors only: the int32 offsets pass through as they are
    cfg16 = dict(cfg, fp16={"enabled": True, "auto_cast": True})
    eng16, _, _, _ = ds.initialize(model=_tiny(), config=cfg16)
    args, kw = eng16._cast_inputs((ids, ), {"cu_seqlens": cu, "x": torch.zeros(2)})
    assert kw["cu_seqlens"] is cu and args[0] is ids and kw["x"].dtype == torch.float16


def test_engine_forwards_packing_kwargs():
    run_distributed(_engine_passes_packing, 1, ())
