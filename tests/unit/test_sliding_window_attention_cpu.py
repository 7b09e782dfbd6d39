"""Causal sliding-window attention (``sliding_window=W``: row i sees keys i - W < j <= i) and Llama training with a window,
CPU tier, fp32 against a float64 band-mask reference."""
import math

import pytest
import torch

from tests.common import run_distributed

D = 16
LENS = [7, 0, 1, 64, 20, 0]
WINDOWS = [1, 5, 16, 66, 67, 200]


def _rope_ref(x, rope, pos):
    """Differentiable rotation of x [L, H, D] at positions pos [L] (same half-split convention as the kernels)."""
    half = rope.rot_dim // 2
    c, s = rope.cos[pos][:, None, :].to(x.dtype), rope.sin[pos][:, None, :].to(x.dtype)
    a, b = x[..., :half], x[..., half:2 * half]
    return torch.cat([a * c - b * s, b * c + a * s, x[..., 2 * half:]], dim=-1)


def _band_ref(qkv, hq, hkv, rope, window):
    """One sequence: [L, (hq + 2 hkv) * D] -> [L, hq * D], float64, row i attending to keys i - window < j <= i."""
    L = qkv.shape[0]
    x = qkv.double().view(L, hq + 2 * hkv, D)
    q, k, v = x[:, :hq], x[:, hq:hq + hkv], x[:, hq + hkv:]
    if rope is not None:
        pos = torch.arange(L)
        q, k = _rope_ref(q, rope, pos), _rope_ref(k, rope, pos)
    rep = hq // hkv
    k, v = k.repeat_interleave(rep, 1), v.repeat_interleave(rep, 1)
    s = torch.einsum("qhd,khd->hqk", q, k) / math.sqrt(D)
    i = torch.arange(L)
    diff = i[:, None] - i[None, :]
    s = s.masked_fill(~((diff >= 0) & (diff < window)), float("-inf"))
    return torch.einsum("hqk,khd->qhd", torch.softmax(s, -1), v).reshape(L, hq * D)


def _cu(lens):
    return torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("use_rope", [False, True])
@pytest.mark.parametrize("hq,hkv", [(2, 2), (4, 2)])
def test_dense_matches_band_reference(window, use_rope, hq, hkv):
    from deepspeed_b200.ops.attention import causal_attention
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    torch.manual_seed(window + hq + 7 * use_rope)
    B, S = 2, 67
    rope = RotaryTable(D, 128, 10000.0) if use_rope else None
    base = torch.randn(B * S, (hq + 2 * hkv) * D)
    leaf = base.clone().requires_grad_(True)
    out = causal_attention(leaf * 1.0, B, S, hq, hkv, D, rope, sliding_window=window)
    gy = torch.randn_like(out)
    out.backward(gy)
    for b in range(B):
        rows = slice(b * S, (b + 1) * S)
        seq = base[rows].clone().requires_grad_(True)
        ref = _band_ref(seq, hq, hkv, rope, window)
        ref.backward(gy[rows].double())
        torch.testing.assert_close(out[rows].double(), ref, atol=2e-6, rtol=1e-5)
        torch.testing.assert_close(leaf.grad[rows].double(), seq.grad.double(), atol=5e-6, rtol=1e-5)


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("use_rope", [False, True])
@pytest.mark.parametrize("hq,hkv", [(2, 2), (4, 2)])
def test_packed_matches_band_reference_per_document(window, use_rope, hq, hkv):
    """The window is measured inside each document."""
    from deepspeed_b200.ops.attention import causal_attention
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    torch.manual_seed(window + hq + 7 * use_rope)
    T = sum(LENS)
    cu = _cu(LENS)
    rope = RotaryTable(D, 128, 10000.0) if use_rope else None
    base = torch.randn(T, (hq + 2 * hkv) * D)
    leaf = base.clone().requires_grad_(True)
    out = causal_attention(leaf * 1.0, 1, T, hq, hkv, D, rope, cu_seqlens=cu, sliding_window=window)
    gy = torch.randn_like(out)
    out.backward(gy)
    for s, e in zip(cu[:-1].tolist(), cu[1:].tolist()):
        if e == s:
            continue
        doc = base[s:e].clone().requires_grad_(True)
        ref = _band_ref(doc, hq, hkv, rope, window)
        ref.backward(gy[s:e].double())
        torch.testing.assert_close(out[s:e].double(), ref, atol=2e-6, rtol=1e-5)
        torch.testing.assert_close(leaf.grad[s:e].double(), doc.grad.double(), atol=5e-6, rtol=1e-5)


@pytest.mark.parametrize("packed", [False, True])
def test_window_one_returns_own_value(packed):
    """W = 1: every query sees only its own key, so the output is the value row of its KV head."""
    from deepspeed_b200.ops.attention import causal_attention
    torch.manual_seed(3)
    hq, hkv = 4, 2
    T = sum(LENS)
    qkv = torch.randn(T, (hq + 2 * hkv) * D)
    kw = dict(cu_seqlens=_cu(LENS)) if packed else {}
    B, S = (1, T) if packed else (2, T // 2)
    out = causal_attention(qkv.clone(), B, S, hq, hkv, D, sliding_window=1, **kw)
    v = qkv.view(T, hq + 2 * hkv, D)[:, hq + hkv:]
    want = v.repeat_interleave(hq // hkv, 1).reshape(T, hq * D)
    assert torch.equal(out, want)


@pytest.mark.parametrize("packed,window", [(False, 46), (False, 1000), (True, 64), (True, 1000)])
def test_window_covering_everything_is_bit_equal_to_none(packed, window):
    from deepspeed_b200.ops.attention import causal_attention
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    torch.manual_seed(5)
    hq, hkv = 4, 2
    T = sum(LENS)  # 92 = 2 x 46
    rope = RotaryTable(D, 128, 10000.0)
    base = torch.randn(T, (hq + 2 * hkv) * D)
    gy = torch.randn(T, hq * D)
    kw = dict(cu_seqlens=_cu(LENS)) if packed else {}
    B, S = (1, T) if packed else (2, T // 2)
    res = []
    for w in (None, window):
        leaf = base.clone().requires_grad_(True)
        out = causal_attention(leaf * 1.0, B, S, hq, hkv, D, rope, sliding_window=w, **kw)
        out.backward(gy)
        res.append((out.detach(), leaf.grad))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


@pytest.mark.parametrize("window", [0, -1, 2.5, True, "8"])
def test_invalid_window_raises(window):
    from deepspeed_b200.ops.attention import causal_attention
    qkv = torch.randn(8, 4 * D)
    with pytest.raises(ValueError, match="sliding_window"):
        causal_attention(qkv, 2, 4, 2, 1, D, sliding_window=window)
    with pytest.raises(ValueError, match="sliding_window"):
        causal_attention(qkv, 2, 4, 2, 1, D, cu_seqlens=torch.tensor([0, 4, 8], dtype=torch.int32), sliding_window=window)


def test_non_causal_window_raises():
    from deepspeed_b200.ops.attention import varlen_attention_sdpa
    from deepspeed_b200.ops.kernels import attention_sm100
    qkv = torch.randn(8, 4 * D)
    with pytest.raises(ValueError, match="causal"):
        varlen_attention_sdpa(qkv, torch.tensor([0, 8], dtype=torch.int32), 2, 1, D, causal=False, sliding_window=4)
    with pytest.raises(ValueError, match="causal"):
        attention_sm100._window(4, causal=False)
    assert attention_sm100._window(None, causal=False) == 0


def _tiny(**kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", vocab_size=97, hidden_size=64, intermediate_size=128, num_attention_heads=4,
                       num_key_value_heads=2, loss_chunk_tokens=8, **kw)
    return LlamaForCausalLM(cfg)


def test_llama_receptive_field():
    """Each layer reaches W - 1 tokens further back: with L layers, token 0 reaches positions up to L (W - 1) and no
    further."""
    W = 8
    model = _tiny(sliding_window=W)
    L = model.cfg.num_hidden_layers
    ids = torch.randint(1, 97, (1, 40), generator=torch.Generator().manual_seed(1))
    ids2 = ids.clone()
    ids2[0, 0] = 0
    with torch.no_grad():
        a, b = model(ids), model(ids2)
    edge = L * (W - 1)
    assert torch.equal(a[:, edge + 1:], b[:, edge + 1:])
    assert not torch.equal(a[:, edge], b[:, edge])
    full = _tiny()  # without a window token 0 reaches every position
    with torch.no_grad():
        assert not torch.equal(full(ids)[:, -1], full(ids2)[:, -1])


def test_flops_per_token_counts_visible_pairs():
    from deepspeed_b200.models.llama import llama_config
    base = llama_config("mistral-7b", sliding_window=None)
    for S in (1024, 4096):
        assert llama_config("mistral-7b").flops_per_token(S) == base.flops_per_token(S)
    S, W = 8192, 4096
    cfg = llama_config("mistral-7b")
    pairs = sum(min(i + 1, W) for i in range(S))
    mm = base.flops_per_token(S) - 3 * 4 * S * base.q_size * base.num_hidden_layers * 0.5
    assert math.isclose(cfg.flops_per_token(S), mm + 3 * 4 * (pairs / S) * cfg.q_size * cfg.num_hidden_layers)
    assert cfg.flops_per_token(S) < base.flops_per_token(S)


def test_mistral_preset_has_its_window():
    from deepspeed_b200.models.llama import llama_config
    cfg = llama_config("mistral-7b")
    assert (cfg.sliding_window, cfg.rope_theta, cfg.vocab_size) == (4096, 10000.0, 32000)
    assert llama_config("llama3-8b").sliding_window is None


def test_llama_window_with_activation_checkpointing():
    """Recompute with a window gives the same loss and gradients as the plain run; the window changes the loss."""
    ids = torch.randint(0, 97, (2, 24), generator=torch.Generator().manual_seed(2))
    grads, losses = [], []
    for ckpt in (0, 2):
        model = _tiny(sliding_window=5, checkpoint_layers=ckpt)
        model.train()
        loss = model(ids, labels=ids)
        loss.backward()
        losses.append(loss.detach())
        grads.append({n: p.grad.clone() for n, p in model.named_parameters()})
    assert torch.equal(losses[0], losses[1])
    for n in grads[0]:
        torch.testing.assert_close(grads[0][n], grads[1][n], atol=0, rtol=0, msg=n)
    with torch.no_grad():
        assert not torch.equal(losses[0], _tiny()(ids, labels=ids))


def _engine_passes_window():
    import deepspeed_b200 as ds
    model = _tiny(sliding_window=5, checkpoint_layers=1)
    ids = torch.randint(0, 97, (2, 24), generator=torch.Generator().manual_seed(4))
    cu = torch.tensor([0, 7, 24, 48], dtype=torch.int32)
    with torch.no_grad():
        want = model(ids, labels=ids)
        unwindowed = _tiny()(ids, labels=ids)
    cfg = {"train_micro_batch_size_per_gpu": 2, "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
           "zero_optimization": {"stage": 0}}
    eng, _, _, _ = ds.initialize(model=model, config=cfg)
    eng.train()
    got = eng(ids, labels=ids)
    assert torch.equal(got.detach(), want) and not torch.equal(want, unwindowed)
    eng.backward(got)
    eng.step()
    got_packed = eng(ids, labels=ids, cu_seqlens=cu)  # packed documents with a window, through the checkpointed layer
    assert torch.isfinite(got_packed)
    eng.backward(got_packed)
    eng.step()


def test_engine_trains_windowed_model_with_checkpointing():
    run_distributed(_engine_passes_window, 1, ())
