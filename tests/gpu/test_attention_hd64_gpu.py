"""GPU tier: head dim 64 in the wgmma training attention -- dense, packed (varlen) and sliding-window kernels against
float64 references and against the head-dim-128 kernels on zero-padded heads, the public op and its routing, and a
head-dim-64 Llama under the ZeRO-3 engine."""
import math

import numpy as np
import pytest
import torch

from tests.numerics import assert_attention_bounded

pytestmark = pytest.mark.gpu

d = 64
# offsets are not multiples of 128: the first document has 5 rows
RAGGED = [5, 1, 63, 64, 65, 0, 127, 128, 129, 200, 1000, 0]
# windows on both sides of the 64-key and 128-row tile edges
SHAPES = [(1, 256, 2, 1, 1), (1, 512, 4, 2, 64), (2, 512, 4, 2, 65), (1, 1024, 8, 2, 127), (1, 1024, 4, 4, 128),
          (1, 2048, 6, 2, 129), (1, 2048, 3, 1, 1000)]


def _A():
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    return A


def _cu(lens):
    return torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")


def _spans(lens):
    cu = np.concatenate([[0], np.cumsum(lens)]).tolist()
    return [(s, e) for s, e in zip(cu[:-1], cu[1:]) if e > s]


def _qkv(T, hq, hkv, seed, scale=1.0, hd=d):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(T, (hq + 2 * hkv) * hd, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _cols(x, hq, hkv, hd=d):
    return x[:, :hq * hd], x[:, hq * hd:(hq + hkv) * hd], x[:, (hq + hkv) * hd:]


def _dense(qkv, d_o, B, S, hq, hkv, causal=True, window=None, hd=d, scale=None):
    A = _A()
    q, k, v = _cols(qkv, hq, hkv, hd)
    o, lse = A.fwd(q, k, v, B, S, hq, hkv, causal=causal, window=window, head_dim=hd, scale=scale)
    dqkv = torch.full_like(qkv, float("nan"))
    dq, dk, dv = _cols(dqkv, hq, hkv, hd)
    A.bwd(d_o, q, k, v, o, lse, B, S, hq, hkv, causal=causal, dq=dq, dk=dk, dv=dv, window=window, head_dim=hd,
          scale=scale)
    return o, lse, dqkv


def _varlen(qkv, d_o, lens, hq, hkv, causal=True, window=None, hd=d, scale=None):
    A = _A()
    q, k, v = _cols(qkv, hq, hkv, hd)
    cu = _cu(lens)
    o, lse = A.fwd_varlen(q, k, v, cu, max(lens), hq, hkv, causal=causal, window=window, head_dim=hd, scale=scale)
    dqkv = torch.full_like(qkv, float("nan"))
    dq, dk, dv = _cols(dqkv, hq, hkv, hd)
    A.bwd_varlen(d_o, q, k, v, o, lse, cu, max(lens), hq, hkv, causal=causal, dq=dq, dk=dk, dv=dv, window=window,
                 head_dim=hd, scale=scale)
    return o, lse, dqkv


def _check_against_ref(qkv, d_o, o, lse_rows, dqkv, hq, hkv, causal=True, window=None, grads=True):
    """One sequence: o [L, hq*d], lse_rows [hq, L], dqkv [L, (hq + 2 hkv) * d] inside the per-element bounds of
    :func:`tests.numerics.attention_bounds` around the float64 reference."""
    L = qkv.shape[0]
    heads = lambda x, n: x.reshape(L, n, d)  # noqa: E731
    q, k, v = (heads(c, n) for c, n in zip(_cols(qkv, hq, hkv), (hq, hkv, hkv)))
    got = {"o": heads(o, hq), "lse": lse_rows}
    if grads:
        got.update(zip(("dq", "dk", "dv"), (heads(c, n) for c, n in zip(_cols(dqkv, hq, hkv), (hq, hkv, hkv)))))
    assert_attention_bounded(got, q, k, v, heads(d_o, hq) if grads else None, None, causal, window)


# ---- 1. dense against float64 ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S", [(1, 128), (2, 128), (1, 384), (2, 384), (1, 1024), (2, 1024)])
@pytest.mark.parametrize("hq,hkv", [(2, 2), (4, 2), (8, 2)])
@pytest.mark.parametrize("causal", [True, False])
def test_dense_matches_float64_reference(B, S, hq, hkv, causal):
    qkv = _qkv(B * S, hq, hkv, 3 + hq + S, 0.7)
    d_o = _qkv(B * S, hq, 0, 4 + S)
    o, lse, dqkv = _dense(qkv, d_o, B, S, hq, hkv, causal)
    assert o.shape == (B * S, hq * d) and lse.shape == (B, hq, S)
    assert torch.isfinite(dqkv.float()).all()  # every gradient element written
    o2, lse2, dqkv2 = _dense(qkv, d_o, B, S, hq, hkv, causal)
    assert torch.equal(o, o2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2)  # deterministic
    for b in range(B):
        rows = slice(b * S, (b + 1) * S)
        _check_against_ref(qkv[rows], d_o[rows], o[rows], lse[b], dqkv[rows], hq, hkv, causal)


@pytest.mark.parametrize("S", [77, 1000])
@pytest.mark.parametrize("causal", [True, False])
def test_dense_fwd_ragged_length(S, causal):
    hq, hkv = 4, 2
    qkv = _qkv(S, hq, hkv, 5 + S, 0.7)
    o, lse = _A().fwd(*_cols(qkv, hq, hkv), 1, S, hq, hkv, causal=causal, head_dim=d)
    _check_against_ref(qkv, None, o, lse[0], None, hq, hkv, causal, grads=False)


# ---- 2. zero-padding oracle: the trusted head-dim-128 kernels on heads padded with 64 zero columns ------------------------
def _pad(x, heads):
    """[T, heads * 64] -> [T, heads * 128], every head followed by 64 zero columns."""
    T = x.shape[0]
    return torch.nn.functional.pad(x.view(T, heads, d), (0, 128 - d)).reshape(T, heads * 128)


def _unpad(x, heads):
    T = x.shape[0]
    y = x.view(T, heads, 128)
    return y[..., :d].reshape(T, heads * d), y[..., d:]


def _bf16_ulp(x):
    """Spacing of bf16 numbers at |x| (8 significant bits); 2^-133 at 0."""
    _, e = torch.frexp(x.float().abs())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float32), e - 8)


def _within_one_ulp(a, b):
    diff = (a.float() - b.float()).abs()
    tol = torch.maximum(_bf16_ulp(a), _bf16_ulp(b))
    return bool((diff <= tol).all()), int((a != b).sum())


@pytest.mark.parametrize("mode", ["dense", "varlen", "window"])
def test_matches_hd128_kernel_on_zero_padded_heads(mode):
    hq, hkv = 4, 2
    H = hq + 2 * hkv
    lens = RAGGED if mode == "varlen" else None
    B, S = (1, sum(RAGGED)) if mode == "varlen" else (2, 512)
    T = B * S
    qkv = _qkv(T, hq, hkv, 71, 0.7)
    d_o = _qkv(T, hq, 0, 72)
    window = 100 if mode == "window" else None
    if mode == "varlen":
        o, lse, g = _varlen(qkv, d_o, lens, hq, hkv)
        o2, lse2, g2 = _varlen(_pad(qkv, H), _pad(d_o, hq), lens, hq, hkv, hd=128, scale=1 / 8)
    else:
        o, lse, g = _dense(qkv, d_o, B, S, hq, hkv, window=window)
        o2, lse2, g2 = _dense(_pad(qkv, H), _pad(d_o, hq), B, S, hq, hkv, window=window, hd=128, scale=1 / 8)
    o2, o_pad = _unpad(o2, hq)
    g2, g_pad = _unpad(g2, H)
    assert float(o_pad.abs().max()) == 0.0 and float(g_pad.abs().max()) == 0.0  # padded output columns exactly 0
    report = {}
    for name, a, b in (("O", o, o2), ("dQ", *[_cols(t, hq, hkv)[0] for t in (g, g2)]),
                       ("dK", *[_cols(t, hq, hkv)[1] for t in (g, g2)]), ("dV", *[_cols(t, hq, hkv)[2] for t in (g, g2)])):
        ok, n_diff = _within_one_ulp(a, b)
        assert ok, (name, n_diff)
        report[name] = n_diff
    report["LSE"] = int((lse != lse2).sum())
    assert (lse - lse2).abs().max().item() <= 1e-5 * lse.abs().max().item() + 1e-6
    print(f"\n[hd64 vs padded hd128, {mode}] elements not bit-equal: {report}")


# ---- 3. packed documents ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hq,hkv,causal", [(4, 2, True), (4, 2, False), (3, 1, True)])
def test_varlen_fwd_equals_dense_launch_per_document(hq, hkv, causal):
    A = _A()
    T = sum(RAGGED)
    qkv = _qkv(T, hq, hkv, 81 + hq + causal)
    q, k, v = _cols(qkv, hq, hkv)
    out = torch.full((T + 3, hq * d), 7.0, device="cuda", dtype=torch.bfloat16)
    _, lse = A.fwd_varlen(q, k, v, _cu(RAGGED), max(RAGGED), hq, hkv, causal=causal, out=out[:T], head_dim=d)
    for s, e in _spans(RAGGED):
        o1, l1 = A.fwd(*_cols(qkv[s:e].clone(), hq, hkv), 1, e - s, hq, hkv, causal=causal, head_dim=d)
        assert torch.equal(out[s:e], o1), (s, e)
        assert torch.equal(lse[:, s:e], l1[0]), (s, e)
    assert float((out[T:].float() - 7.0).abs().max()) == 0.0  # rows past T are never written


@pytest.mark.parametrize("causal", [True, False])
def test_varlen_bwd_equals_dense_launch_per_document(causal):
    hq, hkv = 4, 2
    lens = [5, 128, 256, 77, 384, 0, 128]
    T = sum(lens)
    qkv = _qkv(T, hq, hkv, 11, 0.7)
    d_o = _qkv(T, hq, 0, 12)
    o, _, dqkv = _varlen(qkv, d_o, lens, hq, hkv, causal)
    assert torch.isfinite(dqkv.float()).all()
    for s, e in _spans(lens):
        if (e - s) % 128:
            continue
        o1, _, g1 = _dense(qkv[s:e].clone(), d_o[s:e].clone(), 1, e - s, hq, hkv, causal)
        assert torch.equal(o[s:e], o1)
        assert torch.equal(dqkv[s:e], g1), (s, e)


@pytest.mark.parametrize("hq,hkv", [(2, 2), (3, 1), (8, 2)])
@pytest.mark.parametrize("causal", [True, False])
def test_varlen_matches_float64_reference(hq, hkv, causal):
    T = sum(RAGGED)
    qkv = _qkv(T, hq, hkv, 31 + hq, 0.7)
    d_o = _qkv(T, hq, 0, 32)
    o, lse, dqkv = _varlen(qkv, d_o, RAGGED, hq, hkv, causal)
    assert torch.isfinite(dqkv.float()).all()
    o2, lse2, dqkv2 = _varlen(qkv, d_o, RAGGED, hq, hkv, causal)
    assert torch.equal(o, o2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2)
    for s, e in _spans(RAGGED):
        _check_against_ref(qkv[s:e], d_o[s:e], o[s:e], lse[:, s:e], dqkv[s:e], hq, hkv, causal)


# ---- 4. sliding window -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,S,hq,hkv,W", SHAPES)
def test_window_matches_float64_reference(B, S, hq, hkv, W):
    qkv = _qkv(B * S, hq, hkv, 41 + hq + W, 0.7)
    d_o = _qkv(B * S, hq, 0, 42 + W)
    o, lse, dqkv = _dense(qkv, d_o, B, S, hq, hkv, window=W)
    assert torch.isfinite(dqkv.float()).all()
    o2, lse2, dqkv2 = _dense(qkv, d_o, B, S, hq, hkv, window=W)
    assert torch.equal(o, o2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2)
    for b in range(B):
        rows = slice(b * S, (b + 1) * S)
        _check_against_ref(qkv[rows], d_o[rows], o[rows], lse[b], dqkv[rows], hq, hkv, True, W)


@pytest.mark.parametrize("B,S", [(1, 384), (2, 512)])
def test_window_covering_sequence_equals_unwindowed_kernel(B, S):
    hq, hkv = 4, 2
    qkv = _qkv(B * S, hq, hkv, 7, 0.7)
    d_o = _qkv(B * S, hq, 0, 8)
    base = _dense(qkv, d_o, B, S, hq, hkv)
    for W in (S, S + 1, 10 * S):
        got = _dense(qkv, d_o, B, S, hq, hkv, window=W)
        assert all(torch.equal(a, b) for a, b in zip(base, got)), W


@pytest.mark.parametrize("W", [1, 64, 65, 200])
def test_packed_window_equals_dense_windowed_launch_per_document(W):
    A = _A()
    hq, hkv = 4, 2
    T = sum(RAGGED)
    qkv = _qkv(T, hq, hkv, W)
    q, k, v = _cols(qkv, hq, hkv)
    out = torch.full((T + 3, hq * d), 7.0, device="cuda", dtype=torch.bfloat16)
    _, lse = A.fwd_varlen(q, k, v, _cu(RAGGED), max(RAGGED), hq, hkv, causal=True, out=out[:T], window=W, head_dim=d)
    for s, e in _spans(RAGGED):
        o1, l1 = A.fwd(*_cols(qkv[s:e].clone(), hq, hkv), 1, e - s, hq, hkv, causal=True, window=W, head_dim=d)
        assert torch.equal(out[s:e], o1), (s, e)
        assert torch.equal(lse[:, s:e], l1[0]), (s, e)
    assert float((out[T:].float() - 7.0).abs().max()) == 0.0
    lens = [5, 128, 256, 77, 384, 0, 128]
    T = sum(lens)
    qkv = _qkv(T, hq, hkv, 11 + W, 0.7)
    d_o = _qkv(T, hq, 0, 12 + W)
    o, _, dqkv = _varlen(qkv, d_o, lens, hq, hkv, window=W)
    assert torch.isfinite(dqkv.float()).all()
    for s, e in _spans(lens):
        if (e - s) % 128:
            continue
        o1, _, g1 = _dense(qkv[s:e].clone(), d_o[s:e].clone(), 1, e - s, hq, hkv, window=W)
        assert torch.equal(o[s:e], o1)
        assert torch.equal(dqkv[s:e], g1), (s, e)


@pytest.mark.parametrize("B,S,W,P", [(1, 1024, 64, 128), (2, 512, 129, 200), (1, 1024, 300, 77)])
def test_keys_before_the_window_are_masked(B, S, W, P):
    """K / V rows [0, P) of every sequence get large finite values: rows >= P + W - 1 of O, LSE, dQ, dK and dV do not
    change by a bit."""
    hq, hkv = 4, 2
    qkv = _qkv(B * S, hq, hkv, 61, 0.7)
    d_o = _qkv(B * S, hq, 0, 62)
    o, lse, g = _dense(qkv, d_o, B, S, hq, hkv, window=W)
    pert = qkv.clone()
    for b in range(B):
        _, k, v = _cols(pert[b * S:b * S + P], hq, hkv)
        k.fill_(12.0)
        v.fill_(3000.0)
    o2, lse2, g2 = _dense(pert, d_o, B, S, hq, hkv, window=W)
    keep = (torch.arange(B * S, device="cuda") % S) >= P + W - 1
    assert torch.equal(o[keep], o2[keep])
    assert torch.equal(lse.permute(1, 0, 2).reshape(hq, B * S)[:, keep], lse2.permute(1, 0, 2).reshape(hq, B * S)[:, keep])
    assert torch.equal(g[keep], g2[keep])
    assert not torch.equal(o[~keep], o2[~keep])
    assert torch.isfinite(o2.float()).all() and torch.isfinite(g2.float()).all()


# ---- 5. public op ----------------------------------------------------------------------------------------------------------
def _public_op(backend, kind, base, gy, B, S, hq, hkv, rope):
    from deepspeed_b200.ops.attention import causal_attention
    cu = torch.tensor(np.concatenate([[0], np.cumsum([100, 300, 28, 0, 84])]), dtype=torch.int32)
    kw = {"dense": {}, "packed": dict(cu_seqlens=cu), "window": dict(sliding_window=96),
          "packed_window": dict(cu_seqlens=cu, sliding_window=96)}[kind]
    qkv = base.clone().requires_grad_(True)
    y = causal_attention(qkv * 1.0, B, S, hq, hkv, d, rope, None, backend=backend, **kw)
    y.backward(gy)
    return y.detach().float(), qkv.grad.float()


@pytest.mark.parametrize("kind", ["dense", "packed", "window", "packed_window"])
def test_public_op_native_matches_sdpa(kind):
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    hq, hkv = 4, 2
    B, S = 2, 256
    rope = RotaryTable(d, 512, 10000.0, "cuda")
    base = _qkv(B * S, hq, hkv, 51, 0.5)
    gy = _qkv(B * S, hq, 0, 52)
    ya, ga = _public_op("native", kind, base, gy, B, S, hq, hkv, rope)
    yb, gb = _public_op("cudnn", kind, base, gy, B, S, hq, hkv, rope)
    assert (ya - yb).abs().max().item() < 3e-2
    assert torch.isfinite(ga).all()
    assert torch.nn.functional.cosine_similarity(ga.flatten(), gb.flatten(), dim=0).item() > 0.999


# ---- 6. routing ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,native", [("dense", False), ("packed", True), ("window", True), ("packed_window", True)])
def test_auto_routing_at_head_dim_64_calls_kernel_entry_points(monkeypatch, kind, native):
    """``auto`` takes the native kernels (``fwd`` / ``fwd_varlen``) for packed and windowed inputs; a dense unwindowed
    input stays on SDPA (no measured table entry selects the native kernel for it)."""
    A = _A()
    calls = []
    for name in ("fwd", "fwd_varlen"):
        fn = getattr(A, name)
        monkeypatch.setattr(A, name, lambda *a, _fn=fn, _n=name, **k: (calls.append(_n), _fn(*a, **k))[1])
    hq, hkv, B, S = 4, 2, 2, 256
    base = _qkv(B * S, hq, hkv, 91, 0.5)
    gy = _qkv(B * S, hq, 0, 92)
    y, g = _public_op("auto", kind, base, gy, B, S, hq, hkv, None)
    assert torch.isfinite(y).all() and torch.isfinite(g).all()
    assert bool(calls) == native, calls


# ---- 7. engine -------------------------------------------------------------------------------------------------------------
def _train(backend, steps=3):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=512, intermediate_size=1024, num_attention_heads=8, num_key_value_heads=2,
                       head_dim=64, vocab_size=1024, num_hidden_layers=2, checkpoint_layers=1, attention_backend=backend,
                       max_position_embeddings=1024, sliding_window=128)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    engine, _, _, _ = ds.initialize(model=model, config={
        "train_micro_batch_size_per_gpu": 2,
        "bf16": {"enabled": True},
        "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
        "zero_optimization": {"stage": 3},
    })
    g = torch.Generator(device="cuda").manual_seed(1)
    ids = torch.randint(0, cfg.vocab_size, (2, 512), device="cuda", generator=g)
    cu = torch.tensor([0, 100, 400, 512, 530, 1024], dtype=torch.int32)
    losses = []
    for _ in range(steps):
        loss = engine(ids, labels=ids, cu_seqlens=cu)
        engine.backward(loss)
        engine.step()
        losses.append(float(loss.detach()))
    return losses


def _native_vs_fallback_training():
    native = _train("native")
    sdpa = _train("cudnn")
    assert all(math.isfinite(x) for x in native), native
    assert native[-1] < native[0], native
    for a, b in zip(native, sdpa):
        assert abs(a - b) < 2e-2 * abs(b) + 2e-2, (native, sdpa)


def test_llama_hd64_zero3_trains_packed_with_window():
    """A head-dim-64 Llama on packed documents with a sliding window: the native kernels against the SDPA fallbacks under
    the ZeRO-3 bf16 engine, in a fresh process so no state left by earlier tests in the session reaches the engines."""
    from tests.common import run_distributed
    run_distributed(_native_vs_fallback_training, 1, ())
