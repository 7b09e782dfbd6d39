"""FP8 dropless MoE experts on the host: the configuration and layout rules, the ragged FP8 node's torch reference path
against a float64 evaluation of each recipe per expert, and a tiny ``MixtralConfig(fp8_experts=True)`` trained under the
engine."""
import math

import pytest
import torch

from tests.common import run_distributed
from tests.numerics import U, assert_within, ulp
from deepspeed_b200.ops import fp8 as F8

B = 128
RECIPES = ["tensorwise", "blockwise"]


def _mixtral_cfg(**kw):
    from deepspeed_b200.models.mixtral import MixtralConfig
    d = dict(vocab_size=97, hidden_size=64, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
             num_key_value_heads=2, num_local_experts=4, num_experts_per_tok=2, max_position_embeddings=64,
             loss_chunk_tokens=16)
    d.update(kw)
    return MixtralConfig(**d)


def test_fp8_experts_default_off_and_bf16_experts_unchanged():
    from deepspeed_b200.models.mixtral import MixtralConfig, MixtralForCausalLM
    from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
    assert MixtralConfig().fp8_experts is False
    for fp8 in (False, True):  # ``fp8`` keeps meaning the attention projections
        m = MixtralForCausalLM(_mixtral_cfg(fp8=fp8, drop_tokens=False))
        ex = [x for x in m.modules() if isinstance(x, GroupedSwiGLUExperts)]
        assert ex and all(x.fp8_recipe is None and x.row_align == 64 for x in ex)
    for recipe in RECIPES:
        m = MixtralForCausalLM(_mixtral_cfg(fp8_experts=True, fp8_recipe=recipe, drop_tokens=False))
        ex = [x for x in m.modules() if isinstance(x, GroupedSwiGLUExperts)]
        assert ex and all(x.fp8_recipe == recipe and x.row_align == 128 for x in ex)


@pytest.mark.parametrize("kw", [dict(drop_tokens=True), dict(drop_tokens=False, ep_size=2),
                                dict(drop_tokens=False, fp8_recipe="rowwise")])
def test_fp8_experts_invalid_combinations_raise(kw):
    with pytest.raises(ValueError):
        _mixtral_cfg(fp8_experts=True, **kw)


def test_fp8_experts_refuse_the_capacity_layout():
    from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
    ex = GroupedSwiGLUExperts(2, 64, 64, fp8_recipe="tensorwise")
    with pytest.raises(ValueError, match="dropless"):
        ex(torch.randn(2, 8, 64))
    with pytest.raises(ValueError):
        GroupedSwiGLUExperts(2, 64, 64, fp8_recipe="delayed")


@pytest.mark.parametrize("recipe", [None] + RECIPES)
def test_dropless_buffer_rows(recipe, monkeypatch):
    """The dropless layer pads each expert's segment to ``row_align`` and sizes the buffer by its static bound: bf16
    ``T k + E 63`` exactly as before, FP8 ``T k + E 127`` rounded up to a multiple of 128."""
    from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
    from deepspeed_b200.moe.layer import MoE
    from deepspeed_b200.ops.kernels import moe_ops
    E, H, T, k = 4, 64, 37, 2
    torch.manual_seed(0)
    layer = MoE(H, GroupedSwiGLUExperts(E, H, 64, fp8_recipe=recipe), num_experts=E, k=k, min_capacity=4,
                drop_tokens=False, use_rts=False)
    seen = {}
    real = moe_ops.scatter

    def scatter(x, ids, pos, offsets, k_, cap, out_rows):
        seen["rows"], seen["offsets"] = out_rows, offsets.tolist()
        return real(x, ids, pos, offsets, k_, cap, out_rows)

    monkeypatch.setattr(moe_ops, "scatter", scatter)
    y, _, counts = layer(torch.randn(T, H))
    assert y.shape == (T, H) and bool(torch.isfinite(y).all())
    align = 64 if recipe is None else 128
    want = T * k + E * (align - 1)
    if recipe is not None:
        want = -(-want // 128) * 128
    assert seen["rows"] == want
    off = seen["offsets"]
    assert all(o % align == 0 for o in off) and off[-1] <= want
    assert [b - a for a, b in zip(off, off[1:])] == [-(-int(c) // align) * align for c in counts]


# ---------------------------------------------------------------------------------------------------------------------
# the node's reference path against float64, per expert
# ---------------------------------------------------------------------------------------------------------------------
def _deq_tensor(t, fmt):
    """Independent tensorwise cast: float64 dequantised values."""
    amax = float(t.float().abs().max())
    e = 0 if amax == 0 else math.floor(math.log2(F8.FMAX[fmt] / amax))
    return (t.float() * 2.0**e).to(fmt).double() * 2.0**-e


def _deq_block(q, s, mode):
    """float64 values of a blockwise cast ``q`` with scales ``s`` (``"strip"``: ``[ceil(C/128), R]``; ``"block"``)."""
    R, C = q.shape
    if mode == "strip":
        return q.double() * s.t().double().repeat_interleave(B, dim=1)[:, :C]
    return q.double() * s.double().repeat_interleave(B, dim=0)[:R].repeat_interleave(B, dim=1)[:, :C]


def _operand(t, fmt, recipe, mode, transposed=False):
    """The dequantised operand of one product: ``t`` (or ``t^T``) cast with the recipe's scaling for ``mode``."""
    if recipe == "tensorwise":
        d = _deq_tensor(t, fmt)
        return d.t() if transposed else d
    if transposed:
        _, _, qt, st = F8.quantize_blockwise_reference(t, fmt, row=None, col=mode)
        return _deq_block(qt, st, mode)
    q, s, _, _ = F8.quantize_blockwise_reference(t, fmt, row=mode)
    return _deq_block(q, s, mode)


def _bounded(got, a, b, what):
    """``got`` (bf16) within an fp32 accumulation of ``a @ b^T`` (float64 dequantised operands) rounded to bf16."""
    ref, mag = a @ b.t(), a.abs() @ b.abs().t()
    acc = 2 * (a.shape[1] + 1) * U * mag
    assert_within(got, ref, ulp(ref.abs() + acc, torch.bfloat16) + acc, what)


def _ragged_case(counts, H, I, seed, lead=0, tail=0):
    """Expert-sorted rows with 128-row zero-padded segments after ``lead`` zero rows and before ``tail`` zero rows."""
    g = torch.Generator().manual_seed(seed)
    E = len(counts)
    off = [lead]
    for c in counts:
        off.append(off[-1] + -(-c // B) * B)
    R = off[-1] + tail
    x = torch.zeros(R, H)
    dy = torch.zeros(R, H)
    for e, c in enumerate(counts):
        x[off[e]:off[e] + c] = torch.randn(c, H, generator=g) * (1 + e)
        dy[off[e]:off[e] + c] = torch.randn(c, H, generator=g)
    w13 = torch.randn(E, 2 * I, H, generator=g) * H**-0.5
    w2 = torch.randn(E, H, I, generator=g) * I**-0.5
    w13[1] *= 8  # one expert's weights far larger: a stacked scale is shared, a block scale is not
    return off, x.bfloat16(), dy.bfloat16(), w13.bfloat16(), w2.bfloat16()


@pytest.mark.parametrize("recipe", RECIPES)
def test_fp8_ragged_node_reference_matches_float64(recipe):
    from deepspeed_b200.ops.linear import fp8_ragged_swiglu_mlp
    counts = [130, 0, 1, 256]
    E, H, I = len(counts), 256, 192
    off, x0, dy, w13_0, w2_0 = _ragged_case(counts, H, I, seed=7, lead=128, tail=128)
    offsets = torch.tensor(off, dtype=torch.int32)
    x, w13, w2 = (t.clone().requires_grad_(True) for t in (x0, w13_0, w2_0))
    y = fp8_ragged_swiglu_mlp(x, offsets, w13, w2, recipe=recipe)
    gu = y.grad_fn.saved_tensors[3]
    y.backward(dy)
    assert bool((y[:off[0]] == 0).all()) and bool((y[off[-1]:] == 0).all())

    X = _operand(x0, F8.E4M3, recipe, "strip")
    W13 = _operand(w13_0.reshape(E * 2 * I, H), F8.E4M3, recipe, "block")
    W13T = _operand(w13_0.reshape(E * 2 * I, H), F8.E4M3, recipe, "block", transposed=True)  # [H, E 2I]
    W2 = _operand(w2_0.reshape(E * H, I), F8.E4M3, recipe, "block")
    W2T = _operand(w2_0.reshape(E * H, I), F8.E4M3, recipe, "block", transposed=True)  # [I, E H]
    gu64 = torch.zeros(x0.shape[0], 2 * I, dtype=torch.float64)
    for e in range(E):
        s = slice(off[e], off[e + 1])
        gu64[s] = X[s] @ W13[e * 2 * I:(e + 1) * 2 * I].t()
        if off[e + 1] > off[e]:
            _bounded(gu[s], X[s], W13[e * 2 * I:(e + 1) * 2 * I], f"gate|up expert {e}")
    act = (torch.nn.functional.silu(gu64[:, :I]) * gu64[:, I:]).bfloat16()
    A = _operand(act, F8.E4M3, recipe, "strip")
    AT = _operand(act, F8.E4M3, recipe, "block", transposed=True)  # [I, R]
    DY = _operand(dy, F8.E5M2, recipe, "strip")
    DYT = _operand(dy, F8.E5M2, recipe, "strip", transposed=True)  # [H, R]
    XT = _operand(x0, F8.E4M3, recipe, "block", transposed=True)  # [H, R]
    gb = gu.double()
    dgu = torch.zeros(x0.shape[0], 2 * I, dtype=torch.float64)
    for e in range(E):
        s = slice(off[e], off[e + 1])
        d = DY[s] @ W2T[:, e * H:(e + 1) * H].t()
        g_, u_ = gb[s, :I], gb[s, I:]
        sg = torch.sigmoid(g_)
        dgu[s] = torch.cat([d * u_ * sg * (1 + g_ * (1 - sg)), d * g_ * sg], dim=1)
    dgu = dgu.bfloat16()
    DG = _operand(dgu, F8.E5M2, recipe, "strip")
    DGT = _operand(dgu, F8.E5M2, recipe, "strip", transposed=True)  # [2I, R]
    for e in range(E):
        s = slice(off[e], off[e + 1])
        if off[e + 1] > off[e]:
            _bounded(y[s], A[s], W2[e * H:(e + 1) * H], f"y expert {e}")
            _bounded(x.grad[s], DG[s], W13T[:, e * 2 * I:(e + 1) * 2 * I], f"dx expert {e}")
            _bounded(w2.grad[e], DYT[:, s], AT[:, s], f"dW2 expert {e}")
            _bounded(w13.grad[e], DGT[:, s], XT[:, s], f"dW13 expert {e}")
        else:
            assert not bool(w2.grad[e].any()) and not bool(w13.grad[e].any()), f"empty expert {e}"


def test_fp8_ragged_reference_refuses_unaligned_segments():
    from deepspeed_b200.ops.linear import fp8_ragged_swiglu_mlp
    x = torch.randn(256, 64).bfloat16()
    with pytest.raises(ValueError, match="multiples of 128"):
        fp8_ragged_swiglu_mlp(x, torch.tensor([0, 64, 256], dtype=torch.int32), torch.randn(2, 128, 64).bfloat16(),
                              torch.randn(2, 64, 64).bfloat16())


# ---------------------------------------------------------------------------------------------------------------------
# training under the engine
# ---------------------------------------------------------------------------------------------------------------------
def _train_fp8_mixtral(recipe):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.mixtral import MixtralForCausalLM
    from deepspeed_b200.ops import linear
    calls = {"n": 0}
    real = linear._FP8RaggedSwiGLUFn.apply

    def node(*a):
        calls["n"] += 1
        return real(*a)

    linear._FP8RaggedSwiGLUFn.apply = node
    torch.manual_seed(0)
    model = MixtralForCausalLM(_mixtral_cfg(fp8_experts=True, fp8_recipe=recipe, drop_tokens=False))
    cfg = {"train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
           "optimizer": {"type": "AdamW", "params": {"lr": 3e-3}}, "zero_optimization": {"stage": 2}}
    eng, _, _, _ = ds.initialize(model=model, config=cfg)
    ids = torch.randint(0, 97, (2, 16), generator=torch.Generator().manual_seed(5))
    losses = []
    for _ in range(8):
        loss = eng(ids, labels=ids)
        eng.backward(loss)
        eng.step()
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses), losses
    assert losses[-1] < losses[0] - 0.5, losses
    assert calls["n"] > 0, calls


@pytest.mark.parametrize("recipe", RECIPES)
def test_fp8_mixtral_trains_under_engine(recipe):
    run_distributed(_train_fp8_mixtral, 1, (recipe, ))
