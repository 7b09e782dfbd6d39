"""FP8 training recipe on the host: the scale rule, the casts, the two autograd nodes on their torch reference path and a
tiny ``LlamaConfig(fp8=True)`` model trained under the engine."""
import math

import pytest
import torch

from tests.common import run_distributed
from tests.numerics import U, assert_within, ulp
from deepspeed_b200.ops import fp8 as F8

FMTS = [F8.E4M3, F8.E5M2]


@pytest.mark.parametrize("fmt", FMTS)
def test_scale_rule(fmt):
    fmax = F8.FMAX[fmt]
    # powers of two, values just around them, FMAX and its neighbours, tiny and huge normals
    vals = [2.0**k * m for k in range(-120, 120, 7) for m in (1.0, 1.0 + 2**-23, 1.5, 1.75, 1.75 + 2**-20, 2 - 2**-23)]
    vals += [fmax, math.nextafter(fmax, 0), math.nextafter(fmax, math.inf), 1.0, 3.0e38]
    amax = torch.tensor(vals, dtype=torch.float32)
    scale, scale_inv = F8.scale_from_amax(amax, fmt)
    m, _ = torch.frexp(scale)
    assert bool((m == 0.5).all()), "scales are powers of two"
    assert torch.equal(scale * scale_inv, torch.ones_like(scale))
    a64, s64 = amax.double(), scale.double()
    assert bool((a64 * s64 <= fmax).all()), "no value saturates"
    # the largest such power of two (unless the clamp at 2**126 binds)
    assert bool(((a64 * s64 * 2 > fmax) | (scale == 2.0**126)).all())
    want = torch.floor(torch.log2(torch.tensor(fmax, dtype=torch.float64) / a64)).clamp(-126, 126)
    fine = (a64 * 2.0**want <= fmax)  # float64 log2 is exact away from the binade edges
    assert torch.equal(torch.log2(s64)[fine], want[fine])


@pytest.mark.parametrize("fmt", FMTS)
def test_scale_rule_edges(fmt):
    amax = torch.tensor([0.0, 2.0**-140, 1e-45, math.inf, math.nan], dtype=torch.float32)
    scale, scale_inv = F8.scale_from_amax(amax, fmt)
    assert scale[0] == 1 and scale_inv[0] == 1, "amax 0 gives scale 1"
    assert scale[1] == 2.0**126 and scale[2] == 2.0**126, "subnormal amax: exponent clamped, scale stays finite"
    assert scale_inv[1] == 2.0**-126
    assert bool(scale[3:].isnan().all()) and bool(scale_inv[3:].isnan().all()), "non-finite amax gives NaN scales"


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("shape", [(5, 7), (64, 48), (33, 160)])
def test_quantize_is_torch_cast(fmt, shape):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(shape, generator=g) * torch.logspace(-3, 3, shape[1])).bfloat16()
    q, qt, si = F8.quantize_tensorwise(x, fmt, rowwise=True, colwise=True)
    amax = x.float().abs().max()
    e = math.floor(math.log2(F8.FMAX[fmt] / float(amax)))
    want = (x.float() * 2.0**e).to(fmt)
    assert q.dtype == fmt and qt.dtype == fmt and si.dtype == torch.float32 and si.shape == (1, )
    assert torch.equal(q.view(torch.uint8), want.view(torch.uint8))
    assert torch.equal(qt.view(torch.uint8), want.t().contiguous().view(torch.uint8))
    assert float(si) == 2.0**-e
    assert bool((q.float().abs().amax() <= F8.FMAX[fmt]))


@pytest.mark.parametrize("bad", [math.inf, math.nan])
def test_quantize_nonfinite_is_nan(bad):
    x = torch.ones(4, 8, dtype=torch.bfloat16)
    x[1, 3] = bad
    q, _, si = F8.quantize_tensorwise(x, F8.E4M3)
    assert bool(si.isnan().all()) and bool(q.float().isnan().all())


def _q(t, fmt):
    """Independent cast of the recipe: (dequantised float64 values, float64 scale_inv)."""
    amax = float(t.float().abs().max())
    e = 0 if amax == 0 else math.floor(math.log2(F8.FMAX[fmt] / amax))
    return (t.float() * 2.0**e).to(fmt).double(), 2.0**-e


def _bounded(got, a, b, s, what):
    """``got`` (bf16) within an fp32 accumulation of ``s * a @ b^T`` (float64 operands) rounded to bf16."""
    ref = (a @ b.t()) * s
    mag = (a.abs() @ b.abs().t()) * s
    acc = 2 * a.shape[1] * U * mag
    assert_within(got, ref, ulp(ref.abs() + acc, torch.bfloat16) + acc, what)


def test_fp8_linear_reference_matches_float64():
    from deepspeed_b200.ops.linear import fp8_linear
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 24, 40, generator=g).bfloat16().requires_grad_(True)
    w = (0.05 * torch.randn(56, 40, generator=g)).bfloat16().requires_grad_(True)
    b = torch.randn(56, generator=g).bfloat16().requires_grad_(True)
    dy = torch.randn(2, 24, 56, generator=g).bfloat16()
    y = fp8_linear(x, w, b)
    y.backward(dy)
    x2, dy2 = x.detach().reshape(-1, 40), dy.reshape(-1, 56)
    x8, sx = _q(x2, F8.E4M3)
    w8, sw = _q(w.detach(), F8.E4M3)
    dy8, sdy = _q(dy2, F8.E5M2)
    y0 = fp8_linear(x.detach(), w.detach())
    assert torch.equal(y.detach(), y0 + b.detach())
    _bounded(y0.reshape(-1, 56), x8, w8, sx * sw, "y")
    _bounded(x.grad.reshape(-1, 40), dy8, w8.t(), sdy * sw, "dx")
    _bounded(w.grad, dy8.t(), x8.t(), sdy * sx, "dw")
    torch.testing.assert_close(b.grad, dy2.sum(0))


def test_fp8_swiglu_reference_matches_float64():
    from deepspeed_b200.ops.linear import fp8_swiglu_mlp
    g = torch.Generator().manual_seed(2)
    T, H, I = 48, 32, 64
    x = torch.randn(T, H, generator=g).bfloat16().requires_grad_(True)
    wgu = (0.1 * torch.randn(2 * I, H, generator=g)).bfloat16().requires_grad_(True)
    wd = (0.1 * torch.randn(H, I, generator=g)).bfloat16().requires_grad_(True)
    dy = torch.randn(T, H, generator=g).bfloat16()
    y = fp8_swiglu_mlp(x, wgu, wd)
    y.backward(dy)
    # forward, step by step on the quantised operands
    x8, sx = _q(x.detach(), F8.E4M3)
    wgu8, sgu = _q(wgu.detach(), F8.E4M3)
    gu = (x8 @ wgu8.t()) * (sx * sgu)
    gate, up = gu[:, :I], gu[:, I:]
    act = (torch.nn.functional.silu(gate) * up).bfloat16()
    a8, sa = _q(act, F8.E4M3)
    wd8, sd = _q(wd.detach(), F8.E4M3)
    _bounded(y.detach(), a8, wd8, sa * sd, "y")
    # backward from the saved bf16 gate|up, as the node does
    dy8, sdy = _q(dy, F8.E5M2)
    gub = gu.bfloat16().double()
    gb, ub = gub[:, :I], gub[:, I:]
    d = (dy8 @ wd8) * (sdy * sd)
    s = torch.sigmoid(gb)
    dgu = torch.cat([d * ub * s * (1 + gb * (1 - s)), d * gb * s], dim=1).bfloat16()
    dg8, sg = _q(dgu, F8.E5M2)
    _bounded(x.grad, dg8, wgu8.t(), sg * sgu, "dx")
    _bounded(wd.grad, dy8.t(), a8.t(), sdy * sa, "dw_down")
    _bounded(wgu.grad, dg8.t(), x8.t(), sg * sx, "dw_gate_up")


def test_fp8_nodes_differ_from_bf16_and_stay_close():
    from deepspeed_b200.ops.linear import flat_linear, fp8_linear
    g = torch.Generator().manual_seed(3)
    x = torch.randn(32, 64, generator=g).bfloat16()
    w = (0.05 * torch.randn(48, 64, generator=g)).bfloat16()
    y8, y16 = fp8_linear(x, w), flat_linear(x, w)
    assert not torch.equal(y8, y16)
    assert float((y8.float() - y16.float()).norm() / y16.float().norm()) < 0.1


def _tiny_fp8(fp8=True, **kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", vocab_size=97, hidden_size=64, intermediate_size=128, num_attention_heads=4,
                       num_key_value_heads=2, loss_chunk_tokens=16, fp8=fp8, **kw)
    return LlamaForCausalLM(cfg)


def _train_fp8_llama(stage):
    import deepspeed_b200 as ds
    from deepspeed_b200.ops import linear
    calls = {"lin": 0, "mlp": 0}
    real_lin, real_mlp = linear._FP8LinearFn.apply, linear._FP8SwiGLUMLPFn.apply

    def lin(*a):
        calls["lin"] += 1
        assert a[-1] is False, "a blockwise node ran under the default fp8_recipe='tensorwise'"
        return real_lin(*a)

    def mlp(*a):
        calls["mlp"] += 1
        assert a[-1] is False, "a blockwise node ran under the default fp8_recipe='tensorwise'"
        return real_mlp(*a)

    linear._FP8LinearFn.apply, linear._FP8SwiGLUMLPFn.apply = lin, mlp
    model = _tiny_fp8(checkpoint_layers=1)
    cfg = {"train_micro_batch_size_per_gpu": 2, "gradient_accumulation_steps": 2, "bf16": {"enabled": True},
           "optimizer": {"type": "AdamW", "params": {"lr": 3e-3}}, "zero_optimization": {"stage": stage}}
    if stage == 3:
        cfg["zero_optimization"]["stage3_param_persistence_threshold"] = 0
    eng, _, _, _ = ds.initialize(model=model, config=cfg)
    ids = torch.randint(0, 97, (2, 16), generator=torch.Generator().manual_seed(5))
    losses = []
    for _ in range(8):
        for _ in range(2):
            loss = eng(ids, labels=ids)
            eng.backward(loss)
            eng.step()
        losses.append(float(loss))
    assert all(math.isfinite(v) for v in losses), losses
    assert losses[-1] < losses[0] - 0.5, losses
    # 2 layers x (qkv, o) linears and 2 MLP blocks per forward (the checkpointed layer runs its forward twice)
    assert calls["lin"] > 0 and calls["mlp"] > 0, calls


@pytest.mark.parametrize("stage", [0, 3])
def test_fp8_llama_trains_under_engine(stage):
    run_distributed(_train_fp8_llama, 1, (stage, ))


def test_fp8_config_default_off_and_mixtral_attention_only():
    from deepspeed_b200.models.llama import LlamaAttention, LlamaConfig, LlamaMLP
    from deepspeed_b200.models.mixtral import MixtralConfig, MixtralForCausalLM
    assert LlamaConfig().fp8 is False
    m = _tiny_fp8(fp8=False)
    assert not any(getattr(mod, "fp8", False) for mod in m.modules())
    cfg = MixtralConfig(vocab_size=64, hidden_size=64, intermediate_size=64, num_hidden_layers=1, num_attention_heads=4,
                        num_key_value_heads=2, num_local_experts=2, fp8=True)
    mx = MixtralForCausalLM(cfg)
    attn = [m for m in mx.modules() if isinstance(m, LlamaAttention)]
    assert attn and all(a.qkv_proj.fp8 and a.o_proj.fp8 for a in attn)
    assert not any(isinstance(m, LlamaMLP) for m in mx.modules()), "MoE experts keep their bf16 path"
