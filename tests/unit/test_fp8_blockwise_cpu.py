"""Blockwise FP8 recipe on the host: the per-block casts against an independent block-by-block cast, the two autograd
nodes on their torch reference path against float64 products of the dequantised operands, what the recipe buys when an
activation holds an outlier, the ``fp8_recipe`` config field and a tiny blockwise Llama trained under the engine."""
import math

import pytest
import torch

from tests.common import run_distributed
from tests.numerics import U, assert_within, ulp
from deepspeed_b200.ops import fp8 as F8

FMTS = [F8.E4M3, F8.E5M2]
B = 128


def _blocks(n, size):
    return [(s, min(n, s + size)) for s in range(0, n, size)]


def _cast_by_blocks(x, fmt, rows, cols):
    """Independent cast, one ``rows x cols`` block of ``x`` at a time with :func:`scale_from_amax` and torch's fp8 cast:
    ``(q [R, C], scale_inv [row blocks, column blocks])``."""
    R, C = x.shape
    rbs, cbs = _blocks(R, rows), _blocks(C, cols)
    q = torch.empty(R, C, dtype=fmt)
    si = torch.empty(len(rbs), len(cbs), dtype=torch.float32)
    for i, (r0, r1) in enumerate(rbs):
        for j, (c0, c1) in enumerate(cbs):
            blk = x[r0:r1, c0:c1].float()
            scale, inv = F8.scale_from_amax(blk.abs().max().reshape(1), fmt)
            q[r0:r1, c0:c1] = (blk * scale).to(fmt)
            si[i, j] = inv[0]
    return q, si


def _same_bytes(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _same_scales(a, b):
    return a.shape == b.shape and a.dtype == torch.float32 and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("shape", [(5, 7), (128, 256), (130, 260), (16, 300)])
def test_blockwise_cast_is_torch_cast_block_by_block(fmt, shape):
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(shape, generator=g) * torch.logspace(-3, 3, shape[1])).bfloat16()
    x = x * torch.logspace(-2, 2, shape[0])[:, None].bfloat16()
    # row-major copy in row strips, transposed copy in strips along the rows of x
    q, sq, qt, st = F8.quantize_blockwise(x, fmt, row="strip", col="strip")
    want, si = _cast_by_blocks(x, fmt, 1, B)
    assert _same_bytes(q, want) and _same_scales(sq, si.t().contiguous())  # [ceil(C/128), R]
    want, si = _cast_by_blocks(x, fmt, B, 1)
    assert _same_bytes(qt, want.t().contiguous()) and _same_scales(st, si)  # [ceil(R/128), C]
    # both copies in 128 x 128 blocks: the same bytes, transposed, and transposed scale grids
    q, sq, qt, st = F8.quantize_blockwise(x, fmt, row="block", col="block")
    want, si = _cast_by_blocks(x, fmt, B, B)
    assert _same_bytes(q, want) and _same_scales(sq, si)
    assert _same_bytes(qt, want.t().contiguous()) and _same_scales(st, si.t().contiguous())
    assert float(q.float().abs().max()) <= F8.FMAX[fmt]
    # one copy only
    q, sq, qt, st = F8.quantize_blockwise(x, fmt, row=None, col="block")
    assert q is None and sq is None and _same_bytes(qt, want.t().contiguous())
    q, sq, qt, st = F8.quantize_blockwise(x, fmt, row="strip")
    assert qt is None and st is None and q is not None


def test_blockwise_zero_block_has_scale_one():
    x = torch.ones(130, 300, dtype=torch.bfloat16)
    x[:128, 128:256] = 0
    q, sq, qt, st = F8.quantize_blockwise(x, F8.E4M3, row="strip", col="block")
    assert bool((sq[1, :128] == 1).all()) and bool((sq[1, 128:] != 1).all()) and bool((sq[0] != 1).all())
    assert st[1, 0] == 1 and int((st == 1).sum()) == 1
    assert bool((q[:128, 128:256].float() == 0).all())


@pytest.mark.parametrize("bad", [math.inf, math.nan])
def test_blockwise_nonfinite_poisons_its_block_only(bad):
    x = torch.ones(256, 384, dtype=torch.bfloat16)
    x[130, 200] = bad  # row block 1, column block 1
    q, sq, qt, st = F8.quantize_blockwise(x, F8.E4M3, row="strip", col="block")
    nan = sq.isnan()
    assert bool(nan[1, 130]) and int(nan.sum()) == 1, "one row strip"
    assert bool(q[130, 128:256].float().isnan().all()) and int(q.float().isnan().sum()) == 128
    nan = st.isnan()
    assert bool(nan[1, 1]) and int(nan.sum()) == 1, "one 128 x 128 block"
    assert int(qt.float().isnan().sum()) == 128 * 128 and bool(qt[128:256, 128:256].float().isnan().all())
    _, _, qt, st = F8.quantize_blockwise(x, F8.E5M2, row=None, col="strip")
    assert bool(st[1, 200].isnan()) and int(st.isnan().sum()) == 1, "one column strip"
    assert int(qt.float().isnan().sum()) == 128 and bool(qt[200, 128:256].float().isnan().all())


def test_blockwise_matmul_reference_scales_every_block():
    g = torch.Generator().manual_seed(4)
    a = torch.randn(40, 300, generator=g).bfloat16()
    b = torch.randn(200, 300, generator=g).bfloat16()
    a8, sa, _, _ = F8.quantize_blockwise(a, F8.E4M3, row="strip")
    b8, sb, _, _ = F8.quantize_blockwise(b, F8.E4M3, row="block")
    got = F8.matmul_blockwise_reference(a8, b8, sa, sb)
    ad = a8.double() * sa.t().double().repeat_interleave(B, dim=1)[:, :300]
    bd = b8.double() * sb.double().repeat_interleave(B, dim=0)[:200].repeat_interleave(B, dim=1)[:, :300]
    ref, mag = ad @ bd.t(), ad.abs() @ bd.abs().t()
    assert_within(got, ref, 2 * 300 * U * mag, "blockwise product")


def _dq(t, fmt, rows, cols):
    """float64 dequantised values of ``t`` cast with one scale per ``rows x cols`` block."""
    q, si = _cast_by_blocks(t, fmt, rows, cols)
    full = si.double().repeat_interleave(rows, dim=0)[:t.shape[0]].repeat_interleave(cols, dim=1)[:, :t.shape[1]]
    return q.double() * full


def _bounded(got, a, b, what):
    """``got`` (bf16) within an fp32 accumulation of ``a @ b^T`` (float64 dequantised operands) rounded to bf16."""
    ref = a @ b.t()
    acc = 2 * a.shape[1] * U * (a.abs() @ b.abs().t())
    assert_within(got, ref, ulp(ref.abs() + acc, torch.bfloat16) + acc, what)


def test_fp8_blockwise_linear_reference_matches_float64():
    from deepspeed_b200.ops.linear import fp8_linear
    g = torch.Generator().manual_seed(1)
    T, K, N = 136, 200, 144
    x = (torch.randn(2, T // 2, K, generator=g) * torch.logspace(-1, 1, K)).bfloat16().requires_grad_(True)
    w = (0.05 * torch.randn(N, K, generator=g)).bfloat16().requires_grad_(True)
    b = torch.randn(N, generator=g).bfloat16().requires_grad_(True)
    dy = (torch.randn(2, T // 2, N, generator=g) * torch.logspace(-2, 0, N)).bfloat16()
    y = fp8_linear(x, w, b, recipe="blockwise")
    y.backward(dy)
    x2, dy2, wd = x.detach().reshape(T, K), dy.reshape(T, N), w.detach()
    y0 = fp8_linear(x.detach(), wd, recipe="blockwise")
    assert torch.equal(y.detach(), y0 + b.detach())
    w_dq = _dq(wd, F8.E4M3, B, B)
    _bounded(y0.reshape(T, N), _dq(x2, F8.E4M3, 1, B), w_dq, "y")
    _bounded(x.grad.reshape(T, K), _dq(dy2, F8.E5M2, 1, B), w_dq.t(), "dx")
    # the weight gradient contracts over tokens: dY in strips along them, x in blocks
    _bounded(w.grad, _dq(dy2, F8.E5M2, B, 1).t(), _dq(x2, F8.E4M3, B, B).t(), "dw")
    torch.testing.assert_close(b.grad, dy2.sum(0))
    assert not torch.equal(y0, fp8_linear(x.detach(), wd)), "the two recipes are different computations"


def test_fp8_blockwise_swiglu_reference_matches_float64():
    from deepspeed_b200.ops.linear import fp8_swiglu_mlp
    g = torch.Generator().manual_seed(2)
    T, H, I = 144, 160, 192
    x = torch.randn(T, H, generator=g).bfloat16().requires_grad_(True)
    wgu = (0.1 * torch.randn(2 * I, H, generator=g)).bfloat16().requires_grad_(True)
    wd = (0.1 * torch.randn(H, I, generator=g)).bfloat16().requires_grad_(True)
    dy = torch.randn(T, H, generator=g).bfloat16()
    y = fp8_swiglu_mlp(x, wgu, wd, recipe="blockwise")
    y.backward(dy)
    # forward, step by step on the dequantised operands
    wgu_dq, wd_dq = _dq(wgu.detach(), F8.E4M3, B, B), _dq(wd.detach(), F8.E4M3, B, B)
    gu = _dq(x.detach(), F8.E4M3, 1, B) @ wgu_dq.t()
    act = (torch.nn.functional.silu(gu[:, :I]) * gu[:, I:]).bfloat16()
    _bounded(y.detach(), _dq(act, F8.E4M3, 1, B), wd_dq, "y")
    # backward from the saved bf16 gate|up, as the node does
    gub = gu.bfloat16().double()
    gb, ub = gub[:, :I], gub[:, I:]
    d = _dq(dy, F8.E5M2, 1, B) @ wd_dq
    s = torch.sigmoid(gb)
    dgu = torch.cat([d * ub * s * (1 + gb * (1 - s)), d * gb * s], dim=1).bfloat16()
    _bounded(x.grad, _dq(dgu, F8.E5M2, 1, B), wgu_dq.t(), "dx")
    _bounded(wd.grad, _dq(dy, F8.E5M2, B, 1).t(), _dq(act, F8.E4M3, B, B).t(), "dw_down")
    _bounded(wgu.grad, _dq(dgu, F8.E5M2, B, 1).t(), _dq(x.detach(), F8.E4M3, B, B).t(), "dw_gate_up")


def _cast_errors(x, w):
    """|x - dequantised x| (1 x 128 strips) and |w - dequantised w| (128 x 128 blocks), float64."""
    return (_dq(x, F8.E4M3, 1, B) - x.double()).abs(), (_dq(w, F8.E4M3, B, B) - w.double()).abs()


def test_blockwise_confines_an_outlier_tensorwise_does_not():
    """One element of ``x`` 2**15 times the rest, against the float64 product of the unquantised operands.

    The per-block bound: with ``dx``, ``dw`` what each operand loses when every block is cast with its own scale, the
    product errs by at most ``dx |w| + |x| dw + dx dw`` summed over k, plus the fp32 accumulation and the bf16 rounding.
    The inputs have four significant bits, which e4m3 holds when a block is scaled by its own amax, so ``dx = dw = 0``
    outside the outlier's strip.  Tensorwise, the outlier's scale leaves the rest of ``x`` two bits (e4m3 subnormals),
    every element of it is rounded, and the product's error in the rows the outlier is not in exceeds the per-block bound
    ``FACTOR`` times over."""
    from deepspeed_b200.ops.linear import fp8_linear
    FACTOR = 4.0
    g = torch.Generator().manual_seed(7)
    T, K, N = 64, 512, 128
    odd = lambda shape: (2 * torch.randint(0, 4, shape, generator=g) + 9).float() / 8  # 1.125, 1.375, 1.625, 1.875
    sign = lambda shape: (2 * torch.randint(0, 2, shape, generator=g) - 1).float()
    x = (odd((T, K)) * sign((T, K))).bfloat16()
    w = (odd((N, K)) * sign((N, K)) / 16).bfloat16()
    x[3, 5] = 2.0**15
    exact = x.double() @ w.double().t()
    dx, dw = _cast_errors(x, w)
    others = torch.arange(T) != 3
    assert float(dx[others].max()) == 0 and float(dw.max()) == 0 and float(dx[3, :128].max()) > 0
    xa, wa = x.double().abs(), w.double().abs()
    bound = dx @ wa.t() + xa @ dw.t() + dx @ dw.t() + 2 * K * U * (xa @ wa.t())
    bound = bound + ulp(exact.abs() + bound, torch.bfloat16)
    err_block = (fp8_linear(x, w, recipe="blockwise").double() - exact).abs()
    err_tensor = (fp8_linear(x, w, recipe="tensorwise").double() - exact).abs()
    assert bool((err_block <= bound).all()), float((err_block / bound).max())
    assert float((err_tensor[others] > FACTOR * bound[others]).float().mean()) > 0.5, "most elements, not a stray one"
    assert float((err_tensor[others] / bound[others]).max()) > 10 * FACTOR


def test_blockwise_outlier_on_gaussian_data():
    """The same outlier in Gaussian activations: relative error of the rows the outlier is not in."""
    from deepspeed_b200.ops.linear import fp8_linear
    g = torch.Generator().manual_seed(8)
    T, K, N = 64, 512, 128
    x = torch.randn(T, K, generator=g).bfloat16()
    w = (0.05 * torch.randn(N, K, generator=g)).bfloat16()
    clean = fp8_linear(x, w, recipe="tensorwise").double()
    x[3, 5] = 2.0**15
    exact = x.double() @ w.double().t()
    others = torch.arange(T) != 3
    rel = lambda y: float((y.double() - exact)[others].norm() / exact[others].norm())
    block, tensor = rel(fp8_linear(x, w, recipe="blockwise")), rel(fp8_linear(x, w, recipe="tensorwise"))
    assert block < 0.05 and tensor > 2 * block, (block, tensor)
    assert block <= 1.05 * rel(clean), "blockwise with the outlier is as good as tensorwise without it"


def _tiny(recipe="blockwise", **kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", vocab_size=97, hidden_size=64, intermediate_size=128, num_attention_heads=4,
                       num_key_value_heads=2, loss_chunk_tokens=16, fp8=True, fp8_recipe=recipe, **kw)
    return LlamaForCausalLM(cfg)


def _train_blockwise_llama(stage):
    import deepspeed_b200 as ds
    from deepspeed_b200.ops import linear
    calls = {"lin": 0, "mlp": 0}
    real_lin, real_mlp = linear._FP8LinearFn.apply, linear._FP8SwiGLUMLPFn.apply

    def lin(*a):
        calls["lin"] += 1
        assert a[-1] is True, "a tensorwise node ran under fp8_recipe='blockwise'"
        return real_lin(*a)

    def mlp(*a):
        calls["mlp"] += 1
        assert a[-1] is True, "a tensorwise node ran under fp8_recipe='blockwise'"
        return real_mlp(*a)

    linear._FP8LinearFn.apply, linear._FP8SwiGLUMLPFn.apply = lin, mlp
    model = _tiny(checkpoint_layers=1)
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
    assert calls["lin"] > 0 and calls["mlp"] > 0, calls


@pytest.mark.parametrize("stage", [1, 3])
def test_fp8_blockwise_llama_trains_block_scaled_under_engine(stage):
    run_distributed(_train_blockwise_llama, 1, (stage, ))


def test_fp8_recipe_config():
    from deepspeed_b200.models.llama import LlamaAttention, LlamaConfig, LlamaMLP
    from deepspeed_b200.models.mixtral import MixtralConfig, MixtralForCausalLM
    from deepspeed_b200.ops.linear import fp8_linear, fp8_swiglu_mlp
    assert LlamaConfig().fp8_recipe == "tensorwise" and LlamaConfig().fp8 is False
    with pytest.raises(ValueError, match="fp8_recipe"):
        LlamaConfig(fp8=True, fp8_recipe="rowwise")
    with pytest.raises(ValueError, match="fp8_recipe"):
        MixtralConfig(fp8_recipe="")
    x, w = torch.zeros(4, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="recipe"):
        fp8_linear(x, w, recipe="block")
    with pytest.raises(ValueError, match="recipe"):
        fp8_swiglu_mlp(x, torch.zeros(16, 8, dtype=torch.bfloat16), w, recipe=None)
    m = _tiny()
    mlps = [mod for mod in m.modules() if isinstance(mod, LlamaMLP)]
    attn = [mod for mod in m.modules() if isinstance(mod, LlamaAttention)]
    assert mlps and all(mod.fp8 and mod.fp8_recipe == "blockwise" for mod in mlps)
    assert attn and all(a.qkv_proj.fp8_recipe == "blockwise" and a.o_proj.fp8_recipe == "blockwise" for a in attn)
    assert all(a.qkv_proj.fp8_recipe == "tensorwise" for a in _tiny("tensorwise").modules() if isinstance(a, LlamaAttention))
    cfg = MixtralConfig(vocab_size=64, hidden_size=64, intermediate_size=64, num_hidden_layers=1, num_attention_heads=4,
                        num_key_value_heads=2, num_local_experts=2, fp8=True, fp8_recipe="blockwise")
    mx = MixtralForCausalLM(cfg)
    attn = [mod for mod in mx.modules() if isinstance(mod, LlamaAttention)]
    assert attn and all(a.qkv_proj.fp8 and a.qkv_proj.fp8_recipe == "blockwise" and a.o_proj.fp8_recipe == "blockwise"
                        for a in attn)
