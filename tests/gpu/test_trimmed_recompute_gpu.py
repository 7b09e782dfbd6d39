"""GPU tier: activation-checkpointed Llama layers replay their forward only as far as backward reads.

* the dSwiGLU pass (``gated_act_bwd_kernel``) writes ``act`` bit-identical to ``gated_act_fwd_kernel``;
* loss and every parameter gradient of the trimmed replay equal the whole-layer replay bit for bit, for the tiny and a
  2-layer Llama-3.2-3B-width model, dense, packed and sliding-window, on the library and on the in-tree GEMM paths;
* a replayed layer launches no down-projection GEMM and no ``gated_act_fwd_kernel``.
"""
import pytest
import torch

from deepspeed_b200.ops import gemm
from deepspeed_b200.ops.kernels import transformer_ops as T
from deepspeed_b200.runtime.activation_checkpointing import checkpointing as ckpt
from tests.numerics import assert_bits_equal

pytestmark = pytest.mark.gpu


@pytest.fixture
def backend(request, monkeypatch):
    """Select a GEMM backend for one test without leaving backend or choice state behind."""
    monkeypatch.setattr(gemm, "_backend", request.param)
    monkeypatch.setattr(gemm, "_used", {})
    monkeypatch.setattr(gemm, "_measured", {})
    return request.param


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("tokens,inter", [(1000, 1280), (37, 8192)])
def test_dswiglu_pass_writes_forward_act(dtype, tokens, inter):
    g = torch.Generator(device="cuda").manual_seed(tokens)
    gu = (torch.randn(tokens, 2 * inter, device="cuda", generator=g) * 4).to(dtype)
    dout = torch.randn(tokens, inter, device="cuda", generator=g).to(dtype)
    act = torch.full((tokens, inter), float("nan"), device="cuda", dtype=dtype)
    dgu = T.gated_act_bwd(dout, gu, "silu", act_out=act)
    assert_bits_equal(act, T.gated_act_fwd_raw(gu), "act")
    assert_bits_equal(dgu, T.gated_act_bwd(dout, gu, "silu"), "dgate_up")


@pytest.mark.parametrize("backend", ["own", "lib"], indirect=True)
def test_down_dx_dswiglu_act_out(backend):
    """Either dSwiGLU path hands back the library path's forward ``act``; the gradient is the one without ``act_out``."""
    Tn, H, I = 512, 384, 1280
    g = torch.Generator(device="cuda").manual_seed(3)
    gu = (torch.randn(Tn, 2 * I, device="cuda", generator=g) * 2).bfloat16()
    dy = torch.randn(Tn, H, device="cuda", generator=g).bfloat16()
    w_down = (torch.randn(H, I, device="cuda", generator=g) / I**0.5).bfloat16()
    act = torch.full((Tn, I), float("nan"), device="cuda", dtype=torch.bfloat16)
    dgu = gemm.down_dx_dswiglu(dy, w_down, gu, act_out=act)
    assert gemm.tuning_table().get(f"nn_dswiglu:{Tn}x{I}x{H}", "lib") == backend
    assert_bits_equal(act, T.gated_act_fwd_raw(gu), "act")
    assert_bits_equal(dgu, gemm.down_dx_dswiglu(dy, w_down, gu), "dgate_up")


MODELS = {
    "tiny": dict(hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2),
    "3b-width": dict(hidden_size=3072, intermediate_size=8192, num_attention_heads=24, num_key_value_heads=8),
}
INPUTS = {
    "dense": {},
    "packed": {"cu": torch.tensor([0, 100, 256, 300, 301, 512], dtype=torch.int32)},
    "window": {"sliding_window": 64},
}


def _model(name, **kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", vocab_size=1024, num_hidden_layers=2, attention_backend="native", **MODELS[name], **kw)
    with torch.device("cuda"):
        return LlamaForCausalLM(cfg).to(torch.bfloat16)


def _loss_and_grads(model, ids, cu):
    model.train()
    loss = model(ids, labels=ids, cu_seqlens=cu)
    loss.backward()
    return loss.detach(), {n: p.grad for n, p in model.named_parameters()}


@pytest.mark.parametrize("backend", ["lib", "own"], indirect=True)
@pytest.mark.parametrize("inputs", sorted(INPUTS))
@pytest.mark.parametrize("layers", [0, 1, 2])
@pytest.mark.parametrize("name", sorted(MODELS))
def test_trimmed_replay_matches_whole_replay(name, layers, inputs, backend, monkeypatch):
    """On the in-tree path the fused gate|up kernel's ``act`` is saved (and recomputed by the same kernel in the replay),
    so that path is bit-equal as well."""
    kw = dict(INPUTS[inputs])
    cu = kw.pop("cu", None)
    ids = torch.randint(0, 1024, (2, 256), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    got_loss, got = _loss_and_grads(_model(name, checkpoint_layers=layers, **kw), ids, cu)
    whole = ckpt.checkpoint
    monkeypatch.setattr(ckpt, "checkpoint", lambda fn, *args, replay=None: whole(fn, *args))
    want_loss, want = _loss_and_grads(_model(name, checkpoint_layers=layers, **kw), ids, cu)
    assert_bits_equal(got_loss, want_loss, "loss")
    for n in want:
        assert_bits_equal(got[n], want[n], n)
    I, H = MODELS[name]["intermediate_size"], MODELS[name]["hidden_size"]
    assert gemm.tuning_table().get(f"nt_swiglu:512x{I}x{H}", "lib") == backend


@pytest.mark.parametrize("backend", ["lib"], indirect=True)
def test_replay_launches_no_down_gemm_and_no_swiglu_kernel(backend, monkeypatch):
    """Backward of the 3B-width model with both layers checkpointed: no ``gated_act_fwd_kernel`` and no down-projection
    product; one ``gated_act_bwd_kernel`` per layer (it writes ``act``)."""
    from torch.profiler import ProfilerActivity, profile
    model = _model("3b-width", checkpoint_layers=2)
    H, I = 3072, 8192
    ids = torch.randint(0, 1024, (2, 256), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    model.train()
    loss = model(ids, labels=ids)
    products = []
    real_nt = gemm.matmul_nt
    monkeypatch.setattr(gemm, "matmul_nt", lambda a, b, out=None: products.append((b.shape[0], a.shape[1])) or
                        real_nt(a, b, out))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loss.backward()
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert not any("gated_act_fwd_kernel" in k for k in kernels), kernels
    assert sum("gated_act_bwd_kernel" in k for k in kernels) == 2, kernels
    assert products.count((H, I)) == 0 and products.count((2 * I, H)) == 2, products


def _zero3_steps(trimmed, steps=3):
    import deepspeed_b200 as ds
    from deepspeed_b200.utils.tensor_fragment import safe_get_full_fp32_param
    whole = ckpt.checkpoint
    if not trimmed:
        ckpt.checkpoint = lambda fn, *args, replay=None: whole(fn, *args)
    try:
        engine, _, _, _ = ds.initialize(model=_model("3b-width", checkpoint_layers=1), config={
            "train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
            "optimizer": {"type": "AdamW", "params": {"lr": 1e-4}}, "zero_optimization": {"stage": 3}})
        ids = torch.randint(0, 1024, (2, 256), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        losses = []
        for _ in range(steps):
            loss = engine(ids, labels=ids)
            engine.backward(loss)
            engine.step()
            losses.append(loss.detach().float())
        params = [safe_get_full_fp32_param(p).detach().clone() for p in engine.module.parameters()]
    finally:
        ckpt.checkpoint = whole
    return torch.stack(losses), params


def _zero3_trimmed_vs_whole():
    got_losses, got = _zero3_steps(True)
    want_losses, want = _zero3_steps(False)
    assert_bits_equal(got_losses, want_losses, "losses")
    for i, (a, b) in enumerate(zip(got, want)):
        assert_bits_equal(a, b, f"param {i}")


def test_zero3_engine_trimmed_replay_matches_whole_replay():
    """Under the ZeRO-3 bf16 engine (gathered weights, gradients straight into the flat buffers, the step fused into
    backward), in a fresh process: three steps give the same losses and fp32 master weights bit for bit."""
    from tests.common import run_distributed
    run_distributed(_zero3_trimmed_vs_whole, 1, ())
