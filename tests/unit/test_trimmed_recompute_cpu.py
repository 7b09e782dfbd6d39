"""Activation-checkpointed Llama layers replay their forward only as far as backward reads (CPU tier): no down-projection
GEMM and no SwiGLU pass in the replay, ``act`` for the down weight gradient written by the dSwiGLU pass, and the same
loss and gradients, bit for bit, as the replay of the whole layer."""
import pytest
import torch

from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
from deepspeed_b200.ops import gemm
from deepspeed_b200.ops.kernels import transformer_ops as T
from deepspeed_b200.runtime.activation_checkpointing import checkpointing as ckpt
from tests.common import run_distributed


def _tiny(**kw):
    torch.manual_seed(0)
    cfg = llama_config("tiny", vocab_size=97, hidden_size=64, intermediate_size=96, num_attention_heads=4,
                       num_key_value_heads=2, **kw)
    return LlamaForCausalLM(cfg)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_dswiglu_act_out_equals_forward(dtype):
    g = torch.Generator().manual_seed(0)
    gu = (torch.randn(37, 2 * 48, generator=g) * 3).to(dtype)
    dout = torch.randn(37, 48, generator=g).to(dtype)
    act = torch.full((37, 48), float("nan"), dtype=dtype)
    dgu = T.gated_act_bwd(dout, gu, "silu", act_out=act)
    assert torch.equal(act, T.gated_act_fwd_raw(gu))
    assert torch.equal(dgu, T.gated_act_bwd(dout, gu, "silu"))


def _untrimmed(monkeypatch):
    """Make every checkpointed layer replay its whole forward (the generic checkpoint)."""
    whole = ckpt.checkpoint
    monkeypatch.setattr(ckpt, "checkpoint", lambda fn, *args, replay=None: whole(fn, *args))


def _run(model, ids, cu=None):
    model.train()
    loss = model(ids, labels=ids, cu_seqlens=cu)
    loss.backward()
    return loss.detach(), {n: p.grad.clone() for n, p in model.named_parameters()}


INPUTS = {
    "dense": {},
    "packed": {"cu": torch.tensor([0, 7, 24, 30, 48], dtype=torch.int32)},
    "window": {"sliding_window": 5},
}


@pytest.mark.parametrize("inputs", sorted(INPUTS))
@pytest.mark.parametrize("layers", [0, 1, 2])
def test_trimmed_replay_matches_whole_replay(inputs, layers, monkeypatch):
    """Loss and every parameter gradient with ``checkpoint_layers`` 0, 1 and all equal, bit for bit, the whole-layer
    replay of all layers (which itself equals no recompute)."""
    kw = dict(INPUTS[inputs])
    cu = kw.pop("cu", None)
    ids = torch.randint(0, 97, (2, 24), generator=torch.Generator().manual_seed(1))
    got_loss, got = _run(_tiny(checkpoint_layers=layers, **kw), ids, cu)
    with monkeypatch.context() as m:
        _untrimmed(m)
        want_loss, want = _run(_tiny(checkpoint_layers=2, **kw), ids, cu)
    assert torch.equal(got_loss, want_loss)
    for n in want:
        assert torch.equal(got[n], want[n]), n


def test_fp8_layers_replay_whole(monkeypatch):
    """The FP8 MLP node has no trimmed replay: its checkpointed layers take the generic one."""
    seen = []
    whole = ckpt.checkpoint
    monkeypatch.setattr(ckpt, "checkpoint", lambda fn, *args, replay=None: seen.append(replay) or whole(fn, *args))
    model = _tiny(checkpoint_layers=2, fp8=True)
    assert not model.model.layers[0].mlp.trimmed_recompute
    _run(model, torch.randint(0, 97, (2, 32), generator=torch.Generator().manual_seed(1)))
    assert seen == [None, None]


def test_replay_runs_no_down_gemm_and_no_swiglu_pass(monkeypatch):
    """Backward of a fully checkpointed model: the replays run the gate|up GEMM but no down-projection GEMM and no
    forward SwiGLU pass; the dSwiGLU pass writes ``act`` once per layer."""
    model = _tiny(checkpoint_layers=2)
    H, I = model.cfg.hidden_size, model.cfg.intermediate_size
    nt, fwd_act, bwd_act = [], [], []
    real_nt, real_fwd, real_bwd = gemm.matmul_nt, T.gated_act_fwd_raw, T.gated_act_bwd
    monkeypatch.setattr(gemm, "matmul_nt", lambda a, b, out=None: nt.append((b.shape[0], a.shape[1])) or real_nt(a, b, out))
    monkeypatch.setattr(T, "gated_act_fwd_raw", lambda *a, **k: fwd_act.append(1) or real_fwd(*a, **k))
    monkeypatch.setattr(T, "gated_act_bwd", lambda *a, **k: bwd_act.append(k.get("act_out") is not None) or real_bwd(*a, **k))
    model.train()
    loss = model(torch.randint(0, 97, (2, 24), generator=torch.Generator().manual_seed(1)), labels=None)
    assert (nt.count((H, I)), nt.count((2 * I, H)), len(fwd_act)) == (2, 2, 2)  # forward: both layers in full
    nt.clear(), fwd_act.clear()
    loss.float().sum().backward()
    assert nt.count((H, I)) == 0 and len(fwd_act) == 0, (nt, fwd_act)
    assert nt.count((2 * I, H)) == 2 and bwd_act == [True, True]


def test_mlp_node_saves_input_and_gate_up_only():
    """On the library path the MLP node keeps ``x`` and gate|up for backward, not ``act``."""
    from deepspeed_b200.ops.linear import swiglu_mlp
    x = torch.randn(8, 16, requires_grad=True)
    w_gu, w_down = torch.randn(48, 16, requires_grad=True), torch.randn(16, 24, requires_grad=True)
    saved = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append(tuple(t.shape)) or t, lambda t: t):
        y = swiglu_mlp(x, w_gu, w_down)
    assert sorted(saved) == [(8, 16), (8, 48)]
    y.sum().backward()
    xr, gr, dr = (t.detach().clone().requires_grad_(True) for t in (x, w_gu, w_down))
    gu = xr @ gr.t()
    (torch.nn.functional.silu(gu[:, :24]) * gu[:, 24:] @ dr.t()).sum().backward()
    for got, want in ((x.grad, xr.grad), (w_gu.grad, gr.grad), (w_down.grad, dr.grad)):
        torch.testing.assert_close(got, want)


def _zero3_trimmed_vs_whole():
    import deepspeed_b200 as ds
    conf = {"train_micro_batch_size_per_gpu": 2, "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
            "zero_optimization": {"stage": 3}}
    ids = torch.randint(0, 97, (2, 24), generator=torch.Generator().manual_seed(4))
    runs = []
    whole = ckpt.checkpoint
    for trimmed in (True, False):
        if not trimmed:
            ckpt.checkpoint = lambda fn, *args, replay=None: whole(fn, *args)
        try:
            eng, _, _, _ = ds.initialize(model=_tiny(checkpoint_layers=1), config=conf)
            losses = []
            for _ in range(3):
                loss = eng(ids, labels=ids)
                eng.backward(loss)
                eng.step()
                losses.append(loss.detach())
        finally:
            ckpt.checkpoint = whole
        from deepspeed_b200.utils.tensor_fragment import safe_get_full_fp32_param
        runs.append((losses, [safe_get_full_fp32_param(p).clone() for p in eng.module.parameters()]))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0])), runs
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


def test_zero3_engine_trimmed_replay_matches_whole_replay():
    run_distributed(_zero3_trimmed_vs_whole, 1, ())
