"""GPU tier: the wgmma training attention kernel against an fp32 reference."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(q, k, v, causal):
    """fp32 reference: q [B, hq, S, d], k/v [B, hkv, S, d]."""
    B, hq, S, d = q.shape
    rep = hq // k.shape[1]
    k, v = k.repeat_interleave(rep, 1), v.repeat_interleave(rep, 1)
    s = (q.float() @ k.float().transpose(-1, -2)) / math.sqrt(d)
    if causal:
        s = s.masked_fill(torch.triu(torch.ones(S, S, dtype=torch.bool, device=q.device), 1), float("-inf"))
    return torch.softmax(s, -1) @ v.float(), torch.logsumexp(s, -1)


@pytest.mark.parametrize("B,S,hq,hkv,causal", [(1, 128, 1, 1, True), (1, 256, 2, 1, True), (2, 512, 4, 2, True),
                                               (1, 384, 4, 4, False), (1, 1024, 8, 2, True)])
def test_attn_fwd_matches_fp32(B, S, hq, hkv, causal):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    torch.manual_seed(S + hq)
    d = 128
    qkv = torch.randn(B * S, (hq + 2 * hkv) * d, device="cuda", dtype=torch.bfloat16)
    q2, k2, v2 = A.split_packed(qkv, hq, hkv)
    assert A.supports(qkv, hq, hkv, d, S)
    o, lse = A.fwd(q2, k2, v2, B, S, hq, hkv, causal=causal)
    torch.cuda.synchronize()
    x = qkv.view(B, S, hq + 2 * hkv, d)
    ref_o, ref_lse = _ref(x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2),
                          x[:, :, hq + hkv:].transpose(1, 2), causal)
    got = o.view(B, S, hq, d).transpose(1, 2).float()
    assert torch.isfinite(got).all()
    assert (got - ref_o).abs().max().item() < 2e-2, (got - ref_o).abs().max().item()
    assert (lse - ref_lse).abs().max().item() < 2e-2
    # repeated launches: barrier phases / registers reuse stay correct
    o2, _ = A.fwd(q2, k2, v2, B, S, hq, hkv, causal=causal)
    assert torch.equal(o, o2)


@pytest.mark.parametrize("B,S,hq,hkv,causal", [(1, 128, 1, 1, True), (1, 256, 2, 1, True), (2, 512, 4, 2, True),
                                               (1, 384, 4, 4, False), (1, 1024, 8, 2, True)])
def test_attn_bwd_matches_fp32(B, S, hq, hkv, causal):
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    torch.manual_seed(S + hq)
    d = 128
    qkv = (torch.randn(B * S, (hq + 2 * hkv) * d, device="cuda") * 0.7).to(torch.bfloat16)
    q2, k2, v2 = A.split_packed(qkv, hq, hkv)
    o, lse = A.fwd(q2, k2, v2, B, S, hq, hkv, causal=causal)
    d_o = torch.randn_like(o)
    dqkv = torch.full_like(qkv, float("nan"))
    dq, dk, dv = A.split_packed(dqkv, hq, hkv)
    A.bwd(d_o, q2, k2, v2, o, lse, B, S, hq, hkv, causal=causal, dq=dq, dk=dk, dv=dv)
    torch.cuda.synchronize()
    x = qkv.view(B, S, hq + 2 * hkv, d)
    qr, kr, vr = (t.transpose(1, 2).float().detach().requires_grad_(True)
                  for t in (x[:, :, :hq], x[:, :, hq:hq + hkv], x[:, :, hq + hkv:]))
    ref_o, _ = _ref(qr, kr, vr, causal)
    ref_o.backward(d_o.view(B, S, hq, d).transpose(1, 2).float())
    g = dqkv.view(B, S, hq + 2 * hkv, d)
    assert torch.isfinite(dqkv.float()).all()
    for name, got, ref in (("dq", g[:, :, :hq], qr.grad), ("dk", g[:, :, hq:hq + hkv], kr.grad), ("dv", g[:, :, hq + hkv:], vr.grad)):
        got = got.transpose(1, 2).float()
        cos = torch.nn.functional.cosine_similarity(got.flatten(), ref.flatten(), dim=0).item()
        err = (got - ref).abs().max().item()
        assert cos > 0.999 and err < 3e-2 * ref.abs().max().item() + 2e-2, (name, cos, err, ref.abs().max().item())


def test_packed_attention_autograd_with_rope_matches_sdpa_path():
    """The native kernel inside the model's packed-QKV attention op (in-place RoPE, packed dqkv) vs the cuDNN/SDPA path."""
    from deepspeed_b200.ops.attention import causal_attention
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    torch.manual_seed(0)
    B, S, hq, hkv, d = 2, 256, 4, 2, 128
    rope = RotaryTable(d, 512, 10000.0, "cuda")
    base = (torch.randn(B * S, (hq + 2 * hkv) * d, device="cuda") * 0.5).to(torch.bfloat16)
    outs = {}
    for backend in ("native", "cudnn"):
        qkv = base.clone().requires_grad_(True)
        y = causal_attention(qkv * 1.0, B, S, hq, hkv, d, rope, None, backend=backend)
        gy = torch.randn(B * S, hq * d, device="cuda", dtype=torch.bfloat16, generator=torch.Generator(device="cuda").manual_seed(1))
        y.backward(gy)
        outs[backend] = (y.detach().float(), qkv.grad.float())
    assert (outs["native"][0] - outs["cudnn"][0]).abs().max().item() < 3e-2
    ga, gb = outs["native"][1], outs["cudnn"][1]
    assert torch.nn.functional.cosine_similarity(ga.flatten(), gb.flatten(), dim=0).item() > 0.999


@pytest.mark.parametrize("S,causal", [(200, True), (77, True), (333, False), (129, True)])
def test_attn_fwd_ragged_length(S, causal):
    """Serving prompts: any length with one sequence per launch (ragged last block masked in the kernel, TMA zero-fills
    rows past the end)."""
    from deepspeed_b200.ops.kernels import attention_sm100 as A
    torch.manual_seed(S)
    hq, hkv, d = 4, 2, 128
    qkv = torch.randn(S, (hq + 2 * hkv) * d, device="cuda", dtype=torch.bfloat16)
    q2, k2, v2 = A.split_packed(qkv, hq, hkv)
    assert A.supports_fwd(qkv, hq, hkv, d, 1, S)
    out = torch.full((S + 3, hq * d), 7.0, device="cuda", dtype=torch.bfloat16)
    A.fwd(q2, k2, v2, 1, S, hq, hkv, causal=causal, out=out[:S], need_lse=False)
    x = qkv.view(1, S, hq + 2 * hkv, d)
    ref_o, _ = _ref(x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2), x[:, :, hq + hkv:].transpose(1, 2),
                    causal)
    got = out[:S].view(1, S, hq, d).transpose(1, 2).float()
    assert torch.isfinite(got).all()
    assert (got - ref_o).abs().max().item() < 2e-2
    assert float((out[S:].float() - 7.0).abs().max()) == 0.0  # rows past the sequence are never written
