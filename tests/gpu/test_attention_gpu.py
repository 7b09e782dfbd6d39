"""GPU tier: the wgmma training attention kernel against float64 with the per-element bounds of
:func:`tests.numerics.attention_bounds`."""
import pytest
import torch

from tests.numerics import assert_attention_bounded

pytestmark = pytest.mark.gpu


def _heads(qkv, hq, hkv, d):
    """[T, hq, d], [T, hkv, d], [T, hkv, d] views of a packed projection output."""
    T = qkv.shape[0]
    return qkv[:, :hq * d].view(T, hq, d), qkv[:, hq * d:(hq + hkv) * d].view(T, hkv, d), qkv[:, (hq + hkv) * d:].view(T, hkv, d)


def _seqs(B, S):
    return None if B == 1 else [b * S for b in range(B + 1)]


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
    assert_attention_bounded({"o": o.view(B * S, hq, d), "lse": lse.permute(1, 0, 2).reshape(hq, B * S)},
                             *_heads(qkv, hq, hkv, d), None, _seqs(B, S), causal)
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
    assert torch.isfinite(dqkv.float()).all()
    gq, gk, gv = _heads(dqkv, hq, hkv, d)
    assert_attention_bounded({"o": o.view(B * S, hq, d), "lse": lse.permute(1, 0, 2).reshape(hq, B * S), "dq": gq,
                              "dk": gk, "dv": gv}, *_heads(qkv, hq, hkv, d), d_o.view(B * S, hq, d), _seqs(B, S), causal)


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
    assert_attention_bounded({"o": out[:S].view(S, hq, d)}, *_heads(qkv, hq, hkv, d), None, None, causal)
    assert float((out[S:].float() - 7.0).abs().max()) == 0.0  # rows past the sequence are never written
