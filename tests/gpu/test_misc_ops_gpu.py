"""sm_90a kernels of misc.cu / moe_ragged.cu vs their host (plain PyTorch fp32) definitions (quant.cu: test_quant_exact_gpu.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_attn_softmax_fwd_bwd(dtype):
    from deepspeed_b200.ops.kernels import misc_ops as K
    torch.manual_seed(0)
    s = torch.randn(2, 4, 16, 48)
    mask = torch.zeros(2, 1, 1, 48)
    mask[:, :, :, -7:] = -10000.0
    alibi = torch.tensor([0.5, 0.25, 0.125, 0.0625])
    for kw in (dict(causal=True), dict(mask=mask), dict(causal=True, alibi=alibi), dict(causal=True, window=8)):
        h = s.clone().requires_grad_(True)
        d = s.to(dtype).cuda().requires_grad_(True)
        kw_d = {k: (v.to(dtype).cuda() if k == "mask" else (v.cuda() if torch.is_tensor(v) else v)) for k, v in kw.items()}
        ph = K.attn_softmax(h, scale=0.3, **kw)
        pd = K.attn_softmax(d, scale=0.3, **kw_d)
        tol = 1e-5 if dtype == torch.float32 else 2e-2
        torch.testing.assert_close(pd.float().cpu(), ph, atol=tol, rtol=tol)
        g = torch.randn_like(ph)
        ph.backward(g)
        pd.backward(g.to(dtype).cuda())
        torch.testing.assert_close(d.grad.float().cpu(), h.grad, atol=tol, rtol=tol)


def test_dropout_statistics_and_backward_mask():
    from deepspeed_b200.ops.kernels import misc_ops as K
    x = torch.ones(4096, 64, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    bias = torch.zeros(64, device="cuda", dtype=torch.bfloat16)
    res = torch.full((4096, 64), 2.0, device="cuda", dtype=torch.bfloat16)
    y = K.dropout(x, 0.25, training=True, bias=bias, residual=res, seed=11)
    kept = (y != 2.0)
    assert abs(kept.float().mean().item() - 0.75) < 0.01
    torch.testing.assert_close(y[kept].float(), torch.full_like(y[kept].float(), 2.0 + 1 / 0.75), atol=2e-2, rtol=2e-2)
    y.backward(torch.ones_like(y))
    # backward regenerates exactly the forward mask
    assert torch.equal(x.grad != 0, kept)
    y2 = K.dropout(x.detach(), 0.25, training=True, seed=11)
    assert (y2 != 0).float().mean().item() == pytest.approx(0.75, abs=0.01)


def test_transforms_token_ops_nhwc():
    from deepspeed_b200.ops.kernels import misc_ops as K
    torch.manual_seed(0)
    x = torch.randn(2, 7, 3, 4, 16).bfloat16()
    b = torch.randn(3 * 4 * 16).bfloat16()
    torch.testing.assert_close(K.bias_transform_0213(x.cuda(), b.cuda(), 2, 7, 3, 4, 16).cpu().float(),
                               K.bias_transform_0213(x, b, 2, 7, 3, 4, 16).float(), atol=2e-2, rtol=2e-2)
    t = torch.randn(2, 4, 9, 16).half()
    assert torch.equal(K.transform4d_0213(t.cuda()).cpu(), K.transform4d_0213(t))
    idx = torch.stack([torch.randperm(64)[:20] for _ in range(6)]).to(torch.int32)
    assert torch.equal(K.token_sort_(idx.clone().cuda()).cpu(), idx.sort(-1).values)
    h = torch.randn(3, 64, 32).bfloat16()
    sidx = torch.stack([torch.randperm(64)[:20].sort().values for _ in range(3)]).to(torch.int32)
    g = K.token_gather(h.cuda(), sidx.cuda())
    assert torch.equal(g.cpu(), K.token_gather(h, sidx))
    full = torch.zeros(3, 64, 32).bfloat16()
    assert torch.equal(K.token_scatter_(full.clone().cuda(), g, sidx.cuda()).cpu(), K.token_scatter_(full.clone(), g.cpu(), sidx))
    m = torch.randn(3, 1, 64, 64).bfloat16()
    assert torch.equal(K.mask_gather(m.cuda(), sidx.cuda()).cpu(), K.mask_gather(m, sidx))
    a, o = torch.randn(2, 8, 8, 32).half(), torch.randn(2, 8, 8, 32).half()
    bb, ob = torch.randn(32).half(), torch.randn(32).half()
    torch.testing.assert_close(K.nhwc_bias_add(a.cuda(), bb.cuda(), o.cuda(), ob.cuda()).cpu(), a + bb + o + ob, atol=2e-2,
                               rtol=2e-2)


def test_training_transformer_layer_and_sparse_attention_on_device():
    from deepspeed_b200.ops.sparse_attention import FixedSparsityConfig, SparseSelfAttention
    from deepspeed_b200.ops.transformer import DeepSpeedTransformerConfig, DeepSpeedTransformerLayer
    torch.manual_seed(0)
    cfg = DeepSpeedTransformerConfig(batch_size=2, hidden_size=256, heads=4, attn_dropout_ratio=0.0, hidden_dropout_ratio=0.0,
                                     num_hidden_layers=2, initializer_range=0.02, bf16=True)
    layer = DeepSpeedTransformerLayer(cfg)
    ref = layer.float()
    x = torch.randn(2, 64, 256)
    want = ref(x)
    got = DeepSpeedTransformerLayer(cfg)
    got.load_state_dict(ref.state_dict())
    got = got.cuda().bfloat16()
    out = got(x.cuda().bfloat16())
    assert torch.nn.functional.cosine_similarity(out.float().cpu().flatten(), want.flatten(), dim=0) > 0.999
    out.float().sum().backward()
    att = SparseSelfAttention(FixedSparsityConfig(4, 16, num_local_blocks=2), max_seq_length=128).cuda()
    q = torch.randn(2, 4, 128, 32, device="cuda", dtype=torch.bfloat16)
    y = att(q, q, q)
    assert y.shape == q.shape and torch.isfinite(y.float()).all()


def test_evoformer_attention_device():
    from deepspeed_b200.ops.deepspeed4science import DS4Sci_EvoformerAttention
    torch.manual_seed(0)
    q, k, v = (torch.randn(1, 8, 64, 4, 32, device="cuda", dtype=torch.bfloat16, requires_grad=True) for _ in range(3))
    mask = torch.zeros(1, 8, 1, 1, 64, device="cuda", dtype=torch.bfloat16)
    pair = torch.randn(1, 1, 4, 64, 64, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    out = DS4Sci_EvoformerAttention(q, k, v, [mask, pair])
    qt, kt, vt = (t.float().transpose(-2, -3) for t in (q, k, v))
    ref = (torch.softmax(qt @ kt.transpose(-1, -2) / 32**0.5 + mask.float() + pair.float(), -1) @ vt).transpose(-2, -3)
    assert torch.nn.functional.cosine_similarity(out.float().flatten(), ref.flatten(), dim=0) > 0.999
    out.float().sum().backward()
    assert pair.grad is not None and torch.isfinite(pair.grad.float()).all()


def test_onebit_pack_unpack_kernels_match_torch_path():
    """1-bit compression kernels (sign pack + error feedback, fused unpack + average) vs the torch reference path."""
    import torch
    from deepspeed_b200.runtime.comm import compressed as C
    torch.manual_seed(0)
    n = 8 * 4096 + 8 * 3
    work = torch.randn(n, device="cuda")
    err = torch.empty(n, device="cuda")
    packed, scale = C.compress_with_feedback(work.clone(), err)
    ref_packed = C.pack_signs(work)
    ref_scale = work.norm() / n**0.5
    assert torch.equal(packed, ref_packed) and abs(float(scale - ref_scale)) < 1e-6
    torch.testing.assert_close(err, work - ref_scale * C.unpack_signs(ref_packed))
    R = 4
    pk = torch.stack([C.pack_signs(torch.randn(n, device="cuda")) for _ in range(R)])
    sc = torch.rand(R, device="cuda") + 0.5
    got = C.decompress_average(pk, sc, n)
    ref = (C.unpack_signs(pk.reshape(-1)).view(R, n) * sc.view(R, 1)).sum(0) / R
    torch.testing.assert_close(got, ref, atol=1e-6, rtol=1e-5)
    # single-rank backend round trip through the kernels
    be = C.CompressedBackend(group=None) if torch.distributed.is_initialized() else None
