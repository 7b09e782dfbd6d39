"""FPDT chunked attention on the GPU: native per-pair kernels (wgmma for head dim 128, register-accumulator kernels for
head dim 64) + the double-buffered host offload of q / k / v / o chunks, against dense SDPA."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _dense(x, w1, w2, heads, kv_heads, d):
    S, B, _ = x.shape
    qkv = torch.nn.functional.linear(x, w1)
    q, k, v = torch.split(qkv, [heads * d, kv_heads * d, kv_heads * d], dim=-1)
    q, k, v = q.reshape(S, B, heads, d), k.reshape(S, B, kv_heads, d), v.reshape(S, B, kv_heads, d)
    rep = heads // kv_heads
    k, v = k.repeat_interleave(rep, dim=2), v.repeat_interleave(rep, dim=2)
    q, k, v = (t.permute(1, 2, 0, 3) for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True).permute(2, 0, 1, 3).reshape(S, B, heads * d)
    return torch.nn.functional.linear(o, w2)


@pytest.mark.parametrize("d,heads,kv_heads,offload", [(128, 4, 2, True), (128, 4, 4, False), (64, 8, 4, True)])
def test_fpdt_attention_native_pairs(d, heads, kv_heads, offload):
    from deepspeed_b200.ops import native as N
    from deepspeed_b200.sequence import fpdt_layer as FP
    torch.manual_seed(0)
    S, B = 1024, 2
    Hd = heads * d
    w1 = (torch.randn((heads + 2 * kv_heads) * d, Hd, device="cuda") * Hd**-0.5).bfloat16().requires_grad_(True)
    w2 = (torch.randn(Hd, Hd, device="cuda") * Hd**-0.5).bfloat16()
    attn = FP.FPDT_Attention(first_weight=w1, second_weight=w2, chunk_size=256, enable_offloading=offload, num_heads=heads,
                             num_kv_heads=kv_heads, head_dim=d, return_bias=False)
    x = torch.randn(S, B, Hd, device="cuda").bfloat16().requires_grad_(True)
    g = torch.randn(S, B, Hd, device="cuda").bfloat16()
    n0 = N.launch_count
    y = attn(x)
    y.backward(g)
    assert N.launch_count > n0 + 10, "per-pair attention must run on the native kernels"
    got = (y.detach().float(), x.grad.float().clone(), w1.grad.float().clone())
    x.grad = w1.grad = None
    ref = _dense(x, w1, w2, heads, kv_heads, d)
    ref.backward(g)
    for a, b, nm in zip(got, (ref.detach().float(), x.grad.float(), w1.grad.float()), ("y", "dx", "dw")):
        err = (a - b).abs().max().item()
        assert err <= 3e-2 * b.abs().max().item() + 1e-3, f"{nm}: {err} vs {b.abs().max().item()}"


def test_chunk_store_round_trip_is_stream_ordered():
    from deepspeed_b200.sequence.fpdt_layer import _ChunkStore
    st = _ChunkStore(True, torch.device("cuda", 0))
    ts = [torch.randn(1 << 20, device="cuda") for _ in range(6)]
    for i, t in enumerate(ts):
        st.put(i, t.clone())
    assert st.bytes_offloaded == 6 * 4 * (1 << 20) and not st.dev
    for i in range(6):
        if i + 1 < 6:
            st.prefetch(i + 1)
        torch.testing.assert_close(st.get(i), ts[i])
        st.release(i)


@pytest.mark.parametrize("d,hq,hkv", [(128, 4, 2), (64, 4, 4)])
def test_ring_attention_block_kernels_single_rank(d, hq, hkv):
    """The ring-attention autograd function on its native pair kernels (one rank = one hop, the diagonal causal block):
    forward and dQ / dK / dV against SDPA."""
    import deepspeed_b200 as ds
    from deepspeed_b200.ops import native as N
    from deepspeed_b200.sequence.ring_attention import _RingAttention
    ds.init_distributed(verbose=False)
    torch.manual_seed(0)
    B, S = 2, 512
    q = torch.randn(B, hq, S, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    k = torch.randn(B, hkv, S, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    v = torch.randn(B, hkv, S, d, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    g = torch.randn(B, hq, S, d, device="cuda", dtype=torch.bfloat16)
    n0 = N.launch_count
    out = _RingAttention.apply(q, k, v, None, True, None)
    out.backward(g)
    assert N.launch_count >= n0 + 2
    got = [t.float().clone() for t in (out.detach(), q.grad, k.grad, v.grad)]
    q.grad = k.grad = v.grad = None
    rep = hq // hkv
    ref = torch.nn.functional.scaled_dot_product_attention(q, k.repeat_interleave(rep, 1), v.repeat_interleave(rep, 1), is_causal=True)
    ref.backward(g)
    for a, b, nm in zip(got, (ref.detach(), q.grad, k.grad, v.grad), ("out", "dq", "dk", "dv")):
        err = (a - b.float()).abs().max().item()
        assert err <= 3e-2 * b.float().abs().max().item() + 1e-3, (nm, err)
