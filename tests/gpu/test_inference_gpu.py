"""Ragged inference kernels + engine on an H100: device kernels vs their host definitions, engine vs HF."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(T=37, hq=8, hkv=2, d=64, bs=16, dtype=torch.bfloat16, seqs=3):
    from deepspeed_b200.ops.kernels.transformer_ops import RotaryTable
    g = torch.Generator().manual_seed(0)
    lens = [T - 2 * (seqs - 1)] + [2] * (seqs - 1)
    seen = [0, 5, 40][:seqs]
    seq_of = torch.cat([torch.full((n, ), i, dtype=torch.int32) for i, n in enumerate(lens)])
    pos_of = torch.cat([torch.arange(s, s + n, dtype=torch.int32) for s, n in zip(seen, lens)])
    max_blocks = 8
    perm = torch.randperm(seqs * max_blocks, generator=g).to(torch.int32).view(seqs, max_blocks)
    qkv = torch.randn(T, (hq + 2 * hkv) * d, generator=g).to(dtype)
    cache = torch.randn(seqs * max_blocks, bs, 2, hkv, d, generator=g).to(dtype)
    rope = RotaryTable(d, 256)
    return qkv, cache, rope, seq_of, pos_of, perm, (hq, hkv, d, bs)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_kv_append_and_paged_attention(dtype):
    from deepspeed_b200.ops.kernels import ragged_ops as R
    qkv, cache, rope, seq_of, pos_of, bt, (hq, hkv, d, bs) = _mk(dtype=dtype)
    q_h, c_h = qkv.clone(), cache.clone()
    R.kv_rotary_append(q_h, c_h, rope.cos, rope.sin, seq_of, pos_of, bt, hq, hkv, d, d, bs)
    o_h = R.paged_attention(q_h, c_h, seq_of, pos_of, bt, hq, hkv, d, bs)
    dev = "cuda"
    q_d, c_d = qkv.to(dev), cache.to(dev)
    R.kv_rotary_append(q_d, c_d, rope.cos.to(dev), rope.sin.to(dev), seq_of.to(dev), pos_of.to(dev), bt.to(dev), hq, hkv, d,
                       d, bs)
    o_d = R.paged_attention(q_d, c_d, seq_of.to(dev), pos_of.to(dev), bt.to(dev), hq, hkv, d, bs)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    torch.testing.assert_close(q_d.cpu().float(), q_h.float(), atol=tol, rtol=tol)
    torch.testing.assert_close(c_d.cpu().float(), c_h.float(), atol=tol, rtol=tol)
    torch.testing.assert_close(o_d.cpu().float(), o_h.float(), atol=tol, rtol=tol)


@pytest.mark.parametrize("hq,hkv,d", [(32, 8, 128), (8, 8, 64), (16, 2, 128), (14, 2, 64)])
def test_paged_decode_split_kv_long_context(hq, hkv, d):
    """Decode-shaped batch (1 token per sequence, long contexts): the split-KV / GQA-shared kernel (or the generic
    fallback for the 14/2 head ratio) must match the plain fp32 definition."""
    from deepspeed_b200.ops.kernels import ragged_ops as R
    torch.manual_seed(0)
    bs, seqs, nb = 128, 5, 12
    ctx = [1500, 17, 1024, 129, 1536]
    qkv = (torch.randn(seqs, (hq + 2 * hkv) * d) * 0.5).bfloat16()
    cache = (torch.randn(seqs * nb, bs, 2, hkv, d) * 0.5).bfloat16()
    bt = torch.randperm(seqs * nb).to(torch.int32).view(seqs, nb)
    seq_of = torch.arange(seqs, dtype=torch.int32)
    pos_of = torch.tensor([c - 1 for c in ctx], dtype=torch.int32)
    ref = R.paged_attention(qkv.float(), cache.float(), seq_of, pos_of, bt, hq, hkv, d, bs)
    dev = "cuda"
    got = R.paged_attention(qkv.to(dev), cache.to(dev), seq_of.to(dev), pos_of.to(dev), bt.to(dev), hq, hkv, d, bs)
    torch.testing.assert_close(got.float().cpu(), ref, atol=2e-2, rtol=2e-2)


def test_embed_and_row_gather():
    from deepspeed_b200.ops.kernels import ragged_ops as R
    wte = torch.randn(100, 64).bfloat16()
    wpe = torch.randn(50, 64).bfloat16()
    ids = torch.randint(0, 100, (17, ), dtype=torch.int32)
    pos = torch.randint(0, 40, (17, ), dtype=torch.int32)
    h = R.ragged_embed(ids, wte, pos, wpe, 2)
    d = R.ragged_embed(ids.cuda(), wte.cuda(), pos.cuda(), wpe.cuda(), 2)
    torch.testing.assert_close(d.cpu().float(), h.float(), atol=2e-2, rtol=2e-2)
    idx = torch.tensor([3, 0, 16], dtype=torch.int32)
    torch.testing.assert_close(R.row_gather(d, idx.cuda()).cpu(), d.cpu()[idx.long()])


@pytest.mark.parametrize("mt", ["llama", "mixtral", "gpt2"])
def test_engine_vs_hf_bf16(mt):
    transformers = pytest.importorskip("transformers")
    from transformers import AutoConfig, AutoModelForCausalLM
    from deepspeed_b200.inference.v2 import build_hf_engine
    kw = {"llama": dict(num_key_value_heads=2, intermediate_size=256),
          "mixtral": dict(num_key_value_heads=2, intermediate_size=256, num_local_experts=4, num_experts_per_tok=2),
          "gpt2": dict(n_embd=128, n_layer=2, n_head=4, n_positions=512)}[mt]
    cfg = AutoConfig.for_model(mt, vocab_size=512, hidden_size=128, num_hidden_layers=2, num_attention_heads=4,
                               max_position_embeddings=512, **kw)
    torch.manual_seed(0)
    m = AutoModelForCausalLM.from_config(cfg).to(torch.bfloat16).cuda().eval()
    e = build_hf_engine(m, {"state_manager": {"max_context": 512, "max_ragged_batch_size": 512,
                                              "max_ragged_sequence_count": 16,
                                              "memory_config": {"mode": "allocate", "size": 64}}})
    p0 = torch.randint(0, 512, (70, ))   # dense prefill path
    p1 = torch.randint(0, 512, (9, ))    # paged path
    lg = e.put([0, 1], [p0, p1])
    with torch.no_grad():
        r0 = m(p0[None].cuda()).logits[0, -1]
        r1 = m(p1[None].cuda()).logits[0, -1]
    for a, b in ((lg[0], r0), (lg[1], r1)):
        assert torch.nn.functional.cosine_similarity(a.float(), b.float(), dim=0) > 0.995
    # decode steps (CUDA-graph replay from the second call on) stay consistent with HF
    cur0, cur1 = p0, p1
    for _ in range(3):
        n0, n1 = lg[0].argmax().reshape(1).cpu(), lg[1].argmax().reshape(1).cpu()
        cur0, cur1 = torch.cat([cur0, n0]), torch.cat([cur1, n1])
        lg = e.put([0, 1], [n0, n1])
    with torch.no_grad():
        r0 = m(cur0[None].cuda()).logits[0, -1]
    assert torch.nn.functional.cosine_similarity(lg[0].float(), r0.float(), dim=0) > 0.99


def test_v1_kernel_inject_generate():
    transformers = pytest.importorskip("transformers")
    from transformers import AutoConfig, AutoModelForCausalLM
    import deepspeed_b200 as ds
    cfg = AutoConfig.for_model("llama", vocab_size=512, hidden_size=128, num_hidden_layers=2, num_attention_heads=4,
                               num_key_value_heads=2, intermediate_size=256, max_position_embeddings=512)
    torch.manual_seed(0)
    m = AutoModelForCausalLM.from_config(cfg).to(torch.bfloat16).cuda().eval()
    eng = ds.init_inference(m, dtype=torch.bfloat16, replace_with_kernel_inject=True, max_out_tokens=128,
                            enable_cuda_graph=True)
    ids = torch.randint(0, 512, (2, 12)).cuda()
    out = eng.generate(ids, max_new_tokens=8)
    assert out.shape == (2, 20) and torch.equal(out[:, :12], ids)


@pytest.mark.parametrize("mode", ["int8", "int4", "fp8"])
@pytest.mark.parametrize("M", [1, 5, 16, 27, 32, 100])
def test_weight_only_quantized_linear(mode, M):
    """Decode-sized inputs take the fused dequant+GEMV kernel, larger ones dequantise + tensor cores; both must equal the
    plain definition x @ dequant(W)^T."""
    from deepspeed_b200.inference.quantization.layers import maybe_quantized_linear, quantize_weight, _wq_gemv
    torch.manual_seed(0)
    N, K = 1536, 2048
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    x = torch.randn(M, K, device="cuda").bfloat16()
    qw = quantize_weight(w, mode, group_size=128)
    ref = torch.nn.functional.linear(x.float(), qw.dequantize().float(), b.float())
    got = maybe_quantized_linear(x, qw, b)
    assert (_wq_gemv(x, qw, b) is not None) == (M <= 32)
    torch.testing.assert_close(got.float(), ref, atol=3e-2 * ref.abs().max().item(), rtol=3e-2)


def test_quantized_engine_decode_gpu():
    transformers = pytest.importorskip("transformers")
    from transformers import AutoConfig, AutoModelForCausalLM
    from deepspeed_b200.inference.v2 import build_hf_engine
    cfg = AutoConfig.for_model("llama", vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=4,
                               num_key_value_heads=2, intermediate_size=512, max_position_embeddings=512)
    torch.manual_seed(0)
    m = AutoModelForCausalLM.from_config(cfg).to(torch.bfloat16).cuda().eval()
    sm = {"max_context": 512, "max_ragged_batch_size": 512, "max_ragged_sequence_count": 16,
          "memory_config": {"mode": "allocate", "size": 32}}
    ref = build_hf_engine(m, {"state_manager": sm})
    q8 = build_hf_engine(m, {"state_manager": sm, "quantization": {"quantization_mode": "int8"}})
    p = torch.randint(0, 512, (40, ))
    a, b = ref.put([0], [p])[0], q8.put([0], [p])[0]
    assert torch.nn.functional.cosine_similarity(a.float(), b.float(), dim=0) > 0.99
    n = a.argmax().reshape(1).cpu()
    a2, b2 = ref.put([0], [n])[0], q8.put([0], [n])[0]     # decode step: the GEMV kernel inside a CUDA graph
    assert torch.nn.functional.cosine_similarity(a2.float(), b2.float(), dim=0) > 0.99


def test_graphed_wrappers_replay_on_gpu():
    """DSUNet-style wrapper: one capture per input signature, replays reproduce eager results with fresh inputs."""
    from deepspeed_b200.model_implementations.features.cuda_graph import GraphedCallable
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Conv2d(4, 8, 3, padding=1), torch.nn.SiLU(), torch.nn.Conv2d(8, 4, 3, padding=1)).cuda().half()
    g = GraphedCallable(lambda x, s: net(x) * s)
    for bs in (1, 2, 1, 2, 2):
        x = torch.randn(bs, 4, 16, 16, device="cuda", dtype=torch.half)
        s = torch.rand(1, device="cuda", dtype=torch.half)
        with torch.no_grad():
            ref = net(x) * s
        out = g(x, s)
        torch.testing.assert_close(out, ref, atol=2e-3, rtol=2e-3)
    assert g.captures == 2 and g.replays == 5


def test_layerwise_kernel_injection_bf16_gpu():
    """Policy/container injection on the device (bf16): logits stay close to the Hugging Face model, generate() agrees."""
    import copy
    from types import SimpleNamespace
    transformers = pytest.importorskip("transformers")
    from transformers import AutoConfig, AutoModelForCausalLM
    from deepspeed_b200.module_inject.containers.base import InjectedLayer
    from deepspeed_b200.module_inject.replace_module import replace_transformer_layer
    cfg = AutoConfig.for_model("llama", vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=8,
                               num_key_value_heads=4, intermediate_size=512, max_position_embeddings=256)
    cfg._attn_implementation = "eager"
    torch.manual_seed(0)
    model = AutoModelForCausalLM.from_config(cfg).to(torch.bfloat16).cuda().eval()
    icfg = SimpleNamespace(replace_with_kernel_inject=True, dtype=torch.bfloat16, max_out_tokens=128,
                           tensor_parallel=SimpleNamespace(tp_size=1),
                           quant=SimpleNamespace(enabled=False, weight=SimpleNamespace(post_init_quant=None)))
    inj = replace_transformer_layer(None, copy.deepcopy(model), config=icfg).cuda()
    assert sum(isinstance(m, InjectedLayer) for m in inj.modules()) == 2
    ids = torch.randint(0, 512, (2, 24), device="cuda")
    with torch.no_grad():
        a, b = model(ids).logits.float(), inj(ids).logits.float()
    assert torch.nn.functional.cosine_similarity(a.flatten(), b.flatten(), dim=0) > 0.999
    with torch.no_grad():
        g1 = model.generate(ids[:, :8], max_new_tokens=6, do_sample=False, pad_token_id=0)
        g2 = inj.generate(ids[:, :8], max_new_tokens=6, do_sample=False, pad_token_id=0)
    assert (g1 == g2).float().mean() > 0.9


@pytest.mark.parametrize("mode", ["fp6", "fp8", "int8", "int4"])
@pytest.mark.parametrize("M,N,K", [(48, 256, 512), (200, 384, 1024), (128, 4096, 4096)])
def test_wq_tc_gemm_matches_dequant_reference(mode, M, N, K):
    """Fused dequantise-in-smem + wgmma weight-only GEMM (FP6 / FP8 / INT8 / INT4) vs dequantise + fp32 matmul."""
    import torch
    from deepspeed_b200.inference.quantization.layers import quantize_weight, wq_tc_linear
    torch.manual_seed(M + N)
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    x = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    b = (torch.randn(N, device="cuda") * 0.1).bfloat16()
    qw = quantize_weight(w, mode, group_size=128)
    y = wq_tc_linear(x, qw, b)
    assert y is not None, "shape should be eligible for the wgmma weight-only kernel"
    ref = x.float() @ qw.dequantize().float().t() + b.float()
    assert torch.isfinite(y.float()).all()
    assert (y.float() - ref).abs().max().item() < 2e-2 * ref.abs().max().item() + 2e-2


@pytest.mark.parametrize("mode", ["int8", "fp6"])
def test_mixed_moe_gemm_grouped_single_launch(mode):
    """MixedMoEGEMM: expert-sorted rows x weight-only-quantised expert weights in one grouped wgmma launch (device-side
    expert extents) vs the per-expert dequantise + matmul reference; includes an empty expert and a ragged tail."""
    import torch
    from deepspeed_b200.inference.quantization.layers import quantize_weight
    from deepspeed_b200.inference.v2.kernels.cutlass_ops.moe_gemm.mixed_moe_gemm import MixedMoEGEMM
    torch.manual_seed(0)
    E, N, K = 4, 384, 512
    counts = [200, 0, 37, 150]
    T = sum(counts)
    ws = [quantize_weight((torch.randn(N, K, device="cuda") * 0.05).bfloat16(), mode, group_size=128) for _ in range(E)]
    x = (torch.randn(T, K, device="cuda") * 0.5).bfloat16()
    out = torch.full((T, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    cums = torch.tensor(counts, device="cuda").cumsum(0)
    MixedMoEGEMM(torch.bfloat16, num_bits=8)(out, x, ws, None, cums)
    s = 0
    for e, c in enumerate(counts):
        if c:
            ref = x[s:s + c].float() @ ws[e].dequantize().float().t()
            assert (out[s:s + c].float() - ref).abs().max().item() < 2e-2 * ref.abs().max().item() + 2e-2
        s += c
    assert torch.isfinite(out.float()).all()
