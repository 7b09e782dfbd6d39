"""Head dim 64 in the training attention, CPU tier: the Llama-3.2-1B preset, the native kernels' support gates, the
``backend="native"`` error, and a tiny head-dim-64 Llama on the SDPA fallbacks with packed documents and a window."""
import pytest
import torch

from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
from deepspeed_b200.ops import attention as attn
from deepspeed_b200.ops.kernels import attention_sm100 as A


def test_llama32_1b_preset():
    cfg = llama_config("llama3.2-1b")
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (128256, 2048, 8192, 16)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim) == (32, 8, 64)
    assert cfg.tie_word_embeddings
    assert cfg.rope_theta == 500000.0 and cfg.max_position_embeddings == 131072
    assert cfg.rope_scaling == {"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                "original_max_position_embeddings": 8192}
    assert cfg.sliding_window is None
    assert cfg.num_parameters() == 1_235_814_400  # the published parameter count (tied LM head)
    h, i, L, V = 2048, 8192, 16, 128256
    for S in (2048, 4096):
        mm = 2 * (h * (2048 + 2 * 512) + 2048 * h + 3 * h * i) * L + 2 * h * V
        assert cfg.flops_per_token(S) == 3 * (mm + 4 * S * 2048 * L * 0.5)


class _FakeCudaRows:
    """Stands in for a 16-byte aligned CUDA bf16 ``[T, cols]`` tensor, so the gates' head-dim rule is checked without a
    device."""
    is_cuda = True
    dtype = torch.bfloat16

    def __init__(self, cols):
        self.cols = cols

    def stride(self, dim):
        return 1 if dim == -1 else self.cols

    def data_ptr(self):
        return 0


@pytest.mark.parametrize("d", [16, 32, 64, 80, 96, 128, 256])
def test_support_gates_take_head_dim_64_and_128(d):
    hq, hkv = 4, 2
    fake = _FakeCudaRows((hq + 2 * hkv) * d)
    assert A.supports(fake, hq, hkv, d, 256) == (d in (64, 128))
    assert A.supports_varlen(fake, hq, hkv, d) == (d in (64, 128))
    assert A.supports_fwd(fake, hq, hkv, d, 1, 256) == (d == 128)  # ragged prefill stays at head dim 128
    cpu = torch.zeros(256, (hq + 2 * hkv) * d, dtype=torch.bfloat16)
    assert not A.supports(cpu, hq, hkv, d, 256)
    assert not A.supports_varlen(cpu, hq, hkv, d)


@pytest.mark.parametrize("packed", [False, True])
def test_native_backend_raises_on_unsupported_input(packed):
    hq, hkv, d, S = 4, 2, 64, 128
    qkv = torch.randn(S, (hq + 2 * hkv) * d)
    kw = dict(cu_seqlens=torch.tensor([0, 50, S], dtype=torch.int32)) if packed else {}
    with pytest.raises(RuntimeError, match="head dim 64 or 128"):
        attn.causal_attention(qkv, 1, S, hq, hkv, d, backend="native", **kw)


def test_tiny_hd64_llama_runs_on_sdpa_fallbacks_without_kernel_calls(monkeypatch):
    """On CPU a head-dim-64 Llama with packed documents and a window never reaches the native kernels: the packed input
    goes through the per-document SDPA path (with the band mask), the dense one through the masked SDPA."""

    def no_native(*args, **kwargs):
        raise AssertionError("native attention kernel called on CPU")

    for name in ("fwd", "bwd", "fwd_varlen", "bwd_varlen"):
        monkeypatch.setattr(A, name, no_native)
    calls = {"varlen": 0, "band": 0}
    varlen, band = attn.varlen_attention_sdpa, attn._sdpa_band

    def count(key, fn):
        def wrapped(*args, **kwargs):
            calls[key] += 1
            return fn(*args, **kwargs)
        return wrapped

    monkeypatch.setattr(attn, "varlen_attention_sdpa", count("varlen", varlen))
    monkeypatch.setattr(attn, "_sdpa_band", count("band", band))
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=512, num_hidden_layers=2, head_dim=64, sliding_window=16)
    assert cfg.head_dim == 64
    model = LlamaForCausalLM(cfg)
    ids = torch.randint(0, cfg.vocab_size, (2, 64), generator=torch.Generator().manual_seed(1))
    cu = torch.tensor([0, 20, 64, 100, 128], dtype=torch.int32)
    loss = model(ids, labels=ids, cu_seqlens=cu)
    loss.backward()
    assert torch.isfinite(loss)
    assert calls["varlen"] == cfg.num_hidden_layers and calls["band"] > 0
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)
    calls["band"] = 0
    dense = model(ids, labels=ids)
    assert torch.isfinite(dense) and calls["band"] == cfg.num_hidden_layers
