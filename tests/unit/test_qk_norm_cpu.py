"""CPU tier: QK-norm attention (Qwen3).

* ``LlamaConfig(qk_norm=True)`` loaded from a randomly initialised transformers ``Qwen3ForCausalLM`` matches it in fp32:
  logits, loss and the gradient of every parameter (``q_norm`` / ``k_norm`` included), with default and with explicit
  positions, and greedy decoding;
* the ``qwen3-8b`` / ``qwen3-1.7b`` presets count the parameters HF's models have;
* ``qk_norm=False`` keeps the state-dict keys and parameter count;
* the fp32 torch composition of ``qk_norm_rope_inplace`` and its backward match float64 autograd, including a partial
  rotary table, no table, and weights with zeros and negatives.
"""
import pytest
import torch

from deepspeed_b200.models.llama import PRESETS, LlamaConfig, LlamaForCausalLM, llama_config
from deepspeed_b200.ops.kernels import transformer_ops as T

TINY = dict(vocab_size=97, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
            num_key_value_heads=2, head_dim=32, max_position_embeddings=64, rope_theta=1e6, rms_norm_eps=1e-6)


def _pair(seed=0):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    torch.manual_seed(seed)
    hf = Qwen3ForCausalLM(Qwen3Config(**TINY, tie_word_embeddings=False, attention_bias=False,
                                      attn_implementation="eager")).float().eval()
    with torch.no_grad():  # random norm weights, so a q/k swap or a missing weight cannot pass
        for layer in hf.model.layers:
            layer.self_attn.q_norm.weight.uniform_(-1.5, 1.5)
            layer.self_attn.k_norm.weight.uniform_(-1.5, 1.5)
    cfg = LlamaConfig(**TINY, qk_norm=True)
    m = LlamaForCausalLM(cfg).float().eval()
    m.load_state_dict(LlamaForCausalLM.convert_hf_state_dict(hf.state_dict(), cfg))
    return hf, m


def _hf_grad(hf, name):
    """HF gradient in this model's packed layout (``name`` is this model's parameter name)."""
    p = dict(hf.named_parameters())
    if ".qkv_proj." in name:
        return torch.cat([p[name.replace("qkv_proj", x)].grad for x in ("q_proj", "k_proj", "v_proj")])
    if ".gate_up_proj." in name:
        return torch.cat([p[name.replace("gate_up_proj", x)].grad for x in ("gate_proj", "up_proj")])
    return p[name].grad


def _close(got, want, what, rtol=1e-5):
    scale = want.abs().max().clamp_min(1e-30)
    err = (got - want).abs().max() / scale
    assert err <= rtol, f"{what}: max error {float(err):.3g} of the largest magnitude"


@pytest.mark.parametrize("explicit_positions", [False, True])
def test_matches_hf_qwen3(explicit_positions):
    hf, m = _pair()
    B, S = 2, 24
    ids = torch.randint(0, TINY["vocab_size"], (B, S), generator=torch.Generator().manual_seed(1))
    pos = None
    if explicit_positions:
        pos = torch.randint(0, TINY["max_position_embeddings"], (B, S), generator=torch.Generator().manual_seed(2))
    hf_out = hf(input_ids=ids, labels=ids, position_ids=pos)
    flat = pos.reshape(-1).to(torch.int32) if pos is not None else None
    with torch.no_grad():
        logits = m(ids, positions=flat)
    _close(logits, hf_out.logits.detach(), "logits")
    loss = m(ids, labels=ids, positions=flat)
    _close(loss.detach(), hf_out.loss.detach(), "loss")
    loss.backward()
    hf_out.loss.backward()
    names = [n for n, _ in m.named_parameters()]
    assert sum(".q_norm." in n or ".k_norm." in n for n in names) == 2 * TINY["num_hidden_layers"]
    for n, p in m.named_parameters():
        _close(p.grad, _hf_grad(hf, n), n)


def test_greedy_decode_matches_hf():
    hf, m = _pair(3)
    ids = torch.randint(0, TINY["vocab_size"], (1, 9), generator=torch.Generator().manual_seed(4))
    want = hf.generate(ids, max_new_tokens=8, do_sample=False, pad_token_id=0)
    got = m.generate_greedy(ids, max_new_tokens=8)
    assert got.tolist() == want.tolist()


@pytest.mark.parametrize("name,count", [("qwen3-8b", 8_190_735_360), ("qwen3-1.7b", 1_720_574_976)])
def test_preset_parameter_counts_match_hf(name, count):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    cfg = llama_config(name)
    assert cfg.num_parameters() == count
    hf_cfg = Qwen3Config(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                         num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                         num_key_value_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim,
                         tie_word_embeddings=cfg.tie_word_embeddings, max_position_embeddings=cfg.max_position_embeddings)
    with torch.device("meta"):
        hf = Qwen3ForCausalLM(hf_cfg)
        ours = LlamaForCausalLM(cfg)
    assert sum(p.numel() for p in hf.parameters()) == count
    assert sum(p.numel() for p in ours.parameters()) == count


def test_flag_off_keeps_keys_and_count():
    base = dict(PRESETS["tiny"])
    off, on = LlamaConfig(**base), LlamaConfig(**base, qk_norm=True)
    torch.manual_seed(0)
    keys_off = set(LlamaForCausalLM(off).state_dict())
    keys_on = set(LlamaForCausalLM(on).state_dict())
    assert not any("q_norm" in k or "k_norm" in k for k in keys_off)
    L = base["num_hidden_layers"]
    assert keys_on - keys_off == {f"model.layers.{i}.self_attn.{n}_norm.weight" for i in range(L) for n in "qk"}
    assert keys_off <= keys_on
    assert off.num_parameters() == sum(p.numel() for p in LlamaForCausalLM(off).parameters())
    assert on.num_parameters() == off.num_parameters() + 2 * L * off.head_dim


def _reference(qkv, hq, hkv, d, table, w_q, w_k, eps, positions, seq_len):
    """float64 autograd reference: out-of-place QK-norm then RoPE (rotate-half over ``table.rot_dim``)."""
    tokens = qkv.shape[0]
    x = qkv.view(tokens, hq + 2 * hkv, d)
    q, k, v = x[:, :hq], x[:, hq:hq + hkv], x[:, hq + hkv:]

    def norm(t, w):
        return t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + eps) * w

    def rope(t):
        if table is None:
            return t
        half = table.rot_dim // 2
        pos = positions.long() if positions is not None else torch.arange(tokens) % seq_len
        c, s = table.cos.double()[pos][:, None], table.sin.double()[pos][:, None]
        a, b = t[..., :half], t[..., half:2 * half]
        return torch.cat([a * c - b * s, b * c + a * s, t[..., 2 * half:]], -1)

    return torch.cat([rope(norm(q, w_q)), rope(norm(k, w_k)), v], 1).reshape(tokens, -1)


@pytest.mark.parametrize("d,rot", [(32, 32), (48, 16), (64, None)])
@pytest.mark.parametrize("with_positions", [False, True])
def test_composition_matches_float64_autograd(d, rot, with_positions):
    hq, hkv, tokens, seq_len, eps = 4, 2, 19, 7, 1e-6
    g = torch.Generator().manual_seed(d)
    qkv = torch.randn(tokens, (hq + 2 * hkv) * d, generator=g) * 3
    w_q = torch.randn(d, generator=g)
    w_k = torch.randn(d, generator=g)
    w_q[::5] = 0  # zeros and negatives in both weights
    w_k[1::7] = 0
    table = T.RotaryTable(rot, 64, 10000.0) if rot else None
    positions = torch.randint(0, 64, (tokens, ), generator=g, dtype=torch.int32) if with_positions else None
    dy = torch.randn(tokens, (hq + 2 * hkv) * d, generator=g)

    x64 = qkv.double().requires_grad_(True)
    wq64, wk64 = w_q.double().requires_grad_(True), w_k.double().requires_grad_(True)
    ref = _reference(x64, hq, hkv, d, table, wq64, wk64, eps, positions, seq_len)
    ref.backward(dy.double())

    buf = qkv.clone()
    raw = T.qk_norm_rope_inplace(buf, hq, hkv, d, table, w_q, w_k, eps, positions, seq_len)
    assert torch.equal(raw, qkv[:, :(hq + hkv) * d])
    _close(buf.double(), ref.detach(), "forward")
    assert torch.equal(buf[:, (hq + hkv) * d:], qkv[:, (hq + hkv) * d:])
    dbuf = dy.clone()
    dw_q, dw_k = T.qk_norm_rope_bwd_inplace(dbuf, raw, hq, hkv, d, table, w_q, w_k, eps, positions, seq_len)
    _close(dbuf[:, :(hq + hkv) * d].double(), x64.grad[:, :(hq + hkv) * d], "dQ|dK")
    assert torch.equal(dbuf[:, (hq + hkv) * d:], dy[:, (hq + hkv) * d:])
    _close(dw_q.double(), wq64.grad, "dw_q")
    _close(dw_k.double(), wk64.grad, "dw_k")
    assert T.qk_norm_rope_inplace(qkv.clone(), hq, hkv, d, table, w_q, w_k, eps, positions, seq_len,
                                  need_raw=False) is None
