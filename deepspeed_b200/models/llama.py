"""Llama-family decoder (Llama-2/3, Mistral, Phi-3, Qwen2, Qwen3) built on the deepspeed_b200 kernels.

This is the flagship training model of the framework (``BASELINE.json``: Llama-3-8B ZeRO-3 bf16).
The reference ships no training model; its users bring HF ``LlamaForCausalLM`` whose hot path on
H100 is PyTorch ops.  H100-first choices here:

* packed ``qkv`` and ``gate_up`` projections -> 4 large GEMMs per layer instead of 7;
* residual-add fused into RMSNorm (one pass over the residual stream per norm);
* RoPE applied in place on the packed QKV buffer with precomputed fp32 tables (one launch for Q+K), fused with Qwen3's
  per-head QK-norm when ``qk_norm`` is on;
* SwiGLU as one kernel on the packed gate_up output;
* weight gradients are written **directly into the ZeRO flat gradient buffer** by the linear's
  backward (``out=`` GEMM), bypassing AccumulateGrad and the copy into the reduce bucket;
* LM head + cross entropy chunked over tokens with the softmax gradient produced in place, so the
  ``[tokens, vocab]`` logits never exist (role of the reference ``FPDT_LogitsLoss``,
  ``sequence/fpdt_layer.py:1137``);
* attention core through ``ops.attention`` (cuDNN/flash SDPA library path or the native sm_90a kernel).
"""
import functools
import math
from dataclasses import dataclass, field
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from deepspeed_b200.ops.kernels import transformer_ops as T
from deepspeed_b200.ops.attention import causal_attention, check_cu_seqlens, document_positions
from deepspeed_b200.ops.linear import flat_linear


@dataclass
class LlamaConfig:
    vocab_size: int = 128256
    hidden_size: int = 4096
    intermediate_size: int = 14336
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    head_dim: Optional[int] = None
    max_position_embeddings: int = 8192
    rms_norm_eps: float = 1e-5
    rope_theta: float = 500000.0
    rope_scaling: Optional[dict] = None
    tie_word_embeddings: bool = False
    hidden_act: str = "silu"
    attention_bias: bool = False
    initializer_range: float = 0.02
    # causal sliding-window attention (HF ``sliding_window``): token i attends to tokens i - W < j <= i, inside its document
    # when packed; None attends to the whole causal prefix
    sliding_window: Optional[int] = None
    # FP8 products in the four decoder projections (qkv, o, gate|up with SwiGLU, down), forward and backward, with the
    # tensorwise power-of-two recipe of ``ops/fp8.py``; weights, optimizer, gradients, attention, norms, embedding and
    # LM head stay bf16
    fp8: bool = False
    # scaling granularity when ``fp8`` is on: "tensorwise" (one scale per tensor) or "blockwise" (1 x 128 strips of
    # activations and gradients, 128 x 128 blocks of weights: an outlier costs precision in its own block only)
    fp8_recipe: str = "tensorwise"
    # QK-norm (Qwen3): an RMSNorm with its own learned [head_dim] weight on every query head (``self_attn.q_norm``) and
    # every key head (``self_attn.k_norm``), after the projection and before RoPE, in fp32 (see
    # ``transformer_ops.qk_norm_rope_inplace``)
    qk_norm: bool = False
    # training knobs
    checkpoint_layers: int = 0  # number of decoder layers (from the front) run with activation recompute
    loss_chunk_tokens: int = 2048
    attention_backend: str = "auto"

    def __post_init__(self):
        if self.head_dim is None:
            self.head_dim = self.hidden_size // self.num_attention_heads
        if self.fp8_recipe not in ("tensorwise", "blockwise"):
            raise ValueError(f"fp8_recipe must be 'tensorwise' or 'blockwise', got {self.fp8_recipe!r}")

    @property
    def q_size(self):
        return self.num_attention_heads * self.head_dim

    @property
    def kv_size(self):
        return self.num_key_value_heads * self.head_dim

    def num_parameters(self, include_embeddings=True):
        h, i, L = self.hidden_size, self.intermediate_size, self.num_hidden_layers
        per = h * (self.q_size + 2 * self.kv_size) + self.q_size * h + 3 * h * i + 2 * h
        if self.qk_norm:
            per += 2 * self.head_dim
        n = L * per + h
        if include_embeddings:
            n += self.vocab_size * h * (1 if self.tie_word_embeddings else 2)
        return n

    def flops_per_token(self, seq_len, causal=True):
        """Training FLOPs/token (fwd + bwd = 3x fwd matmul FLOPs; attention counted causal).  With a sliding window
        shorter than ``seq_len`` the attention term counts the visible (query, key) pairs per token."""
        h, i, L = self.hidden_size, self.intermediate_size, self.num_hidden_layers
        mm = 2 * (h * (self.q_size + 2 * self.kv_size) + self.q_size * h + 3 * h * i) * L + 2 * h * self.vocab_size
        W = self.sliding_window
        if causal and W is not None and W < seq_len:
            pairs = seq_len * W - W * (W - 1) / 2  # sum over rows of min(row + 1, W)
            attn = 4 * (pairs / seq_len) * self.q_size * L
        else:
            attn = 4 * seq_len * self.q_size * L * (0.5 if causal else 1.0)
        return 3 * (mm + attn)


PRESETS = {
    # Llama-3.2-3B's shape with an untied LM head (3.6 B parameters): the largest Llama-3 shape whose full ZeRO training
    # state fits one 80 GB card
    "llama3.2-3b": dict(vocab_size=128256, hidden_size=3072, intermediate_size=8192, num_hidden_layers=28,
                        num_attention_heads=24, num_key_value_heads=8, rope_theta=500000.0, max_position_embeddings=8192),
    # Llama-3.2-1B as published (head dim 64, tied LM head, llama3 RoPE scaling)
    "llama3.2-1b": dict(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16,
                        num_attention_heads=32, num_key_value_heads=8, head_dim=64, tie_word_embeddings=True,
                        rope_theta=500000.0, max_position_embeddings=131072,
                        rope_scaling={"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0,
                                      "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}),
    "llama3-8b": dict(vocab_size=128256, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                      num_attention_heads=32, num_key_value_heads=8, rope_theta=500000.0, max_position_embeddings=8192),
    "llama3-70b": dict(vocab_size=128256, hidden_size=8192, intermediate_size=28672, num_hidden_layers=80,
                       num_attention_heads=64, num_key_value_heads=8, rope_theta=500000.0, max_position_embeddings=8192),
    "llama2-7b": dict(vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_hidden_layers=32,
                      num_attention_heads=32, num_key_value_heads=32, rope_theta=10000.0, max_position_embeddings=4096),
    "phi3-mini": dict(vocab_size=32064, hidden_size=3072, intermediate_size=8192, num_hidden_layers=32,
                      num_attention_heads=32, num_key_value_heads=32, rope_theta=10000.0, max_position_embeddings=4096),
    # Mistral-7B v0.1 (rope theta 10 000, 32 000 vocab) was trained with a 4096-token sliding window
    "mistral-7b": dict(vocab_size=32000, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                       num_attention_heads=32, num_key_value_heads=8, rope_theta=10000.0, max_position_embeddings=32768,
                       sliding_window=4096),
    # Qwen3 dense (QK-norm, head dim 128 with hidden / heads != 128 for the 1.7B); the 1.7B ties its LM head
    "qwen3-8b": dict(vocab_size=151936, hidden_size=4096, intermediate_size=12288, num_hidden_layers=36,
                     num_attention_heads=32, num_key_value_heads=8, head_dim=128, rope_theta=1e6, rms_norm_eps=1e-6,
                     max_position_embeddings=40960, qk_norm=True),
    "qwen3-1.7b": dict(vocab_size=151936, hidden_size=2048, intermediate_size=6144, num_hidden_layers=28,
                       num_attention_heads=16, num_key_value_heads=8, head_dim=128, tie_word_embeddings=True,
                       rope_theta=1e6, rms_norm_eps=1e-6, max_position_embeddings=40960, qk_norm=True),
    "tiny": dict(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                 num_key_value_heads=2, max_position_embeddings=256, rope_theta=10000.0),
}


def llama_config(name: str, **overrides) -> LlamaConfig:
    d = dict(PRESETS[name])
    d.update(overrides)
    return LlamaConfig(**d)


class RMSNorm(nn.Module):

    def __init__(self, hidden, eps):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden))
        self.eps = eps

    def forward(self, x, residual=None):
        return T.rms_norm(x, self.weight, self.eps, residual=residual)


class FlatLinear(nn.Module):
    """``nn.Linear`` whose backward writes dW straight into the ZeRO flat gradient buffer."""

    def __init__(self, in_features, out_features, bias=False, fp8=False, fp8_recipe="tensorwise"):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.zeros(out_features)) if bias else None
        self.fp8, self.fp8_recipe = fp8, fp8_recipe

    def forward(self, x):
        if self.fp8:
            from deepspeed_b200.ops.linear import fp8_linear
            return fp8_linear(x, self.weight, self.bias, recipe=self.fp8_recipe)
        return flat_linear(x, self.weight, self.bias)


class LMHead(FlatLinear):
    """Output projection.  ``forward(h)`` -> logits; ``forward(h, labels)`` -> mean cross entropy computed
    chunk-wise without materialising the logits.  Being a module call (not a bare use of ``weight``) keeps
    the ZeRO-3 fetch hooks in the loop; its backward needs no weights (dW/dh are produced in forward)."""
    ds_skip_backward_fetch = True

    def __init__(self, in_features, out_features, defer_ready=False):
        super().__init__(in_features, out_features)
        # the weight is tied to the input embedding, whose backward comes later and marks it ready (see TiedEmbedding)
        self.defer_ready = defer_ready

    def forward(self, h, labels=None, chunk=2048, assumed_scale=1.0):
        if labels is None:
            return flat_linear(h, self.weight, self.bias)
        from deepspeed_b200.ops.linear import chunked_linear_xent
        if self.defer_ready:
            return chunked_linear_xent(h.reshape(-1, h.shape[-1]), self.weight, labels.reshape(-1), chunk=chunk,
                                       assumed_scale=assumed_scale, defer_ready=True)
        return chunked_linear_xent(h.reshape(-1, h.shape[-1]), self.weight, labels.reshape(-1), chunk=chunk,
                                   assumed_scale=assumed_scale)


class TiedEmbedding(nn.Embedding):
    """The input embedding of a model whose LM head shares its weight.  Under ZeRO the head's dW sits in the weight's
    flat gradient view first; this module's backward adds the embedding gradient into the same view with the
    deterministic native kernel and marks the weight ready, once per backward (:func:`ops.linear.embedding`)."""

    def forward(self, input_ids):
        from deepspeed_b200.ops.linear import embedding
        return embedding(input_ids, self.weight)


class LlamaAttention(nn.Module):

    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.cfg = cfg
        self.qkv_proj = FlatLinear(cfg.hidden_size, cfg.q_size + 2 * cfg.kv_size, bias=cfg.attention_bias, fp8=cfg.fp8,
                                   fp8_recipe=cfg.fp8_recipe)
        self.o_proj = FlatLinear(cfg.q_size, cfg.hidden_size, bias=False, fp8=cfg.fp8, fp8_recipe=cfg.fp8_recipe)
        if cfg.qk_norm:
            # weights only: the attention node applies them, fused with RoPE; the module names match HF's keys
            self.q_norm = RMSNorm(cfg.head_dim, cfg.rms_norm_eps)
            self.k_norm = RMSNorm(cfg.head_dim, cfg.rms_norm_eps)

    def forward(self, x, rope, positions=None, cu_seqlens=None, max_seqlen=None):
        cfg = self.cfg
        B, S, _ = x.shape
        qkv = self.qkv_proj(x)  # [B, S, (hq + 2 hkv) d]
        qk_norm = (self.q_norm.weight, self.k_norm.weight, cfg.rms_norm_eps) if cfg.qk_norm else None
        out = causal_attention(qkv.view(B * S, -1), B, S, cfg.num_attention_heads, cfg.num_key_value_heads,
                               cfg.head_dim, rope, positions, backend=cfg.attention_backend, cu_seqlens=cu_seqlens,
                               max_seqlen=max_seqlen, sliding_window=cfg.sliding_window, qk_norm=qk_norm)
        return self.o_proj(out.view(B, S, cfg.q_size))


class LlamaMLP(nn.Module):

    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.gate_up_proj = FlatLinear(cfg.hidden_size, 2 * cfg.intermediate_size, fp8=cfg.fp8, fp8_recipe=cfg.fp8_recipe)
        self.down_proj = FlatLinear(cfg.intermediate_size, cfg.hidden_size, fp8=cfg.fp8, fp8_recipe=cfg.fp8_recipe)
        self.act = cfg.hidden_act
        self.fp8, self.fp8_recipe = cfg.fp8, cfg.fp8_recipe

    @property
    def trimmed_recompute(self) -> bool:
        """Whether this block runs the bf16 fused SwiGLU node, whose replay for activation checkpointing stops at gate|up
        (``forward(x, recompute=True)``).  The FP8 node and the unfused form replay their whole forward."""
        return self.act == "silu" and self.gate_up_proj.bias is None and self.down_proj.bias is None and not self.fp8

    def forward(self, x, recompute=False):
        if self.trimmed_recompute:
            from deepspeed_b200.ops.linear import swiglu_mlp
            return swiglu_mlp(x, self.gate_up_proj.weight, self.down_proj.weight, recompute=recompute)
        assert not recompute, "only the bf16 fused SwiGLU block has a trimmed recompute"
        if self.act == "silu" and self.gate_up_proj.bias is None and self.down_proj.bias is None:
            from deepspeed_b200.ops.linear import fp8_swiglu_mlp
            return fp8_swiglu_mlp(x, self.gate_up_proj.weight, self.down_proj.weight, recipe=self.fp8_recipe)
        return self.down_proj(T.gated_act(self.gate_up_proj(x), self.act))


class LlamaDecoderLayer(nn.Module):
    """Takes and returns ``(delta, residual)``: ``residual`` is the running stream *before* adding
    ``delta`` (the previous branch output), so every add is fused into the following RMSNorm.  ``recompute=True`` is the
    backward replay of an activation-checkpointed layer: the returned ``delta`` (the MLP output, which backward never
    reads) holds no data, see :meth:`LlamaMLP.forward`."""

    def __init__(self, cfg: LlamaConfig, layer_idx: int):
        super().__init__()
        self.layer_idx = layer_idx
        self.input_layernorm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps)
        self.self_attn = LlamaAttention(cfg)
        self.post_attention_layernorm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps)
        self.mlp = LlamaMLP(cfg)

    def forward(self, delta, residual, rope, positions=None, cu_seqlens=None, max_seqlen=None, recompute=False):
        if residual is None:
            residual = delta
            h = self.input_layernorm(delta)
        else:
            h, residual = self.input_layernorm(delta, residual)
        attn = self.self_attn(h, rope, positions, cu_seqlens, max_seqlen)
        h, residual = self.post_attention_layernorm(attn, residual)
        return self.mlp(h, recompute), residual


class LlamaModel(nn.Module):

    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.cfg = cfg
        self.embed_tokens = (TiedEmbedding if cfg.tie_word_embeddings else nn.Embedding)(cfg.vocab_size, cfg.hidden_size)
        self.embed_tokens.ds_skip_backward_fetch = True  # embedding backward is an index-add: no weights needed
        self.layers = nn.ModuleList([LlamaDecoderLayer(cfg, i) for i in range(cfg.num_hidden_layers)])
        self.norm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps)
        self._rope = None

    def rope_table(self, device):
        if self._rope is None or self._rope.cos.device != torch.device(device):
            self._rope = T.RotaryTable(self.cfg.head_dim, self.cfg.max_position_embeddings, self.cfg.rope_theta, device,
                                       self.cfg.rope_scaling)
        return self._rope

    def forward(self, input_ids, positions=None, cu_seqlens=None, max_seqlen=None):
        """``cu_seqlens`` / ``max_seqlen``: packed documents, see :meth:`LlamaForCausalLM.forward`."""
        cfg = self.cfg
        h = self.embed_tokens(input_ids)
        rope = self.rope_table(h.device)
        if cu_seqlens is not None:
            cu_seqlens, max_seqlen = prepare_packed(cu_seqlens, max_seqlen, input_ids.shape, h.device)
            if positions is None:
                positions = document_positions(cu_seqlens, input_ids.numel())
        delta, residual = h, None
        for i, layer in enumerate(self.layers):
            if self.training and i < cfg.checkpoint_layers and torch.is_grad_enabled():
                from deepspeed_b200.runtime.activation_checkpointing import checkpointing as ckpt
                # the replay in backward stops where that backward stops reading: no down GEMM (see LlamaMLP.forward)
                replay = functools.partial(layer, recompute=True) if layer.mlp.trimmed_recompute else None
                delta, residual = ckpt.checkpoint(layer, delta, residual, rope, positions, cu_seqlens, max_seqlen,
                                                  replay=replay)
            else:
                delta, residual = layer(delta, residual, rope, positions, cu_seqlens, max_seqlen)
        h, _ = self.norm(delta, residual)
        return h


def prepare_packed(cu_seqlens, max_seqlen, shape, device):
    """Check packed-document offsets for a ``[B, S]`` batch and return ``(cu_seqlens on device, max_seqlen)``.  A CPU
    tensor is checked in full (including that every row start ``b*S`` is a document boundary) and gives ``max_seqlen``;
    a device tensor is trusted and needs ``max_seqlen``."""
    B, S = shape
    max_seqlen = check_cu_seqlens(cu_seqlens, B * S, max_seqlen)
    if cu_seqlens.device.type == "cpu":
        row_starts = torch.arange(B, dtype=torch.int32) * S
        if not bool(torch.isin(row_starts, cu_seqlens).all()):
            raise ValueError("every row start b*S must be a document boundary in cu_seqlens (documents may not cross rows)")
        cu_seqlens = cu_seqlens.to(device)
    return cu_seqlens, max_seqlen


class LlamaForCausalLM(nn.Module):
    """``forward(input_ids, labels=None)`` -> loss (if labels) or logits.  Labels are next-token
    targets aligned with ``input_ids`` (shifted inside, HF convention) unless ``shift_labels=False``.

    Packed sequences: ``cu_seqlens`` (int32 ``[n_docs + 1]``) gives document offsets into the flattened
    ``input_ids.view(-1)``; each token then attends only within its document.  Documents may not cross rows: every row
    start ``b*S`` must be an offset.  A CPU ``cu_seqlens`` (the usual data-loader output) is validated, ``max_seqlen`` is
    derived from it and it is copied to the device once per forward; a device ``cu_seqlens`` needs ``max_seqlen`` and keeps
    the step free of host syncs.  ``positions`` defaults to the position inside each document (0 at its first token).
    With ``shift_labels=True`` the last token of every document gets target -100, so no token learns to predict the
    next document's first token (ignored targets do not count in the mean).
"""

    def __init__(self, cfg: LlamaConfig):
        super().__init__()
        self.cfg = cfg
        self.model = LlamaModel(cfg)
        self.lm_head = LMHead(cfg.hidden_size, cfg.vocab_size, defer_ready=cfg.tie_word_embeddings)
        if cfg.tie_word_embeddings:
            self.lm_head.weight = self.model.embed_tokens.weight
        self.ds_loss_multiplier = 1.0  # set by the engine: loss_scale / grad_accum_steps
        self.apply(self._init_weights)

    def _init_weights(self, m):
        std = self.cfg.initializer_range
        if isinstance(m, FlatLinear):
            if m.weight.numel():
                nn.init.normal_(m.weight, mean=0.0, std=std)
        elif isinstance(m, nn.Embedding):
            if m.weight.numel():
                nn.init.normal_(m.weight, mean=0.0, std=std)

    def forward(self, input_ids, labels=None, positions=None, shift_labels=True, cu_seqlens=None, max_seqlen=None):
        if cu_seqlens is not None:
            cu_seqlens, max_seqlen = prepare_packed(cu_seqlens, max_seqlen, input_ids.shape, input_ids.device)
        h = self.model(input_ids, positions, cu_seqlens, max_seqlen)
        if labels is None:
            return self.lm_head(h)
        if shift_labels:
            labels = torch.cat([labels[:, 1:], torch.full_like(labels[:, :1], -100)], dim=1)
            if cu_seqlens is not None and labels.numel():
                # each document's last token: (end - 1) mod T also covers empty documents (their "last token" is the
                # previous document's, or with end 0 the batch's final token -- both already document ends)
                ends = (cu_seqlens[1:].long() - 1).remainder(labels.numel())
                labels = labels.reshape(-1).index_fill(0, ends, -100).view_as(labels)
        return self.lm_head(h, labels=labels, chunk=self.cfg.loss_chunk_tokens, assumed_scale=self.ds_loss_multiplier)

    # ---- HF checkpoint interop ---------------------------------------------------------------------
    @staticmethod
    def convert_hf_state_dict(sd, cfg: LlamaConfig):
        """Pack HF ``q_proj/k_proj/v_proj`` and ``gate_proj/up_proj`` into this model's layout.  A tied model's
        ``lm_head.weight``, which HF checkpoint files omit, is the embedding's."""
        out = {}
        for k, v in sd.items():
            if ".self_attn.q_proj." in k:
                base = k.replace(".q_proj.", ".{}.")
                kk, vv = sd[base.format("k_proj")], sd[base.format("v_proj")]
                out[base.format("qkv_proj")] = torch.cat([v, kk, vv], dim=0)
            elif ".self_attn.k_proj." in k or ".self_attn.v_proj." in k:
                continue
            elif ".mlp.gate_proj." in k:
                up = sd[k.replace("gate_proj", "up_proj")]
                out[k.replace("gate_proj", "gate_up_proj")] = torch.cat([v, up], dim=0)
            elif ".mlp.up_proj." in k:
                continue
            elif "rotary_emb.inv_freq" in k:
                continue
            else:
                out[k] = v
        if cfg.tie_word_embeddings and "lm_head.weight" not in out and "model.embed_tokens.weight" in out:
            out["lm_head.weight"] = out["model.embed_tokens.weight"]
        return out

    @torch.no_grad()
    def generate_greedy(self, input_ids, max_new_tokens=16):
        """Reference (no KV cache) greedy decode used by tests; the serving path is inference v2."""
        ids = input_ids
        for _ in range(max_new_tokens):
            logits = self(ids)[:, -1]
            ids = torch.cat([ids, logits.argmax(-1, keepdim=True)], dim=1)
        return ids
