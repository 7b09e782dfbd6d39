"""Mixtral-style sparse-MoE decoder (BASELINE.json config 3: Mixtral 8x7B with expert parallelism).

Llama attention + a top-2 MoE feed-forward whose experts are *stacked* (``GroupedSwiGLUExperts``) so each
projection is one strided-batched GEMM; routing / dispatch / combine run through the index-based kernels of
``csrc/cuda/moe_ragged.cu`` and the EP all-to-all of ``moe/sharded_moe.py``.
"""
from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from deepspeed_b200.models.llama import (LMHead, LlamaAttention, LlamaConfig, RMSNorm)
from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
from deepspeed_b200.moe.layer import MoE
from deepspeed_b200.ops.kernels import transformer_ops as T


@dataclass
class MixtralConfig(LlamaConfig):
    num_local_experts: int = 8
    num_experts_per_tok: int = 2
    router_aux_loss_coef: float = 0.02
    ep_size: int = 1
    capacity_factor: float = 1.25
    drop_tokens: bool = True
    # FP8 products in the experts (gate|up with SwiGLU, down; forward, dgrad and wgrad) under ``fp8_recipe``, independent
    # of ``fp8`` (which keeps meaning the attention projections).  Dropless routing on one expert-parallel rank only
    fp8_experts: bool = False

    def __post_init__(self):
        super().__post_init__()
        if self.fp8_experts and (self.drop_tokens or self.ep_size > 1):
            raise ValueError("fp8_experts=True needs the dropless layout on one expert-parallel rank (drop_tokens=False, "
                             f"ep_size=1); got drop_tokens={self.drop_tokens}, ep_size={self.ep_size}")


MIXTRAL_PRESETS = {
    "mixtral-8x7b": dict(vocab_size=32000, hidden_size=4096, intermediate_size=14336, num_hidden_layers=32,
                         num_attention_heads=32, num_key_value_heads=8, rope_theta=1e6, max_position_embeddings=32768,
                         num_local_experts=8, num_experts_per_tok=2),
    "tiny-moe": dict(vocab_size=512, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4,
                     num_key_value_heads=2, max_position_embeddings=128, rope_theta=10000.0, num_local_experts=4,
                     num_experts_per_tok=2),
}


def mixtral_config(name, **over):
    d = dict(MIXTRAL_PRESETS[name])
    d.update(over)
    return MixtralConfig(**d)


class MixtralDecoderLayer(nn.Module):

    def __init__(self, cfg: MixtralConfig, idx: int):
        super().__init__()
        self.input_layernorm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps)
        self.self_attn = LlamaAttention(cfg)
        self.post_attention_layernorm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps)
        assert cfg.num_local_experts % cfg.ep_size == 0
        experts = GroupedSwiGLUExperts(cfg.num_local_experts // cfg.ep_size, cfg.hidden_size, cfg.intermediate_size,
                                       fp8_recipe=cfg.fp8_recipe if cfg.fp8_experts else None)
        self.block_sparse_moe = MoE(cfg.hidden_size, experts, num_experts=cfg.num_local_experts, ep_size=cfg.ep_size,
                                    k=cfg.num_experts_per_tok, capacity_factor=cfg.capacity_factor,
                                    eval_capacity_factor=cfg.capacity_factor, min_capacity=4,
                                    drop_tokens=cfg.drop_tokens, use_rts=False)

    def forward(self, delta, residual, rope, positions=None):
        if residual is None:
            residual = delta
            h = self.input_layernorm(delta)
        else:
            h, residual = self.input_layernorm(delta, residual)
        attn = self.self_attn(h, rope, positions)
        h, residual = self.post_attention_layernorm(attn, residual)
        out, l_aux, _ = self.block_sparse_moe(h)
        return out, residual, l_aux


class MixtralForCausalLM(nn.Module):

    def __init__(self, cfg: MixtralConfig):
        super().__init__()
        self.cfg = cfg
        self.embed_tokens = nn.Embedding(cfg.vocab_size, cfg.hidden_size)
        self.embed_tokens.ds_skip_backward_fetch = True
        self.layers = nn.ModuleList([MixtralDecoderLayer(cfg, i) for i in range(cfg.num_hidden_layers)])
        self.norm = RMSNorm(cfg.hidden_size, cfg.rms_norm_eps)
        self.lm_head = LMHead(cfg.hidden_size, cfg.vocab_size)
        self.ds_loss_multiplier = 1.0
        self._rope = None
        for m in self.modules():
            if isinstance(m, (nn.Embedding, )):
                nn.init.normal_(m.weight, std=cfg.initializer_range)
            elif hasattr(m, "weight") and isinstance(getattr(m, "weight", None), nn.Parameter) and m.weight.dim() == 2 \
                    and not isinstance(m, nn.Embedding):
                nn.init.normal_(m.weight, std=cfg.initializer_range)

    def forward(self, input_ids, labels=None, positions=None):
        h = self.embed_tokens(input_ids)
        if self._rope is None or self._rope.cos.device != h.device:
            self._rope = T.RotaryTable(self.cfg.head_dim, self.cfg.max_position_embeddings, self.cfg.rope_theta, h.device)
        delta, residual = h, None
        aux = 0.0
        for layer in self.layers:
            delta, residual, l_aux = layer(delta, residual, self._rope, positions)
            aux = aux + l_aux
        h, _ = self.norm(delta, residual)
        if labels is None:
            return self.lm_head(h)
        labels = torch.cat([labels[:, 1:], torch.full_like(labels[:, :1], -100)], dim=1)
        loss = self.lm_head(h, labels=labels, chunk=self.cfg.loss_chunk_tokens, assumed_scale=self.ds_loss_multiplier)
        return loss + self.cfg.router_aux_loss_coef * aux
