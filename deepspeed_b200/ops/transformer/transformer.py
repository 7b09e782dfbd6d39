"""Fused BERT-style training transformer layer.

API parity: reference ``ops/transformer/transformer.py`` (``DeepSpeedTransformerConfig :34``,
``DeepSpeedTransformerLayer :296``) over the ``csrc/transformer`` kernels (N7).  One layer =
``[LN] -> QKV GEMM -> (bias + [b,s,3,h,d]->[3,b,h,s,d]) -> attention (flash, or scores+masked-softmax+dropout when
attention dropout is on) -> out GEMM -> bias+dropout+residual -> [LN] -> FF1 GEMM + bias-GELU -> FF2 GEMM ->
bias+dropout+residual [-> LN]``.  The elementwise stages are this repo's sm_90a kernels (``transformer.cu``,
``misc.cu``); GEMMs go through ``ops.gemm`` (wgmma / cuBLAS).  ``normalize_invertible`` / ``gelu_checkpoint`` /
``attn_dropout_checkpoint`` map to activation recomputation of the corresponding stage.
"""
import json
import math

import torch
from torch import nn
import torch.nn.functional as F
from torch.utils.checkpoint import checkpoint

from deepspeed_b200.ops.kernels import misc_ops as K
from deepspeed_b200.ops.kernels import transformer_ops as T
from deepspeed_b200.ops.linear import flat_linear  # forward + both backward GEMMs on the wgmma kernel (ops.gemm)


class TransformerConfig:

    def __init__(self, batch_size, hidden_size, intermediate_size, heads, attn_dropout_ratio, hidden_dropout_ratio,
                 num_hidden_layers, initializer_range):
        self.layer_id = -1
        self.batch_size = batch_size
        self.hidden_size = hidden_size
        self.intermediate_size = intermediate_size
        self.heads = heads
        self.attn_dropout_ratio = attn_dropout_ratio
        self.hidden_dropout_ratio = hidden_dropout_ratio
        self.num_hidden_layers = num_hidden_layers
        self.initializer_range = initializer_range


class DeepSpeedTransformerConfig(TransformerConfig):

    def __init__(self, batch_size=-1, hidden_size=-1, intermediate_size=-1, heads=-1, attn_dropout_ratio=-1,
                 hidden_dropout_ratio=-1, num_hidden_layers=-1, initializer_range=-1, layer_norm_eps=1e-12, local_rank=-1,
                 seed=-1, fp16=False, pre_layer_norm=True, normalize_invertible=False, gelu_checkpoint=False,
                 adjust_init_range=True, attn_dropout_checkpoint=False, stochastic_mode=False, return_tuple=False,
                 training=True, bf16=False):
        super().__init__(batch_size, hidden_size,
                         intermediate_size if intermediate_size > 0 else 4 * hidden_size, heads, attn_dropout_ratio,
                         hidden_dropout_ratio, num_hidden_layers, initializer_range)
        self.fp16, self.bf16 = fp16, bf16
        self.pre_layer_norm = pre_layer_norm
        self.local_rank = local_rank
        self.seed = seed
        self.normalize_invertible = normalize_invertible
        self.gelu_checkpoint = gelu_checkpoint
        self.adjust_init_range = adjust_init_range
        self.test_gemm = False
        self.layer_norm_eps = layer_norm_eps
        self.training = training
        self.is_grad_enabled = True
        self.attn_dropout_checkpoint = attn_dropout_checkpoint
        self.stochastic_mode = stochastic_mode
        self.return_tuple = return_tuple

    @classmethod
    def from_dict(cls, json_object):
        config = DeepSpeedTransformerConfig()
        for key, value in json_object.items():
            config.__dict__[key] = value
        return config

    @classmethod
    def from_json_file(cls, json_file):
        with open(json_file, "r", encoding="utf-8") as reader:
            return cls.from_dict(json.loads(reader.read()))


class DeepSpeedTransformerLayer(nn.Module):
    layer_id = 0

    def __init__(self, config, initial_weights=None, initial_biases=None):
        super().__init__()
        self.config = config
        self.config.layer_id = DeepSpeedTransformerLayer.layer_id
        DeepSpeedTransformerLayer.layer_id += 1
        h, i = config.hidden_size, config.intermediate_size
        if initial_weights is None and initial_biases is None:
            self.attn_qkvw = nn.Parameter(torch.empty(3 * h, h))
            self.attn_qkvb = nn.Parameter(torch.empty(3 * h))
            self.attn_ow = nn.Parameter(torch.empty(h, h))
            self.attn_ob = nn.Parameter(torch.empty(h))
            self.attn_nw = nn.Parameter(torch.empty(h))
            self.attn_nb = nn.Parameter(torch.empty(h))
            self.inter_w = nn.Parameter(torch.empty(i, h))
            self.inter_b = nn.Parameter(torch.empty(i))
            self.output_w = nn.Parameter(torch.empty(h, i))
            self.output_b = nn.Parameter(torch.empty(h))
            self.norm_w = nn.Parameter(torch.empty(h))
            self.norm_b = nn.Parameter(torch.empty(h))
            self.init_transformer_weights(config.adjust_init_range)
        else:
            q, k, v = initial_weights[0].data, initial_weights[1].data, initial_weights[2].data
            self.attn_qkvw = nn.Parameter(torch.cat((q, k, v)))
            self.attn_qkvb = nn.Parameter(torch.cat([b.data for b in initial_biases[:3]]))
            self.attn_ow, self.attn_ob = initial_weights[3], initial_biases[3]
            self.attn_nw, self.attn_nb = initial_weights[4], initial_biases[4]
            self.inter_w, self.inter_b = initial_weights[5], initial_biases[5]
            self.output_w, self.output_b = initial_weights[6], initial_biases[6]
            self.norm_w, self.norm_b = initial_weights[7], initial_biases[7]
        if config.seed >= 0:
            self._seed = config.seed + config.layer_id
        else:
            self._seed = None

    def init_transformer_weights(self, adjust_init_range=False):
        num_layers = self.config.num_hidden_layers
        std = self.config.initializer_range
        out_std = std / math.sqrt(2.0 * num_layers) if (adjust_init_range and self.config.local_rank >= 0 or
                                                        adjust_init_range) and num_layers > 0 else std
        for w in (self.attn_qkvw, self.inter_w):
            w.data.normal_(mean=0.0, std=std)
        for w in (self.attn_ow, self.output_w):
            w.data.normal_(mean=0.0, std=out_std)
        for b in (self.attn_qkvb, self.attn_ob, self.attn_nb, self.inter_b, self.output_b, self.norm_b):
            b.data.zero_()
        self.attn_nw.data.fill_(1.0)
        self.norm_w.data.fill_(1.0)

    # ---- stages -----------------------------------------------------------------------------------------------------
    def _attention(self, x, mask):
        c = self.config
        B, S, H = x.shape
        nh, d = c.heads, H // c.heads
        qkv = flat_linear(x, self.attn_qkvw)
        qkv = K.bias_transform_0213(qkv, self.attn_qkvb, B, S, 3, nh, d) if not torch.is_grad_enabled() else \
            (qkv + self.attn_qkvb).view(B, S, 3, nh, d).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        p = c.attn_dropout_ratio if self.training else 0.0
        if p > 0.0:
            scores = torch.matmul(q, k.transpose(-1, -2))
            probs = K.attn_softmax(scores, mask=mask, scale=1.0 / math.sqrt(d))
            probs = K.dropout(probs, p, training=True, seed=self._seed)
            ctx = torch.matmul(probs, v)
        else:
            ctx = F.scaled_dot_product_attention(q, k, v, attn_mask=mask.to(q.dtype) if mask is not None else None)
        return ctx.transpose(1, 2).reshape(B, S, H)

    def _ffn(self, x):
        return T.bias_gelu(flat_linear(x, self.inter_w), self.inter_b)

    def forward(self, hidden_states, attention_mask=None, head_mask=None, layer_head_mask=None, encoder_hidden_states=None,
                encoder_attention_mask=None, past_key_value=None, output_attentions=False, grads=None):
        c = self.config
        x = hidden_states
        p = c.hidden_dropout_ratio if self.training else 0.0
        ck = self.training and torch.is_grad_enabled()
        if c.pre_layer_norm:
            a_in = T.layer_norm(x, self.attn_nw, self.attn_nb, c.layer_norm_eps)
        else:
            a_in = x
        if ck and c.attn_dropout_checkpoint:
            ctx = checkpoint(self._attention, a_in, attention_mask, use_reentrant=False)
        else:
            ctx = self._attention(a_in, attention_mask)
        a_out = flat_linear(ctx, self.attn_ow)
        x1 = K.dropout(a_out, p, self.training, bias=self.attn_ob, residual=x, seed=self._seed)
        if c.pre_layer_norm:
            f_in = T.layer_norm(x1, self.norm_w, self.norm_b, c.layer_norm_eps)
        else:
            x1 = T.layer_norm(x1, self.attn_nw, self.attn_nb, c.layer_norm_eps)
            f_in = x1
        inter = checkpoint(self._ffn, f_in, use_reentrant=False) if (ck and c.gelu_checkpoint) else self._ffn(f_in)
        f_out = flat_linear(inter, self.output_w)
        out = K.dropout(f_out, p, self.training, bias=self.output_b, residual=x1, seed=self._seed)
        if not c.pre_layer_norm:
            out = T.layer_norm(out, self.norm_w, self.norm_b, c.layer_norm_eps)
        return (out, ) if c.return_tuple else out


class DeepSpeedTransformerFunction:
    """Functional entry point of the fused training layer (reference ``transformer.py:143``).  The reference routes forward
    and backward through one hand-written autograd ``Function``; here the layer is a composition of fused autograd ops, so
    ``apply`` runs the layer's stages with an explicit parameter list and autograd differentiates it."""

    @staticmethod
    def apply(input, input_mask, self, grads, layer_id, attn_qkvw, attn_qkvb, attn_ow, attn_ob, attn_nw, attn_nb, inter_w,
              inter_b, output_w, output_b, norm_w, norm_b, config):
        names = ("attn_qkvw", "attn_qkvb", "attn_ow", "attn_ob", "attn_nw", "attn_nb", "inter_w", "inter_b", "output_w",
                 "output_b", "norm_w", "norm_b")
        given = (attn_qkvw, attn_qkvb, attn_ow, attn_ob, attn_nw, attn_nb, inter_w, inter_b, output_w, output_b, norm_w, norm_b)
        saved = {n: self._parameters[n] for n in names}
        try:
            for n, t in zip(names, given):  # run with the caller's tensors (they may be views / re-materialised copies)
                self._parameters[n] = t
            out = DeepSpeedTransformerLayer.forward(self, input, input_mask, grads=grads)
        finally:
            self._parameters.update(saved)
        return out[0] if isinstance(out, tuple) else out
