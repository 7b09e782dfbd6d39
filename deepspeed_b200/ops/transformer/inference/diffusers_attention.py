"""Fused (cross-)attention for diffusers UNet / VAE blocks (reference ``ops/transformer/inference/diffusers_attention.py``):
packed QKV GEMM for self-attention, separate q / kv projections for cross-attention, flash SDPA, output projection."""
import torch
import torch.nn.functional as F
from torch import nn


class DeepSpeedDiffusersAttention(nn.Module):
    layer_id = 0

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.config.layer_id = DeepSpeedDiffusersAttention.layer_id
        DeepSpeedDiffusersAttention.layer_id += 1
        h = config.hidden_size
        dt = config.dtype if config.dtype in (torch.float16, torch.bfloat16, torch.float32) else torch.float16
        p = lambda *s: nn.Parameter(torch.empty(*s, dtype=dt), requires_grad=False)
        self.attn_qkvw, self.attn_qkvb = p(3 * h, h), p(3 * h)  # self-attention: packed
        self.attn_qw, self.attn_kw, self.attn_vw = p(h, h), p(h, h), p(h, h)  # cross-attention (context dim set on copy)
        self.attn_qb = None
        self.attn_ow, self.attn_ob = p(h, h), p(h)
        self.heads = config.heads
        self.do_out_bias = True

    def forward(self, input, context=None, input_mask=None):
        return DeepSpeedDiffusersAttentionFunction.apply(input, context, input_mask, self.config, self.attn_qkvw, self.attn_qw,
                                                         self.attn_kw, self.attn_vw, self.attn_qkvb, self.heads, self.attn_ow,
                                                         self.attn_ob, self.do_out_bias)


def load_triton_flash_attn():
    """The reference swaps in a Triton flash-attention for diffusers shapes; the fused SDPA (cuDNN flash on sm_90a) plays
    that role here, so there is nothing to load -- returns the function used."""
    return F.scaled_dot_product_attention


class DeepSpeedDiffusersAttentionFunction(torch.autograd.Function):
    """Inference-only self / cross attention of diffusion U-Nets and VAEs (reference ``diffusers_attention.py:33``): packed QKV
    GEMM for self attention, separate K/V projections of the conditioning for cross attention, flash SDPA, output GEMM."""

    @staticmethod
    def forward(ctx, input, context, input_mask, config, attn_qkvw, attn_qw, attn_kw, attn_vw, attn_qkvb, num_attention_heads_per_partition,
                attn_ow, attn_ob, do_out_bias=True, score_context_func=None, linear_func=None, pad_transform_func=None, rescale_qkv=None):
        b, s, _ = input.shape
        heads = num_attention_heads_per_partition
        if context is None:
            bias = attn_qkvb if attn_qkvb is not None and attn_qkvb.numel() else None
            q, k, v = F.linear(input, attn_qkvw, bias).chunk(3, dim=-1)
        else:
            q, k, v = F.linear(input, attn_qw), F.linear(context, attn_kw), F.linear(context, attn_vw)
        sp = lambda t: t.reshape(b, -1, heads, t.shape[-1] // heads).transpose(1, 2)
        o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v), attn_mask=input_mask)
        out = F.linear(o.transpose(1, 2).reshape(b, s, -1), attn_ow)
        return out + attn_ob if do_out_bias else out

    @staticmethod
    def backward(ctx, grad_output, grad_output1=None, grad_output2=None, grad_output3=None):
        raise RuntimeError("You are running with DeepSpeed Inference mode. Please switch to Training mode for running "
                           "backward!")
