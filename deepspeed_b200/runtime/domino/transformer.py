"""Domino: hide tensor-parallel all-reduces behind the other half of the batch.

Parity target: reference ``runtime/domino/transformer.py`` (``DominoTransformerLayer :228``, ``forward
:349-451``, ``ShardedAttention :137``).  The micro-batch is split in two halves; the row-parallel all-reduce of
half 0 (attention output, then MLP output) is launched asynchronously and waited for only after half 1's
compute of the same stage has been issued, so NVLink traffic overlaps wgmma math.  Backward uses the same
trick through autograd hooks on the async handles (``_AsyncAllReduce``).
"""
import torch
import torch.nn.functional as F
from torch import nn

from deepspeed_b200 import comm as dist
from deepspeed_b200.ops.kernels import transformer_ops as T


import enum


def is_rank_0():
    return not dist.is_initialized() or dist.get_rank() == 0


class DominoModule(nn.Module):
    """Common base of the Domino building blocks (reference ``transformer.py:18``)."""


class LayerType(enum.Enum):
    encoder = 1
    decoder = 2


class AttnType(enum.Enum):
    self_attn = 1
    cross_attn = 2


class AttnMaskType(enum.Enum):
    padding = 1
    causal = 2


class ModelType(enum.Enum):
    encoder_or_decoder = 1
    encoder_and_decoder = 2


# in-flight backward all-reduces, keyed by "<layer>_<half>[_<stage>]": launched by ``_CopyToModelParallelRegionA.backward``,
# drained by the matching ``NoOper.backward`` that autograd reaches only after the OTHER half's backward math was issued
handle_dic = {}


class NoOper(torch.autograd.Function):
    """Identity; in backward it waits for the async gradient all-reduce registered under ``h_id``."""

    @staticmethod
    def forward(ctx, input_, dic_, h_id):
        ctx.dic, ctx.h_id = dic_, h_id
        return input_.view_as(input_)

    @staticmethod
    def backward(ctx, grad_output):
        h = ctx.dic.pop(ctx.h_id, None)
        if h is not None:
            h.wait()
        return grad_output, None, None


def no_oper(input_, dic_, h_id):
    return NoOper.apply(input_, dic_, h_id)


def _group_of(mpu_or_group):
    if mpu_or_group is None or not hasattr(mpu_or_group, "get_tensor_model_parallel_group"):
        return mpu_or_group
    return mpu_or_group.get_tensor_model_parallel_group()


class _CopyToModelParallelRegionA(torch.autograd.Function):
    """Identity forward; backward STARTS the all-reduce of the input gradient and parks the handle in ``dic_[h_id]``
    (``mpu`` may be a Megatron-style mpu or a process group)."""

    @staticmethod
    def forward(ctx, mpu, input_, dic_, h_id):
        ctx.group, ctx.dic, ctx.h_id = _group_of(mpu), dic_, h_id
        return input_.view_as(input_)

    @staticmethod
    def backward(ctx, grad_output):
        if ctx.group is None or dist.get_world_size(ctx.group) == 1:
            return None, grad_output, None, None
        g = grad_output.contiguous()
        ctx.dic[ctx.h_id] = dist.all_reduce(g, group=ctx.group, async_op=True)
        return None, g, None, None


def copy_to_tensor_model_parallel_region_a(mpu, input_, dic_, h_id):
    return _CopyToModelParallelRegionA.apply(mpu, input_, dic_, h_id)


class CoreAttention(DominoModule):
    """Causal SDPA over this rank's heads: ``[b, np, sq, hn]`` in, ``[sq, b, hp]`` out (reference ``:104``)."""

    def __init__(self, config, layer_number, mpu, attn_mask_type=AttnMaskType.causal):
        super().__init__()
        self.layer_number = max(1, layer_number)
        self.att_dropout_p = getattr(config, "attention_dropout", 0.0)
        self.attn_mask_type = attn_mask_type
        world = mpu.get_tensor_model_parallel_world_size() if mpu is not None else 1
        self.hidden_size_per_partition = config.kv_channels * config.num_attention_heads // world

    def forward(self, query_layer, key_layer, value_layer, attention_mask=None):
        ctx = F.scaled_dot_product_attention(query_layer, key_layer, value_layer,
                                             dropout_p=self.att_dropout_p if self.training else 0.0,
                                             is_causal=self.attn_mask_type == AttnMaskType.causal)
        sq, b = ctx.shape[2], ctx.shape[0]
        return ctx.permute(2, 0, 1, 3).reshape(sq, b, self.hidden_size_per_partition)


class _AsyncAllReduce(torch.autograd.Function):
    """Forward: start an async all-reduce and stash the handle; backward: plain identity (input grads of a
    row-parallel output are already complete)."""

    @staticmethod
    def forward(ctx, x, group, holder):
        if group is None or dist.get_world_size(group) == 1:
            return x
        holder.append(dist.all_reduce(x, group=group, async_op=True))
        return x

    @staticmethod
    def backward(ctx, g):
        return g, None, None


class _WaitHandle(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, holder):
        while holder:
            h = holder.pop()
            if h is not None:
                h.wait()
        return x

    @staticmethod
    def backward(ctx, g):
        return g, None


class _CopyToTP(torch.autograd.Function):
    """Identity forward, async all-reduce of the gradient in backward (column-parallel input)."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        return x

    @staticmethod
    def backward(ctx, g):
        if ctx.group is not None and dist.get_world_size(ctx.group) > 1:
            dist.all_reduce(g.contiguous(), group=ctx.group)
        return g, None


class ShardedAttention(DominoModule):

    def __init__(self, hidden, heads, tp_group):
        super().__init__()
        self.tp = dist.get_world_size(tp_group) if tp_group is not None else 1
        self.group = tp_group
        self.local_heads = heads // self.tp
        self.head_dim = hidden // heads
        self.qkv = nn.Linear(hidden, 3 * self.local_heads * self.head_dim)
        self.dense = nn.Linear(self.local_heads * self.head_dim, hidden, bias=False)
        self.dense_bias = nn.Parameter(torch.zeros(hidden))

    def forward(self, x, grad_sync=None):
        B, S, _ = x.shape
        x = _CopyToTP.apply(x, self.group) if grad_sync is None else \
            copy_to_tensor_model_parallel_region_a(self.group, x, handle_dic, grad_sync)
        qkv = self.qkv(x)
        q, k, v = (t.reshape(B, S, self.local_heads, self.head_dim).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, S, -1)
        return self.dense(o)  # partial sum: caller all-reduces


class ShardedMLP(DominoModule):

    def __init__(self, hidden, ffn, tp_group):
        super().__init__()
        self.tp = dist.get_world_size(tp_group) if tp_group is not None else 1
        self.group = tp_group
        self.fc1 = nn.Linear(hidden, ffn // self.tp)
        self.fc2 = nn.Linear(ffn // self.tp, hidden, bias=False)
        self.fc2_bias = nn.Parameter(torch.zeros(hidden))

    def forward(self, x, grad_sync=None):
        x = _CopyToTP.apply(x, self.group) if grad_sync is None else \
            copy_to_tensor_model_parallel_region_a(self.group, x, handle_dic, grad_sync)
        return self.fc2(F.gelu(self.fc1(x), approximate="tanh"))


class DominoTransformerLayer(DominoModule):

    def __init__(self, hidden_size, num_attention_heads, ffn_hidden_size=None, tp_group=None, layernorm_epsilon=1e-5):
        super().__init__()
        self.group = tp_group
        self.input_layernorm = nn.LayerNorm(hidden_size, eps=layernorm_epsilon)
        self.self_attention = ShardedAttention(hidden_size, num_attention_heads, tp_group)
        self.post_attention_layernorm = nn.LayerNorm(hidden_size, eps=layernorm_epsilon)
        self.mlp = ShardedMLP(hidden_size, ffn_hidden_size or 4 * hidden_size, tp_group)

    def forward(self, hidden_states):
        """hidden_states [B, S, H]; B is split into two interleaved halves."""
        x0, x1 = hidden_states.chunk(2, dim=0) if hidden_states.shape[0] > 1 else (hidden_states, None)
        if x1 is None:
            return self._plain(hidden_states)
        h0, h1 = [], []
        k = id(self)
        # Backward overlap: each half's input-gradient all-reduce is STARTED in ``copy_to_..._a.backward`` and WAITED in
        # the ``no_oper`` node created here, i.e. before either half's compute nodes -- autograd replays nodes in reverse
        # creation order, so the other half's backward GEMMs are issued between the start and the wait.
        n0 = no_oper(self.input_layernorm(x0), handle_dic, f"{k}_0_attn")
        n1 = no_oper(self.input_layernorm(x1), handle_dic, f"{k}_1_attn")
        # ---- attention: a0 reduce overlaps attention of half 1 ----
        a0 = _AsyncAllReduce.apply(self.self_attention(n0, f"{k}_0_attn"), self.group, h0)
        a1 = _AsyncAllReduce.apply(self.self_attention(n1, f"{k}_1_attn"), self.group, h1)
        a0 = _WaitHandle.apply(a0, h0)
        r0 = x0 + a0 + self.self_attention.dense_bias
        p0 = no_oper(self.post_attention_layernorm(r0), handle_dic, f"{k}_0_mlp")
        # ---- MLP of half 0 overlaps the a1 reduce ----
        m0 = _AsyncAllReduce.apply(self.mlp(p0, f"{k}_0_mlp"), self.group, h0)
        a1 = _WaitHandle.apply(a1, h1)
        r1 = x1 + a1 + self.self_attention.dense_bias
        p1 = no_oper(self.post_attention_layernorm(r1), handle_dic, f"{k}_1_mlp")
        m1 = _AsyncAllReduce.apply(self.mlp(p1, f"{k}_1_mlp"), self.group, h1)
        m0 = _WaitHandle.apply(m0, h0)
        o0 = r0 + m0 + self.mlp.fc2_bias
        m1 = _WaitHandle.apply(m1, h1)
        o1 = r1 + m1 + self.mlp.fc2_bias
        return torch.cat([o0, o1], dim=0)

    def _plain(self, x):
        a = self.self_attention(self.input_layernorm(x))
        if self.group is not None and dist.get_world_size(self.group) > 1:
            dist.all_reduce(a, group=self.group)
        r = x + a + self.self_attention.dense_bias
        m = self.mlp(self.post_attention_layernorm(r))
        if self.group is not None and dist.get_world_size(self.group) > 1:
            dist.all_reduce(m, group=self.group)
        return r + m + self.mlp.fc2_bias


class DominoTransformer(DominoModule):

    def __init__(self, num_layers, hidden_size, num_attention_heads, ffn_hidden_size=None, tp_group=None):
        super().__init__()
        self.layers = nn.ModuleList([DominoTransformerLayer(hidden_size, num_attention_heads, ffn_hidden_size, tp_group)
                                     for _ in range(num_layers)])
        self.final_layernorm = nn.LayerNorm(hidden_size)

    def forward(self, x):
        for l in self.layers:
            x = l(x)
        return self.final_layernorm(x)
