"""Local expert containers (reference ``moe/experts.py:13``)."""
import copy

import torch
from torch import nn


class Experts(nn.Module):
    """``num_local_experts`` deep copies of a user expert module; parameters are tagged
    ``allreduce=False`` / ``group_name`` so the engine reduces them over the expert-data-parallel group."""

    def __init__(self, expert, num_local_experts=1, expert_group_name=None):
        super().__init__()
        self.deepspeed_experts = nn.ModuleList([copy.deepcopy(expert) for _ in range(num_local_experts)])
        self.num_local_experts = num_local_experts
        for e in self.deepspeed_experts:
            for p in e.parameters():
                p.allreduce = False
                p.group_name = expert_group_name

    def forward(self, inputs):
        """``inputs``: [E_local, tokens, hidden] -> same shape."""
        outs = []
        for x, expert in zip(inputs.unbind(0), self.deepspeed_experts):
            o = expert(x)
            if isinstance(o, tuple):
                o = o[0]
            outs.append(o)
        return torch.stack(outs, dim=0)


class GroupedSwiGLUExperts(nn.Module):
    """Stacked SwiGLU experts evaluated with batched GEMMs: ``w13`` [E, 2I, H], ``w2`` [E, H, I].  The H100
    path for Mixtral-style layers (one strided-batched GEMM per projection instead of E small ones)."""

    def __init__(self, num_local_experts, hidden, intermediate, expert_group_name=None, act="silu", fp8_recipe=None):
        super().__init__()
        if fp8_recipe is not None:
            from deepspeed_b200.ops.linear import _check_recipe
            _check_recipe(fp8_recipe)
        self.num_local_experts = num_local_experts
        # None: bf16 products.  "tensorwise" / "blockwise": FP8 products under that recipe (dropless layout only)
        self.fp8_recipe = fp8_recipe
        # rows per segment of the dropless layout: the ragged kernels' granule (their k-block), 128 for FP8, 64 for bf16
        self.row_align = 64 if fp8_recipe is None else 128
        self.w13 = nn.Parameter(torch.empty(num_local_experts, 2 * intermediate, hidden))
        self.w2 = nn.Parameter(torch.empty(num_local_experts, hidden, intermediate))
        nn.init.normal_(self.w13, std=0.02)
        nn.init.normal_(self.w2, std=0.02)
        self.act = act
        for p in (self.w13, self.w2):
            p.allreduce = False
            p.group_name = expert_group_name

    def forward(self, inputs):
        """``inputs``: [E_local, tokens, hidden] (capacity-padded dispatch buffer) -> same shape; or ``(rows, offsets)``:
        expert-sorted rows [R, hidden] where expert ``e`` owns rows ``[offsets[e], offsets[e+1])`` (int32 on the rows'
        device, ``row_align``-row aligned, zero-padded segments: the dropless layout) -> [R, hidden].  Rows outside
        ``[offsets[0], offsets[E])`` of the result are unspecified (the wgmma path does not write them).  FP8 experts
        take the dropless layout only."""
        if isinstance(inputs, tuple):
            rows, offsets = inputs
            if self.fp8_recipe is not None:
                if self.act != "silu":
                    raise ValueError(f"FP8 experts are SwiGLU experts; act={self.act!r}")
                from deepspeed_b200.ops.linear import fp8_ragged_swiglu_mlp
                return fp8_ragged_swiglu_mlp(rows, offsets, self.w13, self.w2, recipe=self.fp8_recipe)
            from deepspeed_b200.ops.linear import ragged_swiglu_mlp
            return ragged_swiglu_mlp(rows, offsets, self.w13, self.w2, self.act)
        if self.fp8_recipe is not None:
            raise ValueError("FP8 experts take the dropless (rows, offsets) layout, not the capacity-padded "
                             "[E, C, hidden] buffer")
        if inputs.is_cuda and inputs.dtype == torch.bfloat16 and self.act == "silu" and inputs.shape[1] >= 256:
            # wgmma path: per expert the fused gate|up GEMM (+) SwiGLU, down GEMM, and in backward the dSwiGLU-fused
            # input-gradient GEMM plus weight-gradient GEMMs written straight into the stacked parameters' flat ZeRO
            # gradient views (one launch per expert and projection: every problem is [tokens x 14336 x 4096]-sized)
            from deepspeed_b200.ops.linear import grouped_swiglu_mlp
            return grouped_swiglu_mlp(inputs, self.w13, self.w2)
        from deepspeed_b200.ops.kernels.transformer_ops import gated_act
        gu = torch.bmm(inputs, self.w13.transpose(1, 2))
        h = gated_act(gu, self.act)
        return torch.bmm(h, self.w2.transpose(1, 2))
