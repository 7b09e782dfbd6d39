"""``MoE`` layer (reference ``moe/layer.py:17``)."""
from typing import Optional

import torch
from torch import nn

from deepspeed_b200.utils import groups
from deepspeed_b200.utils.logging import log_dist
from .experts import Experts
from .sharded_moe import MOELayer, TopKGate


class MoE(nn.Module):
    """Arguments as in the reference.  ``forward(hidden_states, used_token=None)`` returns
    ``(output, l_aux, exp_counts)``.  ``expert`` is a module copied per local expert, or a grouped container (a module
    with ``num_local_experts``) that takes the ``[E_local, C, hidden]`` dispatch buffer; with ``drop_tokens=False`` and
    ``ep_size == 1`` the grouped container must be :class:`GroupedSwiGLUExperts`, which takes the dropless
    ``(rows, offsets)`` layout."""

    def __init__(self, hidden_size, expert, num_experts=1, ep_size=1, k=1, capacity_factor=1.0,
                 eval_capacity_factor=1.0, min_capacity=4, use_residual=False, noisy_gate_policy: Optional[str] = None,
                 drop_tokens=True, use_rts=True, use_tutel=False, enable_expert_tensor_parallelism=False,
                 top2_2nd_expert_sampling=True):
        super().__init__()
        self.use_residual = use_residual
        self.enable_expert_tensor_parallelism = enable_expert_tensor_parallelism
        assert num_experts % ep_size == 0, f"Number of experts ({num_experts}) should be divisible by expert parallel size ({ep_size})"
        self.ep_size = ep_size
        self.expert_group_name = f"ep_size_{self.ep_size}"
        self.num_experts = num_experts
        self.num_local_experts = num_experts // self.ep_size
        log_dist(f"Creating MoE layer with num_experts: {num_experts} | num_local_experts: {self.num_local_experts} | "
                 f"expert_parallel_size: {self.ep_size}", [0])
        assert noisy_gate_policy is None or noisy_gate_policy in ["None", "Jitter", "RSample"], \
            "Unsupported noisy_gate_policy: " + noisy_gate_policy
        if isinstance(expert, nn.Module) and hasattr(expert, "num_local_experts") and not hasattr(expert, "deepspeed_experts"):
            experts = expert  # already a grouped (stacked) expert container sized for num_local_experts
            for p in experts.parameters():
                p.allreduce = False
                p.group_name = self.expert_group_name
        else:
            experts = Experts(expert, self.num_local_experts, self.expert_group_name)
        self.deepspeed_moe = MOELayer(
            TopKGate(hidden_size, num_experts, k, capacity_factor, eval_capacity_factor, min_capacity,
                     None if noisy_gate_policy == "None" else noisy_gate_policy, drop_tokens, use_rts, None,
                     top2_2nd_expert_sampling), experts, self.expert_group_name, self.ep_size, self.num_local_experts,
            use_tutel=use_tutel)
        self.deepspeed_moe.expert_tp = enable_expert_tensor_parallelism
        if self.use_residual:
            import copy
            self.mlp = copy.deepcopy(expert)
            self.coefficient = nn.Linear(hidden_size, 2)

    def set_deepspeed_parallelism(self, use_data_before_expert_parallel_=False):
        self._create_process_groups(use_data_before_expert_parallel_)

    def _create_process_groups(self, use_data_before_expert_parallel_=False):
        if self.ep_size > 1 or True:
            if groups._get_expert_parallel_group(self.expert_group_name) is None and \
                    self.expert_group_name not in groups._expert_parallel_size:
                groups._create_expert_and_data_parallel(self.ep_size, use_data_before_expert_parallel_)
        if self.enable_expert_tensor_parallelism:
            # experts are themselves tensor-sliced: every TP rank runs the exchange on the full token set
            # (reference groups._create_expert_data_and_model_parallel records the degree the same way)
            groups.expert_tensor_parallel_world_size = max(int(groups._get_model_parallel_world_size() or 1), 1)
        self.deepspeed_moe._set_ep_group(groups._get_expert_parallel_group(self.expert_group_name))

    def forward(self, hidden_states, used_token=None):
        output = self.deepspeed_moe(hidden_states, used_token)
        if self.use_residual:
            out_mlp = self.mlp(hidden_states)
            if isinstance(out_mlp, tuple):
                out_mlp = out_mlp[0]
            coef = torch.nn.functional.softmax(self.coefficient(hidden_states), dim=-1)
            output = output * coef[..., 0:1] + out_mlp * coef[..., 1:]
        return output, self.deepspeed_moe.l_aux, self.deepspeed_moe.exp_counts
