"""Gating + dispatch/combine for expert-parallel MoE.

Parity target: reference ``moe/sharded_moe.py`` (``top1gating :183``, ``top2gating :290``, ``topkgating :374``,
``TopKGate :449``, ``MOELayer :533``, ``_AllToAll :96``).  Differences by design:

* dispatch / combine are **index-based** (scatter rows into an expert-major buffer, weighted gather back)
  through the kernels in ``csrc/cuda/moe_ragged.cu`` instead of the dense ``einsum('sec,sm->ecm')`` with a
  ``[tokens, experts, capacity]`` mask -- O(tokens*k*hidden) instead of O(tokens*experts*capacity);
* with ``ep_size == 1`` the layout is exact (no capacity padding, nothing dropped unless asked);
* with expert parallelism the capacity-padded ``[E, C, H]`` buffer goes through ``all_to_all_single`` over the
  EP group exactly like the reference (fixed message shape), and the differentiable all-to-all is the same
  autograd trick (backward = the inverse all-to-all).
"""
import math
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from deepspeed_b200 import comm as dist
from deepspeed_b200.ops.kernels import moe_ops
from deepspeed_b200.utils import groups

TOPK_GATE_TIMER = "topk_gate"
MOE_TIMER = "moe"
FIRST_ALLTOALL_TIMER = "1st_a2a"
SECOND_ALLTOALL_TIMER = "2nd_a2a"


class _AllToAll(torch.autograd.Function):

    @staticmethod
    def forward(ctx, group, x):
        ctx.group = group
        x = x.contiguous()
        out = torch.empty_like(x)
        dist.all_to_all_single(out, x, group=group)
        return out

    @staticmethod
    def backward(ctx, dy):
        return None, _AllToAll.apply(ctx.group, dy)


def multiplicative_jitter(x, epsilon=1e-2):
    if epsilon == 0:
        return x
    return x * torch.empty_like(x).uniform_(1.0 - epsilon, 1.0 + epsilon)


def gumbel_rsample(shape, device):
    u = torch.rand(shape, device=device).clamp_(1e-9, 1 - 1e-9)
    return -torch.log(-torch.log(u))


def _capacity(num_tokens, num_experts, capacity_factor, min_capacity, k=1):
    cap = int(math.ceil(num_tokens / num_experts * capacity_factor * k))
    return max(cap, int(min_capacity))


class GateOutput:
    """Routing decision in INDEX form (``[T, k]`` expert ids / slots / weights) -- what the permutation kernels consume.
    Indexing or unpacking it yields the reference's dense 4-tuple ``(l_aux, combine_weights [T, E, C], dispatch_mask
    [T, E, C], exp_counts)`` (``sharded_moe.py:374``), materialised on demand for code written against that form.
    ``capacity`` is an int, except for dropless routing on one expert-parallel rank, where it is a 0-dim device tensor."""
    __slots__ = ("l_aux", "expert_ids", "weights", "positions", "offsets", "counts", "capacity", "k")

    def dense(self):
        T, k = self.expert_ids.shape
        E, C = self.counts.numel(), int(self.capacity)
        combine = torch.zeros(T, E, C, dtype=self.weights.dtype, device=self.weights.device)
        pos = self.positions.view(T, k).long()
        ok = (pos >= 0) & (pos < C)
        t = torch.arange(T, device=pos.device)[:, None].expand(T, k)
        combine = combine.index_put((t[ok], self.expert_ids.long()[ok], pos[ok]), self.weights[ok])
        mask = torch.zeros(T, E, C, dtype=torch.bool, device=pos.device)
        mask[t[ok], self.expert_ids.long()[ok], pos[ok]] = True
        return self.l_aux, combine, mask, self.counts

    def __iter__(self):
        return iter(self.dense())

    def __getitem__(self, i):
        return self.dense()[i]

    def __len__(self):
        return 4


def _keep_most_probable(ids, probs, counts, offsets, cap):
    """``drop_policy="probs"`` (reference ``topkgating``): when an expert is over capacity the ``cap`` most probable
    assignments stay; the survivors take their slots in token order. Dropped assignments get slot ``cap``."""
    e = ids.reshape(-1).long()
    n = e.numel()
    ar = torch.arange(n, device=e.device)
    by_w = torch.argsort(probs.reshape(-1), descending=True, stable=True)
    order = by_w[torch.argsort(e[by_w], stable=True)]  # grouped by expert, most probable first
    off = offsets.long()[:counts.numel()]
    rank = torch.empty_like(e)
    rank[order] = ar - off[e[order]]
    kept = rank < cap
    tok = torch.argsort(e, stable=True)  # grouped by expert, token order inside
    kept_t = kept[tok].long()
    before = torch.cumsum(kept_t, 0) - kept_t
    base = before[off.clamp(max=max(n - 1, 0))]
    slot = before - base[e[tok]]
    pos = torch.empty_like(e)
    pos[tok] = torch.where(kept_t.bool(), slot, torch.full_like(slot, cap))
    return pos.to(torch.int32).view_as(ids)


def topkgating(logits, k, capacity_factor, min_capacity, drop_tokens=True, ep_group=None, use_rts=False,
               noisy_gate_policy=None, normalize=True, drop_policy="probs"):
    """Token-choice top-k routing.  Returns a :class:`GateOutput`; ``weights`` are differentiable w.r.t.
    ``logits``; the index tensors are not."""
    T, E = logits.shape
    logits_for_choice = logits
    if noisy_gate_policy == "RSample":
        logits_for_choice = logits + gumbel_rsample(logits.shape, logits.device)
    gates = F.softmax(logits.float(), dim=1)
    _, ids = torch.topk(logits_for_choice if noisy_gate_policy == "RSample" else gates, k, dim=1)
    w = gates.gather(1, ids)
    if normalize and k > 1:
        w = w / w.sum(dim=1, keepdim=True).clamp(min=torch.finfo(w.dtype).eps)
    # load-balancing loss (GShard): fraction of router probability x fraction of tokens, first choice
    me = gates.mean(dim=0)
    if k <= 2:
        ce = F.one_hot(ids[:, 0], E).float().mean(dim=0)
    else:
        ce = F.one_hot(ids, E).float().sum(dim=1).mean(dim=0) / k
    l_aux = torch.sum(me * ce) * E
    out = GateOutput()
    out.l_aux, out.k = l_aux, k
    flat_ids = ids.to(torch.int32).contiguous()
    # per-expert counts without torch.bincount, which waits for the device to size its output
    counts = torch.zeros(E, dtype=torch.int32, device=logits.device).scatter_add_(
        0, ids.reshape(-1), torch.ones(ids.numel(), dtype=torch.int32, device=logits.device))
    if use_rts and k == 1:
        # random token selection: capacity slots go to a random subset instead of the earliest tokens
        perm = torch.randperm(T, device=logits.device)
        pos_p, counts, offsets = moe_ops.route(flat_ids[perm], E, counts=counts)
        positions = torch.empty_like(pos_p)
        positions[perm] = pos_p
    else:
        positions, counts, offsets = moe_ops.route(flat_ids, E, counts=counts)
    if drop_tokens:
        cap = _capacity(T, E, capacity_factor, min_capacity, k)
    elif ep_group is not None and dist.get_world_size(ep_group) > 1:
        mx = counts.max().to(torch.int64)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=ep_group)
        cap = max(int(mx.item()), int(min_capacity))
    else:
        # dropless on one expert-parallel rank: nothing is sized by the capacity, so it stays on the device (reading it,
        # e.g. through the dense view, synchronises)
        cap = counts.max().clamp(min=int(min_capacity))
    if drop_tokens and drop_policy == "probs":
        positions = _keep_most_probable(flat_ids, gates.gather(1, ids), counts, offsets, cap).reshape(positions.shape)
    out.expert_ids, out.weights, out.positions, out.offsets, out.counts, out.capacity = flat_ids, w, positions, offsets, \
        counts, cap
    return out


def top1gating(logits, capacity_factor, min_capacity, used_token=None, noisy_gate_policy=None, drop_tokens=True,
               use_rts=True, ep_group=None, use_tutel=False):
    return topkgating(logits, 1, capacity_factor, min_capacity, drop_tokens, ep_group, use_rts, noisy_gate_policy,
                      drop_policy="position")


def top2gating(logits, capacity_factor, min_capacity, drop_tokens=True, ep_group=None, top2_2nd_expert_sampling=True):
    return topkgating(logits, 2, capacity_factor, min_capacity, drop_tokens, ep_group, drop_policy="position")


class TopKGate(nn.Module):
    """Router (reference ``TopKGate :449``): fp32 linear gate + top-k selection."""

    def __init__(self, model_dim, num_experts, k=1, capacity_factor=1.0, eval_capacity_factor=1.0, min_capacity=8,
                 noisy_gate_policy: Optional[str] = None, drop_tokens=True, use_rts=True, ep_group=None,
                 top2_2nd_expert_sampling=True):
        super().__init__()
        self.wg = nn.Linear(model_dim, num_experts, bias=False)
        self.ep_group = ep_group
        self.k = k
        self.capacity_factor = capacity_factor
        self.eval_capacity_factor = eval_capacity_factor
        self.min_capacity = min_capacity
        self.noisy_gate_policy = noisy_gate_policy
        self.drop_tokens = drop_tokens
        self.use_rts = use_rts
        self.top2_2nd_expert_sampling = top2_2nd_expert_sampling
        self.gate_time = 0.0
        self.wall_clock_breakdown = False

    def _set_ep_group(self, ep_group):
        assert self.ep_group is None, "Attempting to override an existing ep_group"
        self.ep_group = ep_group

    def forward(self, x, used_token=None, use_tutel=False):
        xf = x.float()
        if self.noisy_gate_policy == "Jitter" and self.training:
            xf = multiplicative_jitter(xf)
        logits = F.linear(xf, self.wg.weight.float())
        cf = self.capacity_factor if self.training else self.eval_capacity_factor
        return topkgating(logits, self.k, cf, self.min_capacity, self.drop_tokens, self.ep_group,
                          use_rts=self.use_rts and self.training,
                          noisy_gate_policy=self.noisy_gate_policy if self.training else None,
                          # the reference routes k = 1 / 2 first come first served (top1gating / top2gating) and ranks
                          # by probability only on the general top-k path
                          drop_policy="position" if self.k <= 2 else "probs")


class MOELayer(nn.Module):
    """Route -> (all-to-all) -> local experts -> (all-to-all) -> combine.  Reference ``MOELayer :533``."""

    def __init__(self, gate, experts, ep_group_name, ep_size, num_local_experts, use_tutel=False):
        super().__init__()
        self.gate = gate
        self.experts = experts
        self.ep_group = None
        self.ep_size = ep_size
        self.ep_group_name = ep_group_name
        self.num_local_experts = num_local_experts
        self.l_aux = None
        self.exp_counts = None
        self.wall_clock_breakdown = False

    def _set_ep_group(self, ep_group):
        self.ep_group = ep_group
        self.gate._set_ep_group(ep_group)

    def _symm_state(self, flat):
        """Symmetric-memory exchange state when usable: EP over >1 GPUs of one NVLink domain, 16-bit/32-bit rows,
        grouped experts that take the [E_local, rows, H] layout (``DSB200_MOE_SYMM=0`` forces the NCCL path)."""
        import os
        if self.ep_size <= 1 or not flat.is_cuda or os.environ.get("DSB200_MOE_SYMM", "1") == "0":
            return None
        if self.gate.k > 8 or not self.gate.drop_tokens:
            return None
        if getattr(self, "_symm", False) is False:
            try:
                from deepspeed_b200.moe.symm_ep import SymmEP
                self._symm = SymmEP.get(self.ep_group)
            except Exception:
                self._symm = None
        return self._symm

    def forward(self, *inp):
        x = inp[0]
        H = x.shape[-1]
        flat = x.reshape(-1, H)
        T = flat.shape[0]
        g = self.gate(flat, inp[1] if len(inp) > 1 else None)
        self.l_aux, self.exp_counts = g.l_aux, g.counts
        E = self.ep_size * self.num_local_experts
        k = g.k
        if self.ep_size == 1 and not self.gate.drop_tokens:
            experts = self.experts.deepspeed_experts if hasattr(self.experts, "deepspeed_experts") else None
            if experts is not None:
                # user expert modules: rows sorted by expert, no padding -> ragged per-expert slices
                rows, slots = moe_ops.scatter(flat, g.expert_ids, g.positions, g.offsets, k, 0, T * k)
                outs = []
                for c, ex in zip(rows.split(g.counts.tolist(), dim=0), experts):
                    o = ex(c) if c.shape[0] else c
                    outs.append(o[0] if isinstance(o, tuple) else o)
                eo = torch.cat(outs, dim=0)
            else:
                from deepspeed_b200.moe.experts import GroupedSwiGLUExperts
                if not isinstance(self.experts, GroupedSwiGLUExperts):
                    raise TypeError(f"dropless routing (drop_tokens=False) with ep_size == 1 takes user expert modules "
                                    f"(wrapped in Experts) or GroupedSwiGLUExperts; {type(self.experts).__name__} is a "
                                    f"grouped container that does not take the (rows, offsets) layout")
                # grouped experts: every expert's segment padded to a multiple of the experts' row granule (64 rows bf16,
                # 128 FP8; zero-filled by the scatter), the offsets built on the device and the buffer sized by its
                # static bound T*k + E*(granule - 1) -- no host synchronisation in forward or backward.  FP8 rounds that
                # bound up to a multiple of 128: the transposed casts of the rows need R % 16
                align = self.experts.row_align
                seg = (g.counts + align - 1) // align * align
                offsets = torch.cat([seg.new_zeros(1), torch.cumsum(seg, 0, dtype=torch.int32)])
                R = T * k + E * (align - 1)
                if self.experts.fp8_recipe is not None:
                    R = -(-R // 128) * 128
                rows, slots = moe_ops.scatter(flat, g.expert_ids, g.positions, offsets, k, 0, R)
                eo = self.experts((rows, offsets))
            y = moe_ops.gather(eo, g.weights.to(torch.float32), slots, T, k)
            return y.reshape(x.shape).to(x.dtype)
        C = g.capacity
        # TP > 1 with replicated (non-TP) experts: every TP rank routed the same tokens, so each keeps 1/tp of every
        # expert's capacity rows through the exchange + experts and the slices are re-assembled afterwards
        # (reference sharded_moe.py MOELayer.forward: drop_tokens / gather_tokens).
        from deepspeed_b200.moe.mappings import _tp, drop_tokens, gather_tokens
        tp = 1 if getattr(self, "expert_tp", False) else _tp()[0]
        st = self._symm_state(flat) if tp == 1 else None
        if st is not None:
            # fused path: permutation kernels write / read the peers' symmetric buffers directly (no NCCL all-to-all)
            from deepspeed_b200.moe import symm_ep
            disp = symm_ep.dispatch(st, flat, g.expert_ids, g.positions, k, C, self.num_local_experts)
            eo = self.experts(disp)
            eo = eo[0] if isinstance(eo, tuple) else eo
            y = symm_ep.combine(st, eo, g.weights, g.expert_ids, g.positions, k, C, self.num_local_experts, T)
            return y.reshape(x.shape).to(x.dtype)
        rows, slots = moe_ops.scatter(flat, g.expert_ids, g.positions, g.offsets, k, C, E * C)
        disp = rows.view(E, C, H)
        C_full = C
        if tp > 1:
            if C % tp:
                disp = torch.nn.functional.pad(disp, (0, 0, 0, tp - C % tp))
            disp = drop_tokens(disp, dim=1).contiguous()
            C = disp.shape[1]
        if self.ep_size > 1:
            disp = _AllToAll.apply(self.ep_group, disp)  # [ep, E_local, C, H] flattened on dim 0
        disp = disp.view(self.ep_size, self.num_local_experts, C, H).transpose(0, 1).reshape(
            self.num_local_experts, self.ep_size * C, H)
        eo = self.experts(disp)
        eo = eo.view(self.num_local_experts, self.ep_size, C, H).transpose(0, 1).reshape(E, C, H).contiguous()
        if self.ep_size > 1:
            eo = _AllToAll.apply(self.ep_group, eo)
        if tp > 1:
            eo = gather_tokens(eo, dim=1)[:, :C_full].contiguous()
            C = C_full
        y = moe_ops.gather(eo.reshape(E * C, H), g.weights.to(torch.float32), slots, T, k)
        return y.reshape(x.shape).to(x.dtype)


USE_EINSUM = True


def einsum(rule, a, b):
    """``torch.einsum`` with the handful of contractions MoE gating / dispatch uses rewritten as plain broadcasts and
    matmuls (they hit cuBLAS directly and skip einsum's planning; reference ``sharded_moe.py:117``)."""
    if USE_EINSUM:
        return torch.einsum(rule, a, b)
    if rule == "s,se->se":
        return a.reshape(a.shape[0], -1) * b
    if rule == "se,sc->sec":
        return a.unsqueeze(2) * b.unsqueeze(1)
    if rule == "se,se->s":
        return (a * b).sum(-1)
    if rule == "se,sec->sec":
        return a.unsqueeze(2) * b
    if rule == "sec,sm->ecm":
        s, e, c = a.shape
        return torch.matmul(a.reshape(s, e * c).t(), b).reshape(e, c, b.shape[1])
    if rule == "sec,ecm->sm":
        return torch.matmul(a.reshape(a.shape[0], -1), b.reshape(-1, b.shape[-1]))
    if rule == "ks,ksm->sm":
        return (a.unsqueeze(-1) * b).sum(0)
    return torch.einsum(rule, a, b)
