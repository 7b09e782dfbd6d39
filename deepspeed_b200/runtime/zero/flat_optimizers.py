"""Optimizers that act on the rank-local flat arenas of :class:`ZeroShardedOptimizer`.

A *flat optimizer* owns optimizer state tensors with the same length as the master arena and
updates one contiguous segment per call.  This is how the fused sm_90a kernels are reached: one
launch per (param-group run) instead of the reference's per-tensor multi-tensor-apply chunking
(``ops/adam/fused_adam.py`` + ``csrc/adam/multi_tensor_apply.cuh``).

``TorchOptimizerAdapter`` wraps any client ``torch.optim.Optimizer`` by presenting fp32
``nn.Parameter`` views of the master arena (the reference's ``single_partition_of_fp32_groups``).
"""
from typing import Dict, List, Optional

import torch

from deepspeed_b200.ops.kernels import flat_ops


class FlatOptimizer:
    """Interface: ``init_state``, ``step_segment``, ``state_tensors``."""
    state_names: List[str] = []
    fused = True

    def __init__(self, defaults: dict):
        self.defaults = dict(defaults)
        self.state: Dict[str, torch.Tensor] = {}

    def init_state(self, numel: int, device, dtype=torch.float32, pin=False):
        for n in self.state_names:
            if pin and torch.device(device).type == "cpu" and torch.cuda.is_available():
                from deepspeed_b200.ops.pinned import pinned_empty
                t = pinned_empty(numel, dtype).zero_()  # exact-size page-locked arena (see ops/pinned.py)
            else:
                t = torch.zeros(numel, dtype=dtype, device=device)
            self.state[n] = t

    def step_segment(self, s: int, e: int, p, g, out, group: dict, step: int, grad_scale=1.0, d_gscale=None,
                     d_skip=None):
        """Update arena range [s, e).  ``p`` / ``g`` / ``out`` are already sliced to that range; the
        optimizer state tensors (arena-indexed) are sliced here."""
        raise NotImplementedError

    def state_tensors(self):
        return self.state


class FlatAdam(FlatOptimizer):
    state_names = ["exp_avg", "exp_avg_sq"]

    def __init__(self, defaults, adamw=True):
        d = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, bias_correction=True)
        d.update(defaults)
        super().__init__(d)
        self.adamw = adamw

    def step_segment(self, s, e, p, g, out, group, step, grad_scale=1.0, d_gscale=None, d_skip=None):
        b1, b2 = group.get("betas", self.defaults["betas"])
        m, v = self.state["exp_avg"], self.state["exp_avg_sq"]
        if p.device.type == "cpu" and m.device.type == "cpu" and _cpu_adam_available():
            from deepspeed_b200.ops.adam.cpu_adam import cpu_adam_flat
            cpu_adam_flat(p, g, m[s:e], v[s:e], out,
                          lr=group["lr"], beta1=b1, beta2=b2, eps=group.get("eps", self.defaults["eps"]),
                          weight_decay=group.get("weight_decay", 0.0), step=step, adamw=self.adamw,
                          bias_correction=group.get("bias_correction", True), grad_scale=grad_scale,
                          d_gscale=d_gscale, d_skip=d_skip)
            return
        flat_ops.adam_flat(p, g, m[s:e], v[s:e], out,
                           lr=group["lr"], beta1=b1, beta2=b2, eps=group.get("eps", self.defaults["eps"]),
                           weight_decay=group.get("weight_decay", 0.0), step=step, adamw=self.adamw,
                           bias_correction=group.get("bias_correction", True), grad_scale=grad_scale,
                           d_gscale=d_gscale, d_skip=d_skip)


def _cpu_adam_available():
    try:
        from deepspeed_b200.ops.adam import cpu_adam  # noqa: F401
        return cpu_adam.available()
    except Exception:
        return False


class FlatLion(FlatOptimizer):
    state_names = ["exp_avg"]

    def __init__(self, defaults):
        d = dict(lr=1e-4, betas=(0.9, 0.99), weight_decay=0.0)
        d.update(defaults)
        super().__init__(d)

    def step_segment(self, s, e, p, g, out, group, step, grad_scale=1.0, d_gscale=None, d_skip=None):
        b1, b2 = group.get("betas", self.defaults["betas"])
        flat_ops.lion_flat(p, g, self.state["exp_avg"][s:e], out,
                           lr=group["lr"], beta1=b1, beta2=b2, weight_decay=group.get("weight_decay", 0.0),
                           grad_scale=grad_scale, d_gscale=d_gscale, d_skip=d_skip)


class FlatAdagrad(FlatOptimizer):
    state_names = ["sum"]

    def __init__(self, defaults):
        d = dict(lr=1e-2, eps=1e-10, weight_decay=0.0)
        d.update(defaults)
        super().__init__(d)

    def step_segment(self, s, e, p, g, out, group, step, grad_scale=1.0, d_gscale=None, d_skip=None):
        gs = grad_scale * (float(d_gscale.item()) if d_gscale is not None else 1.0)
        if d_skip is not None and int(d_skip.item()):
            return
        flat_ops.adagrad_flat(p, g, self.state["sum"][s:e], out,
                              lr=group["lr"], eps=group.get("eps", self.defaults["eps"]),
                              weight_decay=group.get("weight_decay", 0.0), grad_scale=gs)


class FlatSGD(FlatOptimizer):
    state_names = ["momentum_buffer"]

    def __init__(self, defaults):
        d = dict(lr=1e-2, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False)
        d.update(defaults)
        super().__init__(d)

    def step_segment(self, s, e, p, g, out, group, step, grad_scale=1.0, d_gscale=None, d_skip=None):
        gs = grad_scale * (float(d_gscale.item()) if d_gscale is not None else 1.0)
        if d_skip is not None and int(d_skip.item()):
            return
        flat_ops.sgd_flat(p, g, self.state["momentum_buffer"][s:e],
                          out, lr=group["lr"],
                          momentum=group.get("momentum", 0.0), dampening=group.get("dampening", 0.0),
                          weight_decay=group.get("weight_decay", 0.0), nesterov=group.get("nesterov", False),
                          first=(step == 1), grad_scale=gs)


class FlatLamb(FlatOptimizer):
    """LAMB needs a per-*tensor* trust ratio, so segments are split at parameter boundaries by the
    caller (``ZeroShardedOptimizer`` passes per-parameter sub-segments when ``per_tensor`` is set).
    Under ZeRO sharding a tensor may straddle ranks; the trust ratio then uses the local piece
    (documented deviation, same as the reference which rejects LAMB under ZeRO)."""
    state_names = ["exp_avg", "exp_avg_sq"]
    per_tensor = True

    def __init__(self, defaults):
        d = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, bias_correction=True, max_coeff=10.0,
                 min_coeff=0.01)
        d.update(defaults)
        super().__init__(d)
        self.lamb_coeffs = []

    def step_segment(self, s, e, p, g, out, group, step, grad_scale=1.0, d_gscale=None, d_skip=None):
        gs = grad_scale * (float(d_gscale.item()) if d_gscale is not None else 1.0)
        if d_skip is not None and int(d_skip.item()):
            return
        b1, b2 = group.get("betas", self.defaults["betas"])
        c = flat_ops.lamb_flat(p, g, self.state["exp_avg"][s:e], self.state["exp_avg_sq"][s:e],
                               out, lr=group["lr"], beta1=b1, beta2=b2,
                               eps=group.get("eps", self.defaults["eps"]), weight_decay=group.get("weight_decay", 0.0),
                               step=step, bias_correction=group.get("bias_correction", True),
                               max_coeff=group.get("max_coeff", self.defaults["max_coeff"]),
                               min_coeff=group.get("min_coeff", self.defaults["min_coeff"]), grad_scale=gs)
        self.lamb_coeffs.append(c)


class TorchOptimizerAdapter(FlatOptimizer):
    """Drive a client ``torch.optim.Optimizer`` over fp32 views of the master arena."""
    fused = False

    def __init__(self, optimizer: torch.optim.Optimizer):
        super().__init__(optimizer.defaults)
        self.optimizer = optimizer
        self.views: List[torch.nn.Parameter] = []

    def bind(self, pieces, n_groups: int):
        """``pieces``: list of ``(group, arena_start, arena_end, fp32_tensor)``; the client's params are
        replaced by one fp32 Parameter per piece."""
        per_group: List[List[torch.nn.Parameter]] = [[] for _ in range(n_groups)]
        self.views = []
        self.ranges = []
        for (g, s, e, t) in pieces:
            if g < 0:
                continue
            p = torch.nn.Parameter(t, requires_grad=True)
            per_group[g].append(p)
            self.views.append(p)
            self.ranges.append((s, e))
        for g, plist in zip(self.optimizer.param_groups, per_group):
            g["params"] = plist
        self.optimizer.state.clear()

    def step_all(self, grad_fp32: torch.Tensor):
        for p, (s, e) in zip(self.views, self.ranges):
            p.grad = grad_fp32[s:e]
        self.optimizer.step()
        for p in self.views:
            p.grad = None


def build_flat_optimizer(name: Optional[str], params: Optional[dict], client_optimizer=None):
    """Map config ``optimizer.type`` (or a client optimizer instance) to a flat optimizer."""
    params = dict(params or {})
    params.pop("torch_adam", None)
    if client_optimizer is not None:
        from deepspeed_b200.ops.adam.fused_adam import FusedAdam
        from deepspeed_b200.ops.adam.cpu_adam import DeepSpeedCPUAdam
        from deepspeed_b200.ops.lion.fused_lion import FusedLion
        if isinstance(client_optimizer, (FusedAdam, DeepSpeedCPUAdam)):
            return FlatAdam(client_optimizer.defaults, adamw=client_optimizer.adam_w_mode)
        if isinstance(client_optimizer, torch.optim.AdamW) and not client_optimizer.defaults.get("amsgrad", False):
            d = {k: client_optimizer.defaults[k] for k in ("lr", "betas", "eps", "weight_decay")}
            return FlatAdam(d, adamw=True)
        if type(client_optimizer) is torch.optim.Adam and not client_optimizer.defaults.get("amsgrad", False):
            d = {k: client_optimizer.defaults[k] for k in ("lr", "betas", "eps", "weight_decay")}
            return FlatAdam(d, adamw=False)
        if isinstance(client_optimizer, FusedLion):
            return FlatLion(client_optimizer.defaults)
        return TorchOptimizerAdapter(client_optimizer)
    n = (name or "adamw").lower()
    if n in ("adam", "adamw", "muadam", "muadamw"):
        adamw = params.pop("adam_w_mode", n in ("adamw", "muadamw") or True)
        if n in ("adam", "muadam") and "adam_w_mode" not in (params or {}):
            adamw = True  # reference default ADAM_W_MODE_DEFAULT = True
        return FlatAdam(params, adamw=adamw)
    if n == "lion":
        return FlatLion(params)
    if n == "adagrad":
        return FlatAdagrad(params)
    if n in ("sgd", "musgd"):
        return FlatSGD(params)
    if n == "lamb":
        return FlatLamb(params)
    raise ValueError(f"optimizer type {name!r} has no flat implementation")
