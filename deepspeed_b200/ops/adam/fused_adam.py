"""``FusedAdam`` -- multi-tensor Adam/AdamW on sm_90a.

Parity target: reference ``ops/adam/fused_adam.py`` + ``csrc/adam/multi_tensor_adam.cu`` (N1).
One kernel launch updates every tensor of a (dtype-homogeneous) param group: a device-resident
table of tensor descriptors + 64 Ki-element chunk descriptors is built once per group (tensor
addresses are stable) and re-uploaded only when gradients are re-allocated.
"""
import ctypes
import struct

import torch

from deepspeed_b200.ops import native as N
from deepspeed_b200.ops.kernels import flat_ops

_CHUNK = 65536


def multi_tensor_adam(chunk_size, noop_flag, tensor_lists, lr, beta1, beta2, eps, step, adam_w_mode, bias_correction,
                      weight_decay):
    """Functional entry point with the reference's signature (``fused_adam_frontend.cpp:21``):
    ``tensor_lists = [grads, params, exp_avgs, exp_avg_sqs]``."""
    grads, params, ms, vs = tensor_lists
    _launch(params, grads, ms, vs, None, lr, beta1, beta2, eps, step, adam_w_mode, bias_correction, weight_decay,
            skip=noop_flag)


def _build_tables(params, grads, ms, vs, outs, device):
    tdesc = bytearray()
    cdesc = bytearray()
    for i, (p, g, m, v) in enumerate(zip(params, grads, ms, vs)):
        o = outs[i].data_ptr() if outs is not None and outs[i] is not None else 0
        n = p.numel()
        tdesc += struct.pack("<QQQQQq", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), o, n)
        for start in range(0, n, _CHUNK):
            cdesc += struct.pack("<iiq", i, 0, start)
    t = torch.frombuffer(bytes(tdesc), dtype=torch.uint8).to(device, non_blocking=False)
    c = torch.frombuffer(bytes(cdesc), dtype=torch.uint8).to(device, non_blocking=False)
    return t, c, len(cdesc) // 16


def _launch(params, grads, ms, vs, outs, lr, beta1, beta2, eps, step, adam_w_mode, bias_correction, weight_decay,
            grad_scale=1.0, d_gscale=None, skip=None, cache=None):
    if not params:
        return
    dev = params[0].device
    if dev.type != "cuda":
        for i, (p, g, m, v) in enumerate(zip(params, grads, ms, vs)):
            flat_ops.adam_flat(p.view(-1), g.reshape(-1), m.view(-1), v.view(-1),
                               outs[i].view(-1) if outs is not None and outs[i] is not None else None, lr=lr,
                               beta1=beta1, beta2=beta2, eps=eps, weight_decay=weight_decay, step=step,
                               adamw=bool(adam_w_mode), bias_correction=bool(bias_correction), grad_scale=grad_scale,
                               d_gscale=d_gscale, d_skip=skip)
        return
    key = tuple(t.data_ptr() for lst in (params, grads, ms, vs) for t in lst)
    if cache is not None and cache.get("key") == key:
        tt, ct, nchunks = cache["tables"]
    else:
        tt, ct, nchunks = _build_tables(params, grads, ms, vs, outs, dev)
        if cache is not None:
            cache["key"], cache["tables"] = key, (tt, ct, nchunks)
    bc1 = 1.0 - beta1**step if bias_correction else 1.0
    bc2 = 1.0 - beta2**step if bias_correction else 1.0
    odt = N.dt(outs[0]) if outs is not None and outs[0] is not None else N.BF16
    skip_ptr = ctypes.c_void_p(skip.data_ptr()) if skip is not None else ctypes.c_void_p(0)
    gs_ptr = ctypes.c_void_p(d_gscale.data_ptr()) if d_gscale is not None else ctypes.c_void_p(0)
    rc = N.cuda().dsb_adam_multi(N.ptr(tt), N.ptr(ct), nchunks, N.dt(params[0]), N.dt(grads[0]), N.dt(ms[0]), odt,
                                 N.c_f(lr), N.c_f(beta1), N.c_f(beta2), N.c_f(eps), N.c_f(weight_decay), N.c_f(bc1),
                                 N.c_f(bc2), int(bool(adam_w_mode)), N.c_f(grad_scale), gs_ptr, skip_ptr, N.stream())
    N.check(rc, "adam_multi")


class FusedAdam(torch.optim.Optimizer):
    """Adam/AdamW with one fused launch per (group, dtype).  Arguments as in the reference
    (``ops/adam/fused_adam.py:18``): ``adam_w_mode=True`` selects decoupled weight decay;
    ``set_grad_none`` mirrors apex; ``amsgrad`` is not supported."""

    def __init__(self, params, lr=1e-3, bias_correction=True, betas=(0.9, 0.999), eps=1e-8, adam_w_mode=True,
                 weight_decay=0.0, amsgrad=False, set_grad_none=True):
        if amsgrad:
            raise RuntimeError("FusedAdam does not support the AMSGrad variant.")
        defaults = dict(lr=lr, bias_correction=bias_correction, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.adam_w_mode = 1 if adam_w_mode else 0
        self.set_grad_none = set_grad_none
        self._caches = {}

    def zero_grad(self, set_to_none=None):
        if self.set_grad_none if set_to_none is None else set_to_none:
            for group in self.param_groups:
                for p in group["params"]:
                    p.grad = None
        else:
            super().zero_grad(set_to_none=False)

    @torch.no_grad()
    def step(self, closure=None, grads=None, output_params=None, scale=None, grad_norms=None, grad_scaler=None):
        if any(x is not None for x in (grads, output_params, scale, grad_norms)):
            raise RuntimeError("FusedAdam has been updated: use the loss scaler / ZeRO optimizer for scaling.")
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            if len(group["params"]) == 0:
                continue
            bias_correction = 1 if group["bias_correction"] else 0
            beta1, beta2 = group["betas"]
            group["step"] = group.get("step", 0) + 1
            buckets = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("FusedAdam does not support sparse gradients")
                st = self.state[p]
                if len(st) == 0:
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                b = buckets.setdefault((p.dtype, p.grad.dtype), ([], [], [], []))
                b[0].append(p)
                b[1].append(p.grad.contiguous())
                b[2].append(st["exp_avg"])
                b[3].append(st["exp_avg_sq"])
            for key, (ps, gs, ms, vs) in buckets.items():
                cache = self._caches.setdefault((gi, key), {})
                _launch(ps, gs, ms, vs, None, group["lr"], beta1, beta2, group["eps"], group["step"],
                        self.adam_w_mode, bias_correction, group["weight_decay"], cache=cache)
        return loss
