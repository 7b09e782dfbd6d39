"""Flat-buffer optimizer / gradient ops (python face of ``csrc/cuda/optim.cu``).

On CUDA tensors these call the sm_90a kernels (a missing native library is a hard error).  On
host tensors they run an equivalent pure-torch implementation so the gloo/CPU test tier exercises
the same engine logic.  Reference counterparts: ``ops/adam/fused_adam.py`` (N1),
``runtime/utils.py`` norm/clip helpers, ``stage3.py:2178 unscale_and_clip_grads``.
"""
import ctypes
import math

import torch

from deepspeed_b200.ops import native as N


def _on_cuda(t):
    return t is not None and t.is_cuda


def _devptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


# ------------------------------------------------------------------------------------------------
# Adam / AdamW on flat buffers
# ------------------------------------------------------------------------------------------------
def adam_flat(p, g, m, v, out=None, *, lr, beta1, beta2, eps, weight_decay, step, adamw=True, bias_correction=True,
              grad_scale=1.0, d_gscale=None, d_skip=None):
    """In-place Adam on flat 1-D buffers.  ``p`` master (fp32 or 16-bit), ``g`` grads, ``m``/``v``
    states, ``out`` optional low-precision copy of the updated params.  ``d_gscale`` (fp32[1]) and
    ``d_skip`` (int32[1]) are optional device scalars: multiply grads / skip the whole update."""
    n = p.numel()
    if n == 0:
        return
    bc1 = 1.0 - beta1**step if bias_correction else 1.0
    bc2 = 1.0 - beta2**step if bias_correction else 1.0
    if _on_cuda(p):
        rc = N.cuda().dsb_adam_flat(N.ptr(p), N.ptr(g), N.ptr(m), N.ptr(v), N.ptr(out), N.c_i64(n), N.dt(p), N.dt(g),
                                    N.dt(m), N.dt(out) if out is not None else N.BF16, N.c_f(lr), N.c_f(beta1),
                                    N.c_f(beta2), N.c_f(eps), N.c_f(weight_decay), N.c_f(bc1), N.c_f(bc2),
                                    int(bool(adamw)), N.c_f(grad_scale), _devptr(d_gscale), _devptr(d_skip),
                                    N.stream())
        N.check(rc, "adam_flat")
        return
    # ---- host reference path ----
    if d_skip is not None and int(d_skip.item()) != 0:
        return
    gs = grad_scale * (float(d_gscale.item()) if d_gscale is not None else 1.0)
    pf = p.float()
    gf = g.float() * gs
    mf, vf = m.float(), v.float()
    if not adamw and weight_decay != 0:
        gf = gf + weight_decay * pf
    mf.mul_(beta1).add_(gf, alpha=1 - beta1)
    vf.mul_(beta2).addcmul_(gf, gf, value=1 - beta2)
    upd = (mf / bc1) / ((vf / bc2).sqrt() + eps)
    if adamw and weight_decay != 0:
        upd = upd + weight_decay * pf
    pf.add_(upd, alpha=-lr)
    p.copy_(pf)
    m.copy_(mf)
    v.copy_(vf)
    if out is not None:
        out.copy_(pf)


def lion_flat(p, g, m, out=None, *, lr, beta1, beta2, weight_decay, grad_scale=1.0, d_gscale=None, d_skip=None):
    n = p.numel()
    if n == 0:
        return
    if _on_cuda(p):
        rc = N.cuda().dsb_lion_flat(N.ptr(p), N.ptr(g), N.ptr(m), N.ptr(out), N.c_i64(n), N.dt(p), N.dt(g), N.dt(m),
                                    N.dt(out) if out is not None else N.BF16, N.c_f(lr), N.c_f(beta1), N.c_f(beta2),
                                    N.c_f(weight_decay), N.c_f(grad_scale), _devptr(d_gscale), _devptr(d_skip),
                                    N.stream())
        N.check(rc, "lion_flat")
        return
    if d_skip is not None and int(d_skip.item()) != 0:
        return
    gs = grad_scale * (float(d_gscale.item()) if d_gscale is not None else 1.0)
    pf, gf, mf = p.float(), g.float() * gs, m.float()
    c = mf * beta1 + gf * (1 - beta1)
    pf.mul_(1 - lr * weight_decay).add_(torch.sign(c), alpha=-lr)
    mf.mul_(beta2).add_(gf, alpha=1 - beta2)
    p.copy_(pf)
    m.copy_(mf)
    if out is not None:
        out.copy_(pf)


def adagrad_flat(p, g, h, out=None, *, lr, eps, weight_decay, grad_scale=1.0):
    n = p.numel()
    if n == 0:
        return
    if _on_cuda(p):
        rc = N.cuda().dsb_adagrad_flat(N.ptr(p), N.ptr(g), N.ptr(h), N.ptr(out), N.c_i64(n), N.dt(p), N.dt(g),
                                       N.dt(out) if out is not None else N.BF16, N.c_f(lr), N.c_f(eps),
                                       N.c_f(weight_decay), N.c_f(grad_scale), N.stream())
        N.check(rc, "adagrad_flat")
        return
    pf, gf = p.float(), g.float() * grad_scale
    if weight_decay != 0:
        gf = gf + weight_decay * pf
    h.addcmul_(gf, gf)
    pf.addcdiv_(gf, h.sqrt() + eps, value=-lr)
    p.copy_(pf)
    if out is not None:
        out.copy_(pf)


def sgd_flat(p, g, buf, out=None, *, lr, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, first=False,
             grad_scale=1.0):
    n = p.numel()
    if n == 0:
        return
    if _on_cuda(p):
        rc = N.cuda().dsb_sgd_flat(N.ptr(p), N.ptr(g), N.ptr(buf), N.ptr(out), N.c_i64(n), N.dt(p), N.dt(g),
                                   N.dt(out) if out is not None else N.BF16, N.c_f(lr), N.c_f(momentum),
                                   N.c_f(dampening), N.c_f(weight_decay), int(nesterov), int(first), N.c_f(grad_scale),
                                   N.stream())
        N.check(rc, "sgd_flat")
        return
    pf, gf = p.float(), g.float() * grad_scale
    if weight_decay != 0:
        gf = gf + weight_decay * pf
    if momentum != 0:
        if first:
            buf.copy_(gf)
        else:
            buf.mul_(momentum).add_(gf, alpha=1 - dampening)
        gf = gf + momentum * buf if nesterov else buf
    pf.add_(gf, alpha=-lr)
    p.copy_(pf)
    if out is not None:
        out.copy_(pf)


def lamb_flat(p, g, m, v, out=None, *, lr, beta1, beta2, eps, weight_decay, step, bias_correction=True, max_coeff=10.0,
              min_coeff=0.01, grad_scale=1.0):
    """LAMB on one flat tensor; returns the trust-ratio coefficient tensor (fp32[1])."""
    n = p.numel()
    bc1 = 1.0 - beta1**step if bias_correction else 1.0
    bc2 = 1.0 - beta2**step if bias_correction else 1.0
    if _on_cuda(p):
        lib = N.cuda()
        grid = lib.dsb_lamb_grid(N.c_i64(n))
        upd = torch.empty(n, dtype=torch.float32, device=p.device)
        partials = torch.empty(2 * grid, dtype=torch.float32, device=p.device)
        coeff = torch.empty(1, dtype=torch.float32, device=p.device)
        rc = lib.dsb_lamb_flat(N.ptr(p), N.ptr(g), N.ptr(m), N.ptr(v), N.ptr(out), N.ptr(upd), N.ptr(partials),
                               N.ptr(coeff), N.c_i64(n), N.dt(p), N.dt(g), N.dt(out) if out is not None else N.BF16,
                               N.c_f(lr), N.c_f(beta1), N.c_f(beta2), N.c_f(eps), N.c_f(weight_decay), N.c_f(bc1),
                               N.c_f(bc2), N.c_f(max_coeff), N.c_f(min_coeff), N.c_f(grad_scale), N.stream())
        N.check(rc, "lamb_flat")
        return coeff
    pf, gf = p.float(), g.float() * grad_scale
    m.mul_(beta1).add_(gf, alpha=1 - beta1)
    v.mul_(beta2).addcmul_(gf, gf, value=1 - beta2)
    u = (m / bc1) / ((v / bc2).sqrt() + eps) + weight_decay * pf
    pn, un = pf.norm(), u.norm()
    coeff = torch.ones((), dtype=torch.float32)
    if pn != 0 and un != 0:
        coeff = (pn / un).clamp(min_coeff, max_coeff)
    pf.add_(u, alpha=-lr * float(coeff))
    p.copy_(pf)
    if out is not None:
        out.copy_(pf)
    return coeff.reshape(1)


# ------------------------------------------------------------------------------------------------
# gradient utilities
# ------------------------------------------------------------------------------------------------
class GradStats:
    """Device-resident accumulator: sum of squares, inf/nan flag, clip coefficient, skip flag.

    All members are 1-element device tensors so the overflow / clip decision never syncs the host.
    """

    def __init__(self, device):
        self.device = torch.device(device)
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=device)
        self.found_inf = torch.zeros(1, dtype=torch.int32, device=device)
        self.gscale = torch.ones(1, dtype=torch.float32, device=device)
        self.skip = torch.zeros(1, dtype=torch.int32, device=device)
        self.norm = torch.zeros(1, dtype=torch.float32, device=device)
        self._partials = None

    def reset(self):
        self.sumsq.zero_()
        self.found_inf.zero_()

    def partials(self, n):
        if self.device.type != "cuda":
            return None
        need = N.cuda().dsb_sumsq_grid(N.c_i64(n))
        if self._partials is None or self._partials.numel() < need:
            self._partials = torch.empty(max(need, 1024), dtype=torch.float32, device=self.device)
        return self._partials

    def accumulate(self, x):
        """sumsq += ||x||^2 ; found_inf |= any(!finite(x))."""
        n = x.numel()
        if n == 0:
            return
        if x.is_cuda:
            rc = N.cuda().dsb_sumsq(N.ptr(x), N.c_i64(n), N.dt(x), N.ptr(self.partials(n)), N.ptr(self.sumsq),
                                    N.ptr(self.found_inf), 1, N.stream())
            N.check(rc, "sumsq")
        else:
            xf = x.float()
            self.sumsq += (xf * xf).sum()
            if not torch.isfinite(xf).all():
                self.found_inf.fill_(1)

    def finalize(self, inv_loss_scale=1.0, max_norm=0.0):
        """Compute gscale = inv_loss_scale * min(1, max_norm/(norm+eps)); skip = overflow."""
        if self.device.type == "cuda":
            rc = N.cuda().dsb_clip_coeff(N.ptr(self.sumsq), N.ptr(self.found_inf), N.c_f(inv_loss_scale),
                                         N.c_f(max_norm), N.ptr(self.gscale), N.ptr(self.skip), N.ptr(self.norm),
                                         N.stream())
            N.check(rc, "clip_coeff")
        else:
            ss = float(self.sumsq.item())
            bad = bool(self.found_inf.item()) or not math.isfinite(ss)
            norm = math.sqrt(ss) * inv_loss_scale if not bad else float("inf")
            c = inv_loss_scale
            if max_norm > 0 and not bad:
                clip = max_norm / (norm + 1e-6)
                if clip < 1:
                    c *= clip
            self.gscale.fill_(0.0 if bad else c)
            self.skip.fill_(1 if bad else 0)
            self.norm.fill_(norm)


def scale_cast(x, y, scale=1.0, accumulate=False, d_scale=None):
    """y = scale*x (+ y).  Handles dtype conversion; flat contiguous tensors."""
    n = x.numel()
    assert y.numel() == n
    if n == 0:
        return y
    if x.is_cuda:
        rc = N.cuda().dsb_scale_cast(N.ptr(x), N.ptr(y), N.c_i64(n), N.dt(x), N.dt(y), N.c_f(scale), int(accumulate),
                                     _devptr(d_scale), N.stream())
        N.check(rc, "scale_cast")
        return y
    s = scale * (float(d_scale.item()) if d_scale is not None else 1.0)
    if accumulate:
        y.copy_(y.float() + x.float() * s)
    else:
        y.copy_(x.float() * s)
    return y
