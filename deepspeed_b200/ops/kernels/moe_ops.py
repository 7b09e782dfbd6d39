"""Python face of the MoE routing / ragged kernels (``csrc/cuda/moe_ragged.cu``) with autograd glue.

``route`` (positions + offsets), ``scatter`` (tokens -> expert-major rows), ``gather`` (weighted combine).
Host tensors use equivalent torch code.  Reference counterparts: ``moe_scatter`` / ``moe_gather`` /
``top_k_gating`` (N9b) and the dense einsum dispatch/combine of ``moe/sharded_moe.py:609,669``.
"""
import ctypes

import torch

from deepspeed_b200.ops import native as N


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def top_k_gating(logits, k, normalize=True):
    """Fused softmax + top-k (inference path, no autograd).  Returns ids [T,k] int32, weights [T,k] fp32,
    counts [E] int32.  Ties go to the lowest expert index.  A row whose softmax is not finite (a NaN or +inf logit, or no
    finite logit) routes to experts 0..k-1 with NaN weights."""
    T, E = logits.shape
    if logits.is_cuda:
        ids = torch.empty(T, k, dtype=torch.int32, device=logits.device)
        w = torch.empty(T, k, dtype=torch.float32, device=logits.device)
        counts = torch.zeros(E, dtype=torch.int32, device=logits.device)
        rc = N.cuda().dsb_top_k_gating(_p(logits.contiguous()), _p(ids), _p(w), _p(counts), ctypes.c_void_p(0), T, E, k,
                                       int(normalize), N.dt(logits), N.stream())
        N.check(rc, "top_k_gating")
        return ids, w, counts
    probs = torch.softmax(logits.float(), dim=-1)
    w, ids = torch.sort(probs, dim=-1, descending=True, stable=True)  # stable: ties to the lowest index
    w, ids = w[:, :k].contiguous(), ids[:, :k].contiguous()
    if normalize:
        w = w / w.sum(-1, keepdim=True)
    # a NaN or +inf logit, or a row without a finite logit, leaves nothing to rank (the kernel's contract): experts
    # 0..k-1 with NaN weights
    bad = torch.isnan(probs).any(-1)
    if bool(bad.any()):
        ids[bad] = torch.arange(k, dtype=ids.dtype)
        w[bad] = float("nan")
    counts = torch.bincount(ids.reshape(-1), minlength=E).to(torch.int32)
    return ids.to(torch.int32), w, counts


def route(expert_ids, num_experts, counts=None):
    """positions [T*k] (slot inside the expert, token-major order), counts [E], offsets [E+1].  Passing the ``counts`` the
    gating kernel already produced avoids ``torch.bincount`` (which synchronises and cannot be graph-captured)."""
    flat = expert_ids.reshape(-1).to(torch.int32).contiguous()
    n = flat.numel()
    dev = flat.device
    if flat.is_cuda:
        if counts is None:
            counts = torch.bincount(flat, minlength=num_experts).to(torch.int32)
        positions = torch.empty(n, dtype=torch.int32, device=dev)
        offsets = torch.empty(num_experts + 1, dtype=torch.int32, device=dev)
        rc = N.cuda().dsb_moe_assign_positions(_p(flat), _p(counts), _p(positions), _p(offsets), n, num_experts,
                                               N.stream())
        N.check(rc, "moe_assign_positions")
        return positions, counts, offsets
    onehot = torch.nn.functional.one_hot(flat.long(), num_experts)
    positions = ((onehot.cumsum(0) - 1) * onehot).sum(1).to(torch.int32)
    counts = onehot.sum(0).to(torch.int32)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int32), counts.cumsum(0).to(torch.int32)])
    return positions, counts, offsets


def _slots(expert_ids, positions, offsets, capacity):
    e = expert_ids.reshape(-1).long()
    pos = positions.long()
    if capacity > 0:
        slot = e * capacity + pos
        return torch.where(pos < capacity, slot, torch.full_like(slot, -1)).to(torch.int32)
    return (offsets.long()[e] + pos).to(torch.int32)


class _Scatter(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, expert_ids, positions, offsets, k, capacity, out_rows):
        T, H = x.shape
        n = T * k
        out = torch.zeros(out_rows, H, dtype=x.dtype, device=x.device)
        if x.is_cuda:
            slots = torch.empty(n, dtype=torch.int32, device=x.device)
            rc = N.cuda().dsb_moe_scatter(_p(x.contiguous()), _p(out), _p(expert_ids), _p(positions), _p(offsets),
                                          _p(slots), n, k, H, capacity, N.dt(x), N.stream())
            N.check(rc, "moe_scatter")
        else:
            slots = _slots(expert_ids, positions, offsets, capacity)
            ok = slots >= 0
            src = torch.arange(n, device=x.device) // k
            out[slots[ok].long()] = x[src[ok]]
        ctx.save_for_backward(slots)
        ctx.k, ctx.T = k, T
        ctx.mark_non_differentiable(slots)
        return out, slots

    @staticmethod
    def backward(ctx, dout, _):
        (slots, ) = ctx.saved_tensors
        k, T = ctx.k, ctx.T
        ones = torch.ones(T * k, dtype=torch.float32, device=dout.device)
        dx = gather_rows(dout.contiguous(), ones, slots, T, k)
        return dx, None, None, None, None, None, None


def gather_rows(expert_out, weights, slots, T, k):
    """y[t] = sum_k weights[t,k] * expert_out[slots[t*k+k']] (no autograd)."""
    H = expert_out.shape[1]
    if expert_out.is_cuda:
        y = torch.empty(T, H, dtype=expert_out.dtype, device=expert_out.device)
        rc = N.cuda().dsb_moe_gather(_p(expert_out), _p(y), _p(weights.contiguous().float()), _p(slots), T, k, H,
                                     N.dt(expert_out), N.stream())
        N.check(rc, "moe_gather")
        return y
    s = slots.long().reshape(T, k)
    w = weights.reshape(T, k).float()
    rows = expert_out[s.clamp(min=0)].float() * (s >= 0)[..., None]
    return (rows * w[..., None]).sum(1).to(expert_out.dtype)


class _Gather(torch.autograd.Function):

    @staticmethod
    def forward(ctx, expert_out, weights, slots, T, k):
        ctx.save_for_backward(expert_out, weights, slots)
        ctx.T, ctx.k = T, k
        return gather_rows(expert_out.contiguous(), weights.reshape(-1), slots, T, k)

    @staticmethod
    def backward(ctx, dy):
        expert_out, weights, slots = ctx.saved_tensors
        T, k = ctx.T, ctx.k
        H = expert_out.shape[1]
        n = T * k
        w = weights.reshape(-1).float().contiguous()
        if dy.is_cuda:
            d_eo = torch.zeros_like(expert_out)
            dw = torch.empty(n, dtype=torch.float32, device=dy.device)
            rc = N.cuda().dsb_moe_gather_bwd(_p(dy.contiguous()), _p(expert_out), _p(d_eo), _p(dw), _p(w), _p(slots), n, k,
                                             H, N.dt(dy), N.stream())
            N.check(rc, "moe_gather_bwd")
        else:
            s = slots.long()
            ok = s >= 0
            src = torch.arange(n, device=dy.device) // k
            d_eo = torch.zeros_like(expert_out)
            d_eo[s[ok]] = (dy[src[ok]].float() * w[ok, None]).to(expert_out.dtype)
            dw = torch.zeros(n, dtype=torch.float32, device=dy.device)
            dw[ok] = (dy[src[ok]].float() * expert_out[s[ok]].float()).sum(-1)
        return d_eo, dw.reshape(weights.shape).to(weights.dtype), None, None, None


def scatter(x, expert_ids, positions, offsets, k, capacity, out_rows):
    return _Scatter.apply(x, expert_ids.reshape(-1).to(torch.int32).contiguous(), positions, offsets, k, capacity,
                          out_rows)


def gather(expert_out, weights, slots, T, k):
    return _Gather.apply(expert_out, weights, slots, T, k)
