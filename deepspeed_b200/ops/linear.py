"""Linear layers that cooperate with the ZeRO flat gradient buffers.

* :func:`flat_linear` -- ``y = x W^T (+ b)``; its backward computes ``dW`` with an ``out=`` GEMM directly
  into the unit's flat gradient buffer (``ZeroShardedOptimizer.grad_view_for``) and never saves the
  gathered weight (it is re-read from the parameter at backward time, so ZeRO-3 can release it after
  forward).  Role parity: reference ``runtime/zero/linear.py:50 LinearFunctionForZeroStage3`` (P17)
  plus the bucket copy in ``stage3.py:1275 __add_grad_to_ipg_bucket`` which this design removes.
* :func:`chunked_linear_xent` -- LM head + softmax cross-entropy over token chunks; logits gradient is
  produced in place by the fused kernel, ``dh`` and ``dW`` are accumulated per chunk, so the
  ``[tokens, vocab]`` logits tensor is never materialised (role: reference ``FPDT_LogitsLoss``).
"""
import torch
import torch.nn.functional as F

from deepspeed_b200.ops.kernels.transformer_ops import softmax_xent_fwd_bwd, xent_valid


def _zo_of(w):
    ref = getattr(w, "_ds_zero", None)
    zo = ref() if ref is not None else None
    if zo is None or getattr(w, "ds_no_direct_grad", False) or not w.requires_grad:
        return None
    return zo


def _gemm(a, b_t):
    """a [M, K] @ b_t[N, K]^T -> [M, N] through the active GEMM backend."""
    from deepspeed_b200.ops import gemm
    return gemm.matmul_nt(a, b_t)


class _FlatLinearFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.weight_ref = weight
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x)
        x2 = x.reshape(-1, x.shape[-1])
        y = _gemm(x2, weight)
        if bias is not None:
            y = y + bias
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        (x, ) = ctx.saved_tensors
        w = ctx.weight_ref
        dy2 = dy.reshape(-1, dy.shape[-1])
        x2 = x.reshape(-1, x.shape[-1])
        dx = None
        if ctx.needs_input_grad[0]:
            from deepspeed_b200.ops import gemm
            dx = gemm.matmul_nn(dy2, w).view(x.shape)
        dw = None
        if ctx.needs_input_grad[1]:
            zo = _zo_of(w)
            if zo is not None:
                gv = zo.grad_view_for(w)
                if gv.dtype == dy2.dtype:
                    from deepspeed_b200.ops import gemm
                    # first micro step: overwrite; later ones: accumulate in the GEMM epilogue (no addmm, no memset)
                    gemm.matmul_tn(dy2, x2, out=gv, accumulate=not zo.grad_is_fresh(w))
                else:
                    g = torch.mm(dy2.t(), x2)
                    gv.copy_(g) if zo.grad_is_fresh(w) else gv.add_(g)
                zo.mark_grad_ready(w)
            else:
                dw = torch.mm(dy2.t(), x2)
        db = dy2.sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        return dx, dw, db


def flat_linear(x, weight, bias=None):
    if not torch.is_grad_enabled() or not (x.requires_grad or weight.requires_grad):
        x2 = x.reshape(-1, x.shape[-1])
        y = _gemm(x2, weight)
        if bias is not None:
            y = y + bias
        return y.view(*x.shape[:-1], weight.shape[0])
    return _FlatLinearFn.apply(x, weight, bias)


def _write_weight_grad(w, dy2, x2):
    """dW = dy2^T x2 for parameter ``w``: straight into the ZeRO flat gradient view when there is one (returns None),
    else returned for autograd."""
    from deepspeed_b200.ops import gemm
    zo = _zo_of(w)
    if zo is None:
        return gemm.matmul_tn(dy2, x2)
    gv = zo.grad_view_for(w)
    if gv.dtype == dy2.dtype:
        gemm.matmul_tn(dy2, x2, out=gv, accumulate=not zo.grad_is_fresh(w))
    else:
        g = torch.mm(dy2.t(), x2)
        gv.copy_(g) if zo.grad_is_fresh(w) else gv.add_(g)
    zo.mark_grad_ready(w)
    return None


class _SwiGLUMLPFn(torch.autograd.Function):
    """``down(silu(gate(x)) * up(x))`` as ONE autograd node over three GEMM launches per direction:

    forward   gate|up GEMM with the SwiGLU applied in its epilogue (gate|up saved for backward from the same
              accumulators) -> down GEMM;
    backward  ``dY W_down`` GEMM with the SwiGLU *backward* applied in its epilogue (the ``[tokens, I]`` intermediate
              gradient never reaches memory) -> dW_down, dX and dW_gate_up GEMMs, weight gradients written (or
              accumulated, GAS > 1) directly into the ZeRO flat gradient views.
    Reference role: the three ``nn.Linear`` + ``ACT2FN`` of an HF MLP block / ``csrc/transformer/gelu_kernels.cu``
    (``fused_bias_gelu``) -- there the activation is a separate pass over the intermediate tensor."""

    @staticmethod
    def forward(ctx, x, w_gu, w_down):
        from deepspeed_b200.ops import gemm
        x2 = x.reshape(-1, x.shape[-1])
        need_grad = any(ctx.needs_input_grad)  # (grad mode is off inside Function.forward)
        act, gu = gemm.gate_up_swiglu(x2, w_gu, save_gate_up=need_grad)
        y = gemm.matmul_nt(act, w_down)
        ctx.w_gu, ctx.w_down = w_gu, w_down
        ctx.save_for_backward(x2, gu, act)
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], w_down.shape[0])

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops import gemm
        x2, gu, act = ctx.saved_tensors
        w_gu, w_down = ctx.w_gu, ctx.w_down
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dgu = gemm.down_dx_dswiglu(dy2, w_down, gu)
        dw_down = _write_weight_grad(w_down, dy2, act) if ctx.needs_input_grad[2] else None
        dx = gemm.matmul_nn(dgu, w_gu).view(ctx.x_shape) if ctx.needs_input_grad[0] else None
        dw_gu = _write_weight_grad(w_gu, dgu, x2) if ctx.needs_input_grad[1] else None
        return dx, dw_gu, dw_down


def swiglu_mlp(x, w_gate_up, w_down):
    """Fused SwiGLU MLP block (no biases): see :class:`_SwiGLUMLPFn`."""
    return _SwiGLUMLPFn.apply(x, w_gate_up, w_down)


class _GroupedSwiGLUFn(torch.autograd.Function):
    """Stacked SwiGLU experts on a capacity-padded dispatch buffer ``x [E, C, H]`` with ``w13 [E, 2I, H]``, ``w2 [E, H, I]``
    (the MoE training path, reference ``moe/experts.py:13`` + ``sharded_moe.py:586``): per expert the same three fused GEMM
    launches per direction as :class:`_SwiGLUMLPFn`; the per-expert weight gradients (K = that expert's token rows) land
    in the expert's slice of the stacked parameter's flat ZeRO gradient view."""

    @staticmethod
    def forward(ctx, x, w13, w2):
        from deepspeed_b200.ops import gemm
        E, C, H = x.shape
        need_grad = any(ctx.needs_input_grad)
        y = torch.empty(E, C, w2.shape[1], dtype=x.dtype, device=x.device)
        gus, acts = [], []
        for e in range(E):
            act, gu = gemm.gate_up_swiglu(x[e], w13[e], save_gate_up=need_grad)
            gemm.matmul_nt(act, w2[e], out=y[e])
            gus.append(gu)
            acts.append(act)
        ctx.w13, ctx.w2 = w13, w2
        ctx.saved = (x, gus, acts) if need_grad else None
        return y

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops import gemm
        x, gus, acts = ctx.saved
        ctx.saved = None
        w13, w2 = ctx.w13, ctx.w2
        E = x.shape[0]
        dy = dy.contiguous()
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        views = {}
        for w, need in ((w13, ctx.needs_input_grad[1]), (w2, ctx.needs_input_grad[2])):
            if not need:
                views[id(w)] = (None, None, False)
                continue
            zo = _zo_of(w)
            if zo is not None and zo.grad_view_for(w).dtype == dy.dtype:
                views[id(w)] = (zo, zo.grad_view_for(w), not zo.grad_is_fresh(w))
            else:
                views[id(w)] = (None, torch.empty_like(w), False)
        for e in range(E):
            dgu = gemm.down_dx_dswiglu(dy[e], w2[e], gus[e])
            _, g2, acc2 = views[id(w2)]
            if g2 is not None:
                gemm.matmul_tn(dy[e], acts[e], out=g2[e], accumulate=acc2)
            if dx is not None:
                gemm.matmul_nn(dgu, w13[e], out=dx[e])
            _, g13, acc13 = views[id(w13)]
            if g13 is not None:
                gemm.matmul_tn(dgu, x[e], out=g13[e], accumulate=acc13)
            gus[e] = acts[e] = None
        outs = []
        for w in (w13, w2):
            zo, g, _ = views[id(w)]
            if zo is not None:
                zo.mark_grad_ready(w)
                outs.append(None)
            else:
                outs.append(g)
        return dx, outs[0], outs[1]


def grouped_swiglu_mlp(x, w13, w2):
    return _GroupedSwiGLUFn.apply(x, w13, w2)


class _ChunkedLinearXent(torch.autograd.Function):

    @staticmethod
    def forward(ctx, h, weight, labels, chunk, ignore_index, assumed_scale):
        from deepspeed_b200.ops import gemm
        T, H = h.shape
        n_valid = xent_valid(labels, weight.shape[0], ignore_index).sum().clamp(min=1).to(torch.float32)
        inv_n = (assumed_scale / n_valid).reshape(1)  # device scalar: no host sync
        need_dh = h.requires_grad
        need_dw = weight.requires_grad
        dh = torch.empty_like(h) if need_dh else None
        # Where the weight gradient accumulates over the token chunks: straight in the ZeRO flat gradient view when this is
        # the first contribution of the micro step (the chunk GEMMs' epilogues store / accumulate there: no [V, H] scratch,
        # no copy); otherwise a per-call scratch (several forwards may precede their backwards, so it cannot be shared).
        dw_tmp, direct = None, False
        if need_dw:
            zo = _zo_of(weight)
            if zo is not None and zo.grad_is_fresh(weight):
                gv = zo.grad_view_for(weight)
                if gv.dtype == weight.dtype and weight.is_cuda:
                    dw_tmp, direct = gv, True
            if dw_tmp is None:
                dw_tmp = torch.empty(weight.shape, dtype=weight.dtype, device=weight.device)
        total = torch.zeros((), dtype=torch.float32, device=h.device)
        first = True
        for s in range(0, T, chunk):
            e = min(s + chunk, T)
            hc = h[s:e]
            logits = _gemm(hc, weight)  # [c, V]
            loss_rows, grad = softmax_xent_fwd_bwd(logits, labels[s:e].contiguous(), 1.0, inv_n, ignore_index, True)
            total = total + loss_rows.sum()
            if need_dh:
                gemm.matmul_nn(grad, weight, out=dh[s:e])
            if need_dw:
                gemm.matmul_tn(grad, hc, out=dw_tmp, accumulate=not first)  # accumulate in the GEMM epilogue
            first = False
        ctx.weight_ref = weight
        ctx.assumed_scale = assumed_scale
        ctx.need_dw = need_dw
        ctx.dh = dh
        ctx.dw_tmp = dw_tmp
        ctx.direct = direct
        return total / n_valid

    @staticmethod
    def backward(ctx, dloss):
        w = ctx.weight_ref
        r = (dloss / ctx.assumed_scale).to(torch.float32)  # == 1 when the engine's multiplier was assumed
        dh = None
        if ctx.dh is not None:
            dh = ctx.dh.mul_(r.to(ctx.dh.dtype))
        dw = None
        if ctx.need_dw:
            zo = _zo_of(w)
            if ctx.direct and zo is not None:
                # the gradient already sits in the flat view; fold the (almost always unit) upstream factor in place -- the
                # kernel returns before touching memory when the device-resident factor is exactly 1
                from deepspeed_b200.ops.kernels import flat_ops
                flat = ctx.dw_tmp.view(-1)
                flat_ops.scale_cast(flat, flat, scale=1.0, d_scale=r.reshape(1))
                zo.mark_grad_ready(w)
            elif zo is not None:
                gv = zo.grad_view_for(w)
                if zo.grad_is_fresh(w):
                    torch.mul(ctx.dw_tmp, r.to(ctx.dw_tmp.dtype), out=gv) if gv.dtype == ctx.dw_tmp.dtype else gv.copy_(
                        ctx.dw_tmp.float() * r)
                else:
                    gv.add_((ctx.dw_tmp.float() * r).to(gv.dtype))
                zo.mark_grad_ready(w)
            else:
                dw = ctx.dw_tmp * r.to(ctx.dw_tmp.dtype)
        ctx.dh = None
        ctx.dw_tmp = None
        return dh, dw, None, None, None, None


def chunked_linear_xent(h, weight, labels, chunk=2048, ignore_index=-100, assumed_scale=1.0):
    """Mean cross entropy of ``softmax(h W^T)`` vs ``labels`` without materialising the logits."""
    if not torch.is_grad_enabled():
        total = torch.zeros((), dtype=torch.float32, device=h.device)
        n = xent_valid(labels, weight.shape[0], ignore_index).sum().clamp(min=1)
        for s in range(0, h.shape[0], chunk):
            e = min(s + chunk, h.shape[0])
            logits = _gemm(h[s:e], weight)
            rows, _ = softmax_xent_fwd_bwd(logits, labels[s:e].contiguous(), 1.0, None, ignore_index, False)
            total = total + rows.sum()
        return total / n
    return _ChunkedLinearXent.apply(h, weight, labels, chunk, ignore_index, float(assumed_scale) or 1.0)
