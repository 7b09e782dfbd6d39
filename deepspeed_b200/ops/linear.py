"""Linear layers that cooperate with the ZeRO flat gradient buffers.

* :func:`flat_linear` -- ``y = x W^T (+ b)``; its backward computes ``dW`` with an ``out=`` GEMM directly
  into the unit's flat gradient buffer (``ZeroShardedOptimizer.grad_view_for``) and never saves the
  gathered weight (it is re-read from the parameter at backward time, so ZeRO-3 can release it after
  forward).  Role parity: reference ``runtime/zero/linear.py:50 LinearFunctionForZeroStage3`` (P17)
  plus the bucket copy in ``stage3.py:1275 __add_grad_to_ipg_bucket`` which this design removes.
* :func:`chunked_linear_xent` -- LM head + softmax cross-entropy over token chunks; logits gradient is
  produced in place by the fused kernel, ``dh`` and ``dW`` are accumulated per chunk, so the
  ``[tokens, vocab]`` logits tensor is never materialised (role: reference ``FPDT_LogitsLoss``).
* :func:`embedding` -- the input embedding of a model with a tied LM head: its backward adds into the flat gradient
  view the head's dW already sits in, with the deterministic native embedding backward, and marks the weight ready.
"""
import functools

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


def _weight_grad_sink(w, dtype, into, product, unowned=None):
    """Where the gradient of the 2-D weight ``w`` goes.  With a ZeRO owner it lands in the flat gradient view
    ``grad_view_for(w)``, stored on the micro step's first contribution and accumulated on later ones, and ``w`` is
    marked ready (returns None): ``into(out=view, accumulate=...)`` writes it there when the view has the product's
    ``dtype``; a view of another dtype (fp32 accumulation) takes ``product()`` by copy or add.  Without an owner
    ``unowned()`` (default ``product()``) is returned to autograd.

    Marking a unit's last gradient reduces it, which under ZeRO-3 releases the gathered weights and with the step fused
    into backward rewrites them: a node reads no weight after it has marked all of them."""
    zo = _zo_of(w)
    if zo is None:
        return (unowned or product)()
    gv = zo.grad_view_for(w)
    if gv.dtype == dtype:
        into(out=gv, accumulate=not zo.grad_is_fresh(w))
    else:
        g = product()
        gv.copy_(g) if zo.grad_is_fresh(w) else gv.add_(g)
    zo.mark_grad_ready(w)
    return None


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
        from deepspeed_b200.ops import gemm
        (x, ) = ctx.saved_tensors
        w = ctx.weight_ref
        dy2 = dy.reshape(-1, dy.shape[-1])
        x2 = x.reshape(-1, x.shape[-1])
        dx = gemm.matmul_nn(dy2, w).view(x.shape) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1]:
            # into the view: stored on the first micro step, accumulated in the GEMM epilogue later (no addmm, no memset)
            dw = _weight_grad_sink(w, dy2.dtype, functools.partial(gemm.matmul_tn, dy2, x2),
                                   lambda: torch.mm(dy2.t(), x2))
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


class _SwiGLUMLPFn(torch.autograd.Function):
    """``down(silu(gate(x)) * up(x))`` as ONE autograd node over three GEMM launches per direction:

    forward   gate|up GEMM with the SwiGLU applied in its epilogue (gate|up saved for backward from the same
              accumulators) -> down GEMM;
    backward  ``dY W_down`` GEMM with the SwiGLU *backward* applied in its epilogue (the ``[tokens, I]`` intermediate
              gradient never reaches memory) -> dW_down, dX and dW_gate_up GEMMs, weight gradients written (or
              accumulated, GAS > 1) directly into the ZeRO flat gradient views.
    Only ``x`` and gate|up are saved: the library path's dSwiGLU pass writes ``act`` for dW_down again from the same bf16
    gate|up, bit for bit.  When the gate|up GEMM ran the own fused kernel, whose ``act`` comes from the fp32 accumulators,
    ``act`` is saved too.

    ``recompute``: the forward is a replay for backward (activation checkpointing) that stops at what backward reads --
    gate|up, and ``act`` where it is saved -- and returns a placeholder of the output's shape with no data: backward never
    reads the output, so the down GEMM (and, on the library path, the SwiGLU pass) is not run.
    Reference role: the three ``nn.Linear`` + ``ACT2FN`` of an HF MLP block / ``csrc/transformer/gelu_kernels.cu``
    (``fused_bias_gelu``) -- there the activation is a separate pass over the intermediate tensor."""

    @staticmethod
    def forward(ctx, x, w_gu, w_down, recompute):
        from deepspeed_b200.ops import gemm
        x2 = x.reshape(-1, x.shape[-1])
        out_shape = (*x.shape[:-1], w_down.shape[0])
        if recompute:
            if gemm.gate_up_swiglu_in_tree(x2, w_gu):
                act, gu = gemm.gate_up_swiglu(x2, w_gu)
            else:
                act, gu = None, gemm.matmul_nt(x2, w_gu)
            y = x2.new_empty(1).expand(out_shape)
        else:
            need_grad = any(ctx.needs_input_grad)  # (grad mode is off inside Function.forward)
            act, gu = gemm.gate_up_swiglu(x2, w_gu, save_gate_up=need_grad)
            y = gemm.matmul_nt(act, w_down).view(out_shape)
            if not gemm.gate_up_swiglu_in_tree(x2, w_gu):
                act = None
        ctx.w_gu, ctx.w_down = w_gu, w_down
        ctx.save_for_backward(x2, gu, act)
        ctx.x_shape = x.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops import gemm
        x2, gu, act = ctx.saved_tensors
        w_gu, w_down = ctx.w_gu, ctx.w_down
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        act_out = None
        if act is None and ctx.needs_input_grad[2]:
            act = act_out = torch.empty(gu.shape[0], gu.shape[1] // 2, dtype=gu.dtype, device=gu.device)
        dgu = gemm.down_dx_dswiglu(dy2, w_down, gu, act_out=act_out)

        def weight_grad(w, a, b):  # dW = a^T b
            mm = functools.partial(gemm.matmul_tn, a, b)
            return _weight_grad_sink(w, a.dtype, mm, lambda: torch.mm(a.t(), b), unowned=mm)

        dw_down = weight_grad(w_down, dy2, act) if ctx.needs_input_grad[2] else None
        dx = gemm.matmul_nn(dgu, w_gu).view(ctx.x_shape) if ctx.needs_input_grad[0] else None
        dw_gu = weight_grad(w_gu, dgu, x2) if ctx.needs_input_grad[1] else None
        return dx, dw_gu, dw_down, None


def swiglu_mlp(x, w_gate_up, w_down, recompute=False):
    """Fused SwiGLU MLP block (no biases): see :class:`_SwiGLUMLPFn`.  ``recompute=True`` is the trimmed replay of an
    activation-checkpointed block: its output holds no data, only its gradient is used."""
    return _SwiGLUMLPFn.apply(x, w_gate_up, w_down, recompute)


def _fp8_native(x2, *ws, inter=None) -> bool:
    """Whether the FP8 nodes run the wgmma kernels: CUDA bf16 rows ``x2 [T, K]`` and weights, every dimension (and, for
    the SwiGLU block, ``2 I``) a multiple of 16 -- each is a K of some product or the row count of a transposed cast --
    and ``I % 64 == 0`` for the SwiGLU epilogue's tile."""
    ts = (x2, ) + ws
    if not all(t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 for t in ts):
        return False
    if any(d % 16 for t in ts for d in t.shape):
        return False
    return inter is None or inter % 64 == 0


FP8_RECIPES = ("tensorwise", "blockwise")


def _check_recipe(recipe):
    if recipe not in FP8_RECIPES:
        raise ValueError(f"fp8 recipe must be one of {FP8_RECIPES}, got {recipe!r}")


def _fp8_cast4(native, block):
    """``cast(x, fmt, row, col) -> (q, sq, qt, sqt)`` for either recipe (``block``: blockwise), on the cast kernels
    (``native``) or the torch reference: the modes of :func:`fp8.quantize_blockwise`; under the tensorwise recipe a mode
    only asks for its copy, and both copies share the one scale."""
    from deepspeed_b200.ops import fp8
    if block:
        return fp8.quantize_blockwise if native else fp8.quantize_blockwise_reference
    q = fp8.quantize_tensorwise if native else fp8.quantize_reference

    def cast(x, fmt, row="strip", col=None):
        a, at, s = q(x, fmt, rowwise=row is not None, colwise=col is not None)
        return a, s, at, s

    return cast


class _FP8LinearFn(torch.autograd.Function):
    """``y = x W^T (+ b)`` in FP8 under either recipe of :mod:`deepspeed_b200.ops.fp8` (``block``: blockwise).  Forward
    saves only the transposed cast of ``x`` and its scales; backward re-reads the weight (as :class:`_FlatLinearFn`, so
    ZeRO-3 may release it after forward) to cast ``W^T``, and dW lands in the ZeRO flat gradient view.  Under the
    blockwise recipe the ``A`` of each product is scaled in 1 x 128 strips along its contraction, the ``B`` in 128 x 128
    blocks (tensorwise: one scale per cast):

    forward  ``x`` -> e4m3 strips (and, in the same pass, ``x^T`` in blocks for dW, the only copy saved); ``W`` in blocks;
    dgrad    ``dY`` -> e5m2 strips along the output features; ``W^T`` in blocks, cast from the re-read weight;
    wgrad    ``dY^T`` -> e5m2 strips along the tokens (same pass as dgrad's copy, different scales); saved ``x^T``."""

    @staticmethod
    def forward(ctx, x, weight, bias, block):
        from deepspeed_b200.ops import fp8
        x2 = x.reshape(-1, x.shape[-1])
        native = _fp8_native(x2, weight)
        cast = _fp8_cast4(native, block)
        x8, sx, x8t, sxt = cast(x2, fp8.E4M3, row="strip", col="block" if ctx.needs_input_grad[1] else None)
        w8, sw, _, _ = cast(weight, fp8.E4M3, row="block")
        y = fp8.gemm(x8, w8, sx, sw, native, block=block).to(x.dtype)
        if bias is not None:
            y = y + bias
        ctx.weight_ref = weight
        ctx.has_bias = bias is not None
        ctx.native, ctx.block = native, block
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.save_for_backward(x8t, sxt)
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops import fp8
        x8t, sxt = ctx.saved_tensors
        w, native, block = ctx.weight_ref, ctx.native, ctx.block
        cast = _fp8_cast4(native, block)
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dx = dw = None
        if need_dx or need_dw:
            dy8, sdy, dy8t, sdyt = cast(dy2, fp8.E5M2, row="strip" if need_dx else None, col="strip" if need_dw else None)
            if need_dx:
                _, _, w8t, swt = cast(w, fp8.E4M3, row=None, col="block")
                dx = fp8.gemm(dy8, w8t, sdy, swt, native, block=block).to(ctx.x_dtype).view(ctx.x_shape)
            if need_dw:
                mm = functools.partial(fp8.gemm, dy8t, x8t, sdyt, sxt, native, block=block)
                dw = _weight_grad_sink(w, torch.bfloat16, mm, mm, lambda: mm().to(w.dtype))
        db = dy2.sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        return dx, dw, db, None


def fp8_linear(x, weight, bias=None, recipe="tensorwise"):
    """``x W^T (+ b)`` with FP8 products (see :class:`_FP8LinearFn`).  CUDA bf16 operands whose dimensions are multiples
    of 16 run the wgmma kernels; anything else runs the torch reference of the same recipe (never a bf16 product)."""
    _check_recipe(recipe)
    return _FP8LinearFn.apply(x, weight, bias, recipe == "blockwise")


class _FP8SwiGLUMLPFn(torch.autograd.Function):
    """``down(silu(gate(x)) * up(x))`` in FP8, one node like :class:`_SwiGLUMLPFn` (``block``: the blockwise recipe):

    forward   x -> e4m3 (+ transposed); gate|up FP8 GEMM with the SwiGLU epilogue (gate|up saved in bf16);
              act -> e4m3 (+ transposed); FP8 down GEMM;
    backward  dY -> e5m2 (+ transposed); FP8 ``dY W_down`` GEMM with the dSwiGLU epilogue; dgate|dup -> e5m2 (+ transposed);
              FP8 dX, dW_down and dW_gate_up, the weight gradients into the ZeRO flat gradient views.
    Operand by operand as in :class:`_FP8LinearFn`: the row-major casts (``x``, ``act``, ``dY``, ``dgate|dup``) are scaled
    in 1 x 128 strips, the weights and the saved ``x^T`` and ``act^T`` in 128 x 128 blocks, ``dY^T`` and ``dgate|dup^T``
    in strips along the tokens.  Every read of a weight comes before either weight's gradient is marked ready (marking a
    unit's last gradient reduces it, which under ZeRO-3 releases the gathered weights and with the step fused into
    backward rewrites them)."""

    @staticmethod
    def forward(ctx, x, w_gu, w_down, block):
        from deepspeed_b200.ops import fp8
        x2 = x.reshape(-1, x.shape[-1])
        native = _fp8_native(x2, w_gu, w_down, inter=w_down.shape[1])
        cast = _fp8_cast4(native, block)
        need_grad = any(ctx.needs_input_grad)
        x8, sx, x8t, sxt = cast(x2, fp8.E4M3, row="strip", col="block" if ctx.needs_input_grad[1] else None)
        wgu8, sgu, _, _ = cast(w_gu, fp8.E4M3, row="block")
        act, gu = fp8.gemm_swiglu(x8, wgu8, sx, sgu, native, save_gate_up=need_grad, block=block)
        act8, sa, act8t, sat = cast(act, fp8.E4M3, row="strip", col="block" if ctx.needs_input_grad[2] else None)
        wd8, sd, _, _ = cast(w_down, fp8.E4M3, row="block")
        y = fp8.gemm(act8, wd8, sa, sd, native, block=block).to(x.dtype)
        ctx.w_gu, ctx.w_down, ctx.native, ctx.block = w_gu, w_down, native, block
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        ctx.save_for_backward(x8t, sxt, gu, act8t, sat)
        return y.view(*x.shape[:-1], w_down.shape[0])

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops import fp8
        x8t, sxt, gu, act8t, sat = ctx.saved_tensors
        w_gu, w_down, native, block = ctx.w_gu, ctx.w_down, ctx.native, ctx.block
        cast = _fp8_cast4(native, block)
        need_dx, need_dgu, need_dd = ctx.needs_input_grad[:3]
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dy8, sdy, dy8t, sdyt = cast(dy2, fp8.E5M2, row="strip", col="strip" if need_dd else None)
        _, _, wd8t, sdt = cast(w_down, fp8.E4M3, row=None, col="block")
        dgu = fp8.gemm_dswiglu(dy8, wd8t, sdy, sdt, gu, native, block=block)
        wgu8t = sgut = None
        if need_dx:
            _, _, wgu8t, sgut = cast(w_gu, fp8.E4M3, row=None, col="block")
        dx = dw_gu = dw_down = None
        if need_dx or need_dgu:
            dgu8, sg, dgu8t, sgt = cast(dgu, fp8.E5M2, row="strip" if need_dx else None, col="strip" if need_dgu else None)
            if need_dx:
                dx = fp8.gemm(dgu8, wgu8t, sg, sgut, native, block=block).to(ctx.x_dtype).view(ctx.x_shape)
        # weights are not read past this point
        if need_dd:
            mm = functools.partial(fp8.gemm, dy8t, act8t, sdyt, sat, native, block=block)
            dw_down = _weight_grad_sink(w_down, torch.bfloat16, mm, mm, lambda: mm().to(w_down.dtype))
        if need_dgu:
            mm = functools.partial(fp8.gemm, dgu8t, x8t, sgt, sxt, native, block=block)
            dw_gu = _weight_grad_sink(w_gu, torch.bfloat16, mm, mm, lambda: mm().to(w_gu.dtype))
        return dx, dw_gu, dw_down, None


def fp8_swiglu_mlp(x, w_gate_up, w_down, recipe="tensorwise"):
    """SwiGLU MLP block (no biases) with FP8 products: see :class:`_FP8SwiGLUMLPFn`.  CUDA bf16 operands with ``T, H, 2I``
    multiples of 16 and ``I % 64 == 0`` run the wgmma kernels; anything else runs the torch reference of the same recipe
    (never a bf16 product)."""
    _check_recipe(recipe)
    return _FP8SwiGLUMLPFn.apply(x, w_gate_up, w_down, recipe == "blockwise")


def _stacked_grad_target(w, dtype):
    """-> (zo, gradient tensor, accumulate) for a stacked expert weight: its flat ZeRO gradient view when it has one of
    ``dtype`` (None: of any dtype) -- the GEMM epilogue stores or accumulates there -- else a fresh tensor returned to
    autograd.  :func:`_mark_or_return` finishes it."""
    zo = _zo_of(w)
    if zo is not None and (dtype is None or zo.grad_view_for(w).dtype == dtype):
        return zo, zo.grad_view_for(w), not zo.grad_is_fresh(w)
    return None, torch.empty_like(w), False


def _mark_or_return(zo, w, g):
    """The gradient ``g`` of ``w`` from :func:`_stacked_grad_target`, once written: ``w`` marked ready when ``g`` is its
    owner's view (returns None), else ``g`` for autograd."""
    if zo is None:
        return g
    zo.mark_grad_ready(w)
    return None


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
        no_grad = (None, None, False)
        zo13, g13, acc13 = _stacked_grad_target(w13, dy.dtype) if ctx.needs_input_grad[1] else no_grad
        zo2, g2, acc2 = _stacked_grad_target(w2, dy.dtype) if ctx.needs_input_grad[2] else no_grad
        for e in range(E):
            dgu = gemm.down_dx_dswiglu(dy[e], w2[e], gus[e])
            if g2 is not None:
                gemm.matmul_tn(dy[e], acts[e], out=g2[e], accumulate=acc2)
            if dx is not None:
                gemm.matmul_nn(dgu, w13[e], out=dx[e])
            if g13 is not None:
                gemm.matmul_tn(dgu, x[e], out=g13[e], accumulate=acc13)
            gus[e] = acts[e] = None
        return dx, _mark_or_return(zo13, w13, g13), _mark_or_return(zo2, w2, g2)


def grouped_swiglu_mlp(x, w13, w2):
    return _GroupedSwiGLUFn.apply(x, w13, w2)


class _RaggedSwiGLUFn(torch.autograd.Function):
    """Dropless SwiGLU experts on expert-sorted rows ``x [R, H]``: expert ``e`` owns rows ``[offsets[e], offsets[e+1])``
    (``offsets`` int32 ``[E + 1]`` on the device, segments 64-row aligned and zero-padded -- see
    ``dsb_gemm_ragged_bf16``), ``w13 [E, 2I, H]``, ``w2 [E, H, I]``.  Every projection is ONE launch over all experts, with
    no host synchronisation: forward gate|up (+) SwiGLU and down; backward down-dX (+) dSwiGLU, the variable-K dW2 and
    dW13 and the dX of gate|up.  Weight gradients land in the stacked parameters' flat ZeRO gradient views (accumulated in
    the epilogue on later micro steps), like :class:`_GroupedSwiGLUFn`."""

    @staticmethod
    def forward(ctx, x, offsets, w13, w2):
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        R = x.shape[0]
        I = w2.shape[2]
        need_grad = any(ctx.needs_input_grad)
        gu = torch.empty(R, 2 * I, dtype=x.dtype, device=x.device) if need_grad else None
        act = K.ragged_matmul(x, w13, offsets, False, epi=K.EPI_SWIGLU, out2=gu)
        y = K.ragged_matmul(act, w2, offsets, False)
        ctx.w13, ctx.w2 = w13, w2
        if need_grad:
            ctx.save_for_backward(x, offsets, gu, act)
        return y

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        x, offsets, gu, act = ctx.saved_tensors
        w13, w2 = ctx.w13, ctx.w2
        E, I = w2.shape[0], w2.shape[2]
        dy = dy.contiguous()
        dgu = torch.empty(x.shape[0], 2 * I, dtype=dy.dtype, device=dy.device)
        K.ragged_matmul(dy, w2, offsets, True, out=dgu[:, :I], epi=K.EPI_DSWIGLU, aux=gu, out2=dgu)
        # every read of w13 / w2 comes before either weight is marked ready: marking the unit's last gradient ready
        # reduces it, which under ZeRO-3 releases the gathered weights and with the step fused into backward rewrites them
        dx = K.ragged_matmul(dgu, w13, offsets, True) if ctx.needs_input_grad[0] else None
        outs = {}
        for i, (w, a, b) in ((3, (w2, dy, act)), (2, (w13, dgu, x))):
            if not ctx.needs_input_grad[i]:
                outs[i] = None
                continue
            zo, g, accumulate = _stacked_grad_target(w, dy.dtype)
            K.ragged_wgrad(a, b, offsets, E, out=g, accumulate=accumulate)
            outs[i] = _mark_or_return(zo, w, g)
        return dx, None, outs[2], outs[3]


def ragged_swiglu_reference(x, offsets, w13, w2, act="silu"):
    """The per-expert torch loop with the contract of :class:`_RaggedSwiGLUFn` (any device and dtype, autograd through
    torch).  Rows outside ``[offsets[0], offsets[E])`` come out as zeros here.  Reads the offsets on the host."""
    from deepspeed_b200.ops.kernels.transformer_ops import gated_act
    off = offsets.tolist()
    pieces = [x.new_zeros(off[0], w2.shape[1])]
    for e in range(w13.shape[0]):
        xe = x[off[e]:off[e + 1]]
        pieces.append(gated_act(xe @ w13[e].t(), act) @ w2[e].t() if xe.shape[0] else xe.new_zeros(0, w2.shape[1]))
    pieces.append(x.new_zeros(x.shape[0] - off[-1], w2.shape[1]))
    return torch.cat(pieces, dim=0)


def ragged_swiglu_native(x, offsets, w13, w2, act="silu") -> bool:
    """Whether :func:`ragged_swiglu_mlp` runs the wgmma kernels for these operands: CUDA bf16, SwiGLU, ``H % 64 == 0``,
    ``I % 128 == 0`` and at most 256 experts."""
    from deepspeed_b200.ops.kernels import gemm_sm100 as K
    return (act == "silu" and K.supports_ragged(x, w13, offsets) and x.shape[1] % 64 == 0 and w2.shape[2] % 128 == 0
            and w2.is_contiguous() and w2.dtype == torch.bfloat16)


def ragged_swiglu_mlp(x, offsets, w13, w2, act="silu"):
    """SwiGLU experts over expert-sorted rows ``x [R, H]`` with ``w13 [E, 2I, H]``, ``w2 [E, H, I]`` and ``offsets [E + 1]``:
    see :class:`_RaggedSwiGLUFn`; other devices, dtypes, activations and shapes take :func:`ragged_swiglu_reference`.
    Rows outside ``[offsets[0], offsets[E])`` of the result (and of ``x``'s gradient) are unspecified on the wgmma path,
    which does not write them: callers read only the experts' rows."""
    E, I = w13.shape[0], w2.shape[-1]
    H = x.shape[-1]
    if (x.dim() != 2 or w13.dim() != 3 or tuple(w13.shape) != (E, 2 * I, H) or tuple(w2.shape) != (E, H, I)
            or offsets.dim() != 1 or offsets.numel() != E + 1):
        raise ValueError(f"ragged_swiglu_mlp: rows {tuple(x.shape)}, w13 {tuple(w13.shape)}, w2 {tuple(w2.shape)} and "
                         f"offsets {tuple(offsets.shape)} are not [R, H], [E, 2I, H], [E, H, I] and [E + 1]")
    if ragged_swiglu_native(x, offsets, w13, w2, act):
        return _RaggedSwiGLUFn.apply(x, offsets, w13, w2)
    return ragged_swiglu_reference(x, offsets, w13, w2, act)


class _FP8RaggedSwiGLUFn(torch.autograd.Function):
    """:class:`_RaggedSwiGLUFn` with FP8 products (tensorwise, or ``block``: blockwise, operand by operand as in
    :class:`_FP8SwiGLUMLPFn`), on 128-row segments.  The stacked weights are cast as the 2-D matrices
    ``w13 [E 2I, H]`` and ``w2 [E H, I]`` (one tensorwise scale per stacked weight); forward and dgrad take expert e's
    row slab of the cast or column slab of its transposed cast, and the variable-K wgrad sums each expert's rows of the
    transposed activation and gradient copies.  The forward saves only those transposed copies, their scales and the
    bf16 gate|up; backward re-reads the weights for their transposed casts, finishes every weight read before either
    gradient is marked ready, and stores or accumulates dW13 / dW2 straight into the stacked parameters' flat ZeRO
    gradient views.  No host synchronisation on the kernels (``native``); otherwise the torch reference of the recipe.
    ``act`` and dgate|dup are zero outside the segments: their casts read every row, and a stray value there would
    enter every expert's tensorwise scale."""

    @staticmethod
    def forward(ctx, x, offsets, w13, w2, block, native):
        from deepspeed_b200.ops import fp8
        E, H, I = w2.shape
        w13f, w2f = w13.reshape(E * 2 * I, H), w2.reshape(E * H, I)
        cast = _fp8_cast4(native, block)
        need_grad = any(ctx.needs_input_grad)
        need_d13, need_d2 = ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        x8, sx, x8t, sxt = cast(x, fp8.E4M3, row="strip", col="block" if need_d13 else None)
        w13_8, s13, _, _ = cast(w13f, fp8.E4M3, row="block")
        act, gu = fp8.ragged_gemm_swiglu(x8, w13_8, offsets, sx, s13, E, native, save_gate_up=need_grad, block=block)
        act8, sa, act8t, sat = cast(act, fp8.E4M3, row="strip", col="block" if need_d2 else None)
        w2_8, s2, _, _ = cast(w2f, fp8.E4M3, row="block")
        y = fp8.ragged_gemm(act8, w2_8, offsets, sa, s2, E, native, block=block)
        ctx.w13, ctx.w2, ctx.block, ctx.native = w13, w2, block, native
        if need_grad:
            ctx.save_for_backward(offsets, x8t, sxt, gu, act8t, sat)
        return y

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops import fp8
        offsets, x8t, sxt, gu, act8t, sat = ctx.saved_tensors
        w13, w2, block, native = ctx.w13, ctx.w2, ctx.block, ctx.native
        E, H, I = w2.shape
        w13f, w2f = w13.reshape(E * 2 * I, H), w2.reshape(E * H, I)
        cast = _fp8_cast4(native, block)
        need_dx, need_d13, need_d2 = ctx.needs_input_grad[0], ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        dy = dy.contiguous()
        dy8, sdy, dy8t, sdyt = cast(dy, fp8.E5M2, row="strip", col="strip" if need_d2 else None)
        _, _, w2_8t, s2t = cast(w2f, fp8.E4M3, row=None, col="block")
        dgu = fp8.ragged_gemm_dswiglu(dy8, w2_8t, offsets, sdy, s2t, gu, E, native, block=block)
        dx = dgu8t = sgt = None
        if need_dx or need_d13:
            dgu8, sg, dgu8t, sgt = cast(dgu, fp8.E5M2, row="strip" if need_dx else None, col="strip" if need_d13 else None)
            if need_dx:
                _, _, w13_8t, s13t = cast(w13f, fp8.E4M3, row=None, col="block")
                dx = fp8.ragged_gemm(dgu8, w13_8t, offsets, sg, s13t, E, native, block=block)
        # weights are not read past this point
        grads = {}
        for i, w, a8t, b8t, s_a, s_b in ((3, w2, dy8t, act8t, sdyt, sat), (2, w13, dgu8t, x8t, sgt, sxt)):
            if not ctx.needs_input_grad[i]:
                grads[i] = None
                continue
            # the kernels write a bf16 view; the torch reference one of any dtype
            zo, g, accumulate = _stacked_grad_target(w, torch.bfloat16 if native else None)
            fp8.ragged_wgrad(a8t, b8t, offsets, s_a, s_b, E, native, out=g, accumulate=accumulate, block=block)
            grads[i] = _mark_or_return(zo, w, g)
        return dx, None, grads[2], grads[3], None, None


def fp8_ragged_swiglu_native(x, offsets, w13, w2) -> bool:
    """Whether :func:`fp8_ragged_swiglu_mlp` runs the wgmma kernels: CUDA bf16 contiguous rows and stacked weights, int32
    device offsets, at most 256 experts, ``R % 16 == 0`` (the transposed casts), ``H % 128 == 0`` (the down projection's
    dgrad takes 128-column expert slabs of its transposed cast) and ``I % 64 == 0`` (the SwiGLU tile, and 128-column
    slabs for the gate|up dgrad)."""
    from deepspeed_b200.ops.kernels import gemm_sm100 as K
    R, H = x.shape
    I = w2.shape[2]
    return (K.supports_ragged(x, w13, offsets) and x.is_contiguous() and w2.is_cuda and w2.dtype == torch.bfloat16
            and w2.is_contiguous() and R > 0 and R % 16 == 0 and H % 128 == 0 and I % 64 == 0)


def fp8_ragged_swiglu_mlp(x, offsets, w13, w2, recipe="tensorwise"):
    """SwiGLU experts over expert-sorted rows ``x [R, H]`` with FP8 products (see :class:`_FP8RaggedSwiGLUFn`): ``w13
    [E, 2I, H]``, ``w2 [E, H, I]``, ``offsets [E + 1]`` non-decreasing multiples of 128, segments zero-padded and the rows
    outside them finite (the dropless MoE layer's are zero).  Operands the kernels cannot take (see
    :func:`fp8_ragged_swiglu_native`) run the same recipe through the torch reference, never a bf16 product.  Rows of
    the result outside ``[offsets[0], offsets[E])`` are unspecified on the wgmma path."""
    _check_recipe(recipe)
    E, I = w13.shape[0], w2.shape[-1]
    H = x.shape[-1]
    if (x.dim() != 2 or w13.dim() != 3 or tuple(w13.shape) != (E, 2 * I, H) or tuple(w2.shape) != (E, H, I)
            or offsets.dim() != 1 or offsets.numel() != E + 1):
        raise ValueError(f"fp8_ragged_swiglu_mlp: rows {tuple(x.shape)}, w13 {tuple(w13.shape)}, w2 {tuple(w2.shape)} "
                         f"and offsets {tuple(offsets.shape)} are not [R, H], [E, 2I, H], [E, H, I] and [E + 1]")
    native = fp8_ragged_swiglu_native(x, offsets, w13, w2)
    return _FP8RaggedSwiGLUFn.apply(x, offsets, w13, w2, recipe == "blockwise", native)


class _ChunkedLinearXent(torch.autograd.Function):

    @staticmethod
    def forward(ctx, h, weight, labels, chunk, ignore_index, assumed_scale, defer_ready):
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
        ctx.defer_ready = defer_ready
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
                _mark_or_note(zo, w, ctx.defer_ready)
            elif zo is not None:
                gv = zo.grad_view_for(w)
                if zo.grad_is_fresh(w):
                    torch.mul(ctx.dw_tmp, r.to(ctx.dw_tmp.dtype), out=gv) if gv.dtype == ctx.dw_tmp.dtype else gv.copy_(
                        ctx.dw_tmp.float() * r)
                else:
                    gv.add_((ctx.dw_tmp.float() * r).to(gv.dtype))
                _mark_or_note(zo, w, ctx.defer_ready)
            else:
                dw = ctx.dw_tmp * r.to(ctx.dw_tmp.dtype)
        ctx.dh = None
        ctx.dw_tmp = None
        return dh, dw, None, None, None, None, None


def _mark_or_note(zo, w, defer_ready):
    """``w``'s gradient view holds this node's contribution: mark ``w`` ready, or with ``defer_ready`` only note the
    write, so that a later producer of the same weight accumulates and marks it."""
    if defer_ready:
        zo.note_grad_written(w)
    else:
        zo.mark_grad_ready(w)


def chunked_linear_xent(h, weight, labels, chunk=2048, ignore_index=-100, assumed_scale=1.0, defer_ready=False):
    """Mean cross entropy of ``softmax(h W^T)`` vs ``labels`` without materialising the logits.  ``defer_ready``: the
    weight has another producer whose backward runs later (a tied input embedding, see :func:`embedding`), which marks
    it ready; this node's dW is left in the ZeRO gradient view for it to accumulate onto."""
    if not torch.is_grad_enabled():
        total = torch.zeros((), dtype=torch.float32, device=h.device)
        n = xent_valid(labels, weight.shape[0], ignore_index).sum().clamp(min=1)
        for s in range(0, h.shape[0], chunk):
            e = min(s + chunk, h.shape[0])
            logits = _gemm(h[s:e], weight)
            rows, _ = softmax_xent_fwd_bwd(logits, labels[s:e].contiguous(), 1.0, None, ignore_index, False)
            total = total + rows.sum()
        return total / n
    return _ChunkedLinearXent.apply(h, weight, labels, chunk, ignore_index, float(assumed_scale) or 1.0, defer_ready)


class _EmbeddingFn(torch.autograd.Function):
    """``weight[ids]`` whose backward adds the weight gradient straight into the ZeRO flat gradient view with the
    deterministic embedding backward (:func:`transformer_ops.embedding_bwd_`): only the rows of ids that occur are
    touched, so a tied LM head's dW may already sit in the view (stored there on a fresh view, which is zeroed first),
    and the weight is marked ready once both have landed.  Without an owner the gradient is a zero ``[V, H]`` tensor
    accumulated into and returned to autograd.  Backward reads no weight."""

    @staticmethod
    def forward(ctx, ids, weight):
        ctx.save_for_backward(ids)
        ctx.weight_ref = weight
        return F.embedding(ids, weight)

    @staticmethod
    def backward(ctx, dy):
        from deepspeed_b200.ops.kernels.transformer_ops import embedding_bwd_
        (ids, ) = ctx.saved_tensors
        w = ctx.weight_ref
        zo = _zo_of(w)
        if zo is None:
            return None, embedding_bwd_(dy, ids, torch.zeros(w.shape, dtype=w.dtype, device=dy.device))
        gv = zo.grad_view_for(w)
        if zo.grad_is_fresh(w):
            gv.zero_()
        embedding_bwd_(dy, ids, gv)
        zo.mark_grad_ready(w)
        return None, None


def embedding(ids, weight):
    """``F.embedding(ids, weight)`` whose weight gradient goes through :class:`_EmbeddingFn`."""
    if not torch.is_grad_enabled() or not weight.requires_grad:
        return F.embedding(ids, weight)
    return _EmbeddingFn.apply(ids, weight)
