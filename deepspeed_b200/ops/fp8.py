"""FP8 training recipes: current scaling with power-of-two scales, one scale per tensor (torchao's "tensorwise", with
Transformer Engine's HYBRID formats) or one per block (below).

* Activations and weights are ``float8_e4m3fn`` (max 448); gradients flowing backward are ``float8_e5m2`` (max 57344).
* Each tensor gets one fp32 scale computed on the device from its amax when it is cast: no history, no delayed scaling,
  no host synchronisation.  ``scale = 2**e`` with ``e = floor(log2(FMAX / amax))`` clamped to ``[-126, 126]`` (so the
  scale and its inverse are finite normal floats); ``amax == 0`` gives ``scale = 1``; a non-finite amax gives NaN scales,
  so the overflow shows in every result computed from the tensor instead of being clipped away.
* ``q = fp8_rne(x * scale)``.  Since ``amax * scale <= FMAX`` nothing saturates, and the result is bit-equal to
  ``(x.float() * scale).to(fmt)``.  Power-of-two scales make scaling and unscaling exact.
* A product of two cast tensors is ``sa_inv * sb_inv * (a8 @ b8^T)`` accumulated in fp32 and rounded once to bf16.

The wgmma path is ``csrc/cuda/fp8_cast.cu`` (amax, cast, cast-transpose) and ``dsb_gemm_fp8`` in ``csrc/cuda/gemm_sm90.cu``.
The ``*_reference`` functions here do the same casts and scales in torch, with an fp32 matmul: they are the path for
operands the kernels cannot take (CPU tensors, other dtypes and shapes) and the tests' oracle.

Blockwise recipe (DeepSeek-V3's granularity): the same formats, scale rule and cast, with the amax taken per block --
one scale per 1 x 128 strip along the contraction for the ``A`` operand of a product (activations, gradients), one per
128 x 128 block for its ``B`` operand (weights; in the weight gradient, the transposed input).  A trailing partial block
takes its amax over the elements that exist.  ``C = epi(sum_kb sa_inv[kb, m] * sb_inv[n // 128, kb] * (A8[m, kb] @
B8[n, kb]^T))``: the block partials are scaled and summed in fp32 and rounded once.  An outlier costs the precision of
its own strip or block only.  ``dsb_fp8_cast_block`` finds the amaxes inside the tile it casts (one pass, no atomics on
global memory) and ``dsb_gemm_fp8_block`` applies the scales where it promotes each k-block.
"""
import torch

E4M3 = torch.float8_e4m3fn
E5M2 = torch.float8_e5m2
FMAX = {E4M3: 448.0, E5M2: 57344.0}
_EMAX = {E4M3: 8, E5M2: 15}  # FMAX = 1.75 * 2**emax


def scale_from_amax(amax, fmt):
    """``(scale, scale_inv)`` (fp32, the shape of ``amax``) for a tensor of max magnitude ``amax``: the recipe's rule,
    evaluated exactly from amax's exponent and significand (no rounding of ``FMAX / amax``)."""
    a = amax.float()
    m, x = torch.frexp(a)  # a = m * 2**x, m in [0.5, 1): a * 2**e <= 1.75 * 2**emax  <=>  e <= emax - x + 1 - [m > 0.875]
    e = (_EMAX[fmt] - x.int() + 1 - (m > 0.875).int()).clamp(-126, 126)
    e = torch.where(a == 0, 0, e)
    scale = torch.ldexp(torch.ones_like(a), e)
    scale_inv = torch.ldexp(torch.ones_like(a), -e)
    bad = ~torch.isfinite(a)
    nan = torch.full_like(a, float("nan"))
    return torch.where(bad, nan, scale), torch.where(bad, nan, scale_inv)


def quantize_reference(x, fmt, rowwise=True, colwise=False):
    """Torch implementation of the cast: ``(q or None, q^T contiguous or None, scale_inv [1])``."""
    x2 = x.reshape(-1, x.shape[-1]) if x.dim() != 2 else x
    amax = x2.float().abs().amax().reshape(1) if x2.numel() else torch.zeros(1, device=x.device)
    scale, scale_inv = scale_from_amax(amax, fmt)
    q = (x2.float() * scale).to(fmt)
    return (q if rowwise else None), (q.t().contiguous() if colwise else None), scale_inv


def native_cast_ok(x, colwise=False) -> bool:
    """Whether the cast kernels take ``x``: a 2-D CUDA bf16 matrix with unit column stride (and ``R % 16 == 0`` for a
    transposed output)."""
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1 and x.shape[0] >= 1
            and x.shape[1] >= 1 and x.data_ptr() % 2 == 0 and (not colwise or x.shape[0] % 16 == 0))


def quantize_tensorwise(x, fmt, rowwise=True, colwise=False):
    """Cast the matrix ``x`` with its own power-of-two scale: returns ``(data [R, C] or None, transposed data [C, R] or
    None, scale_inv [1] fp32)``, all on ``x``'s device.  CUDA bf16 matrices go through the native amax and cast kernels
    (no host synchronisation); anything else through :func:`quantize_reference`, which is bit-equal."""
    if native_cast_ok(x, colwise):
        from deepspeed_b200.ops.kernels import fp8_ops
        return fp8_ops.fp8_cast(x, fp8_ops.fp8_amax(x), fmt, rowwise=rowwise, colwise=colwise)
    return quantize_reference(x, fmt, rowwise, colwise)


def matmul_reference(a8, b8, sa_inv, sb_inv):
    """fp32 ``sa_inv * sb_inv * (a8 @ b8^T)`` of two cast matrices (before the bf16 rounding)."""
    return (a8.float() @ b8.float().t()) * (sa_inv * sb_inv)


BLOCK = 128


def _block_amax(x, rows, cols):
    """amax of the fp32 matrix ``x [R, C]`` over blocks of ``rows x cols`` (trailing partial blocks over what exists):
    ``[ceil(R / rows), ceil(C / cols)]``."""
    R, C = x.shape
    rb, cb = -(-R // rows), -(-C // cols)
    a = torch.zeros(rb * rows, cb * cols, dtype=torch.float32, device=x.device)
    a[:R, :C] = x.abs()
    return a.view(rb, rows, cb, cols).permute(0, 2, 1, 3).reshape(rb, cb, -1).amax(dim=2)


def quantize_blockwise_reference(x, fmt, row="strip", col=None):
    """Torch implementation of the blockwise cast of the matrix ``x [R, C]``: ``(q, sq, qt, st)``.

    ``row`` scales the row-major copy ``q [R, C]``: ``"strip"`` -- one scale per 1 x 128 strip of a row (``q`` is the ``A``
    of a product contracting over ``C``), ``sq [ceil(C/128), R]``; ``"block"`` -- one per 128 x 128 block (``q`` is a
    ``B``), ``sq [ceil(R/128), ceil(C/128)]``; None -- no row-major copy.  ``col`` scales the transposed copy
    ``qt [C, R]`` the same way, its strips running along ``R``: ``st [ceil(R/128), C]`` or ``[ceil(C/128), ceil(R/128)]``.
    The scale tensors hold ``scale_inv`` (fp32).  Strip scales are stored k-block-major, the layout the GEMM reads.  A
    block of ``x`` and the same block of ``qt`` share a scale, so ``row="block", col="block"`` gives ``st == sq.t()`` and
    ``qt == q.t()``; with any strip scaling the two copies are different casts of ``x``."""
    xf = x.float()
    R, C = xf.shape

    def cast(mode, transposed):
        if mode is None:
            return None, None
        if mode == "block":
            amax = _block_amax(xf, BLOCK, BLOCK)
        elif transposed:
            amax = _block_amax(xf, BLOCK, 1)  # [ceil(R/128), C]
        else:
            amax = _block_amax(xf, 1, BLOCK)  # [R, ceil(C/128)]
        scale, scale_inv = scale_from_amax(amax, fmt)
        full = scale
        if amax.shape[0] != R:
            full = full.repeat_interleave(BLOCK, dim=0)[:R]
        if amax.shape[1] != C:
            full = full.repeat_interleave(BLOCK, dim=1)[:, :C]
        q = (xf * full).to(fmt)
        if transposed:
            return q.t().contiguous(), (scale_inv.t().contiguous() if mode == "block" else scale_inv)
        return q, (scale_inv if mode == "block" else scale_inv.t().contiguous())

    q, sq = cast(row, False)
    qt, st = cast(col, True)
    return q, sq, qt, st


def quantize_blockwise(x, fmt, row="strip", col=None):
    """Blockwise cast of the matrix ``x`` (see :func:`quantize_blockwise_reference` for the arguments and the result).
    CUDA bf16 matrices go through the single-pass native kernel (no amax launch, no host synchronisation); anything
    else through the reference, which is bit-equal."""
    if native_cast_ok(x, col is not None):
        from deepspeed_b200.ops.kernels import fp8_ops
        return fp8_ops.fp8_cast_block(x, fmt, row=row, col=col)
    return quantize_blockwise_reference(x, fmt, row, col)


def matmul_blockwise_reference(a8, b8, sa_inv, sb_inv):
    """fp32 ``sum_kb sa_inv[kb, m] * sb_inv[n // 128, kb] * (a8[m, kb] @ b8[n, kb]^T)`` (before the bf16 rounding), one
    k-block of 128 after the other as the kernel promotes them."""
    M, K = a8.shape
    Nn = b8.shape[0]
    a, b = a8.float(), b8.float()
    acc = torch.zeros(M, Nn, dtype=torch.float32, device=a8.device)
    for kb in range(-(-K // BLOCK)):
        k = slice(kb * BLOCK, min(K, (kb + 1) * BLOCK))
        s = sa_inv[kb][:, None] * sb_inv[:, kb].repeat_interleave(BLOCK)[:Nn][None, :]
        acc = acc + (a[:, k] @ b[:, k].t()) * s
    return acc


def silu32(g):
    return g / (1 + torch.exp(-g))


def dsilu32(g):
    s = 1 / (1 + torch.exp(-g))
    return s * (1 + g * (1 - s))


# ---- the products of the two training nodes, on the kernels or in torch -------------------------------------------------
# ``block`` selects the blockwise recipe: ``sa`` / ``sb`` are then the strip and block scale tensors.
def _native_matmul(block):
    from deepspeed_b200.ops.kernels import gemm_sm100 as K
    return K, (K.fp8_matmul_block if block else K.fp8_matmul)


def _reference_matmul(block):
    return matmul_blockwise_reference if block else matmul_reference


def gemm(a8, b8, sa, sb, native, out=None, accumulate=False, block=False):
    """bf16 ``[M, N]`` = ``sa sb a8 b8^T`` (``accumulate``: added to ``out`` before the one rounding)."""
    if native:
        K, mm = _native_matmul(block)
        return mm(a8, b8, sa, sb, out=out, epi=K.EPI_ACCUM if accumulate else K.EPI_STORE)
    c = _reference_matmul(block)(a8, b8, sa, sb)
    if accumulate:
        c = c + out.float()
    if out is None:
        return c.to(torch.bfloat16)
    return out.copy_(c)


def gemm_swiglu(a8, b8, sa, sb, native, save_gate_up=True, block=False):
    """``(act [M, I], gate|up [M, 2I] or None)`` for ``b8 = [gate; up] [2I, K]``: silu applied to the fp32 products."""
    if native:
        K, mm = _native_matmul(block)
        I = b8.shape[0] // 2
        gu = torch.empty(a8.shape[0], 2 * I, dtype=torch.bfloat16, device=a8.device) if save_gate_up else None
        return mm(a8, b8, sa, sb, epi=K.EPI_SWIGLU, out2=gu), gu
    gu = _reference_matmul(block)(a8, b8, sa, sb)
    g, u = gu.chunk(2, dim=1)
    return (silu32(g) * u).to(torch.bfloat16), (gu.to(torch.bfloat16) if save_gate_up else None)


def gemm_dswiglu(a8, b8, sa, sb, gu, native, block=False):
    """dgate|dup ``[M, 2I]`` (bf16) for the SwiGLU whose gate|up ``gu`` was saved: ``d = sa sb a8 b8^T`` in fp32, then
    ``dgate = d * u * silu'(g)`` and ``dup = d * silu(g)``."""
    if native:
        K, mm = _native_matmul(block)
        out2 = torch.empty(gu.shape, dtype=torch.bfloat16, device=gu.device)
        mm(a8, b8, sa, sb, epi=K.EPI_DSWIGLU, aux=gu, out2=out2)
        return out2
    d = _reference_matmul(block)(a8, b8, sa, sb)
    g, u = gu.float().chunk(2, dim=1)
    return torch.cat([d * u * dsilu32(g), d * silu32(g)], dim=1).to(torch.bfloat16)


# ---- the ragged (dropless MoE) products --------------------------------------------------------------------------------
# Rows are sorted by expert, expert e owning rows [offsets[e], offsets[e+1]) (multiples of 128).  The stacked weights are
# cast as one 2-D matrix [E * Nb, K] (and its transpose [K, E * Nb]), so expert e's operand is a row slab of the cast or a
# column slab of the transposed cast, and its block scales are the matching slab of the scale tensor.  The references
# below loop over the experts with the offsets read on the host; rows outside the segments come out as zeros there.
def _host_segments(offsets):
    off = offsets.tolist()
    if any(o % BLOCK for o in off) or any(b < a for a, b in zip(off, off[1:])):
        raise ValueError(f"ragged FP8 segments must start at non-decreasing multiples of {BLOCK} rows, got {off}")
    return off


def _dequant(q, s, mode):
    """fp32 values of the blockwise cast ``q [R, C]``: ``mode`` "strip" (``s [ceil(C/128), R]``) or "block"."""
    R, C = q.shape
    if mode == "strip":
        return q.float() * s.t().repeat_interleave(BLOCK, dim=1)[:, :C]
    return q.float() * s.repeat_interleave(BLOCK, dim=0)[:R].repeat_interleave(BLOCK, dim=1)[:, :C]


def _expert_operands(a8, b8, sa, sb, e, E, lo, hi, block):
    """Expert e's operands: its rows of ``a8`` and a row slab of the stacked weight's cast (forward, e4m3 ``a8``) or a
    column slab of its transposed cast (dgrad, e5m2 ``a8``), with their scales.  Blockwise, the operands come back
    dequantised (exact in fp32) with unit scales, so a slab need not start on a 128-row block."""
    one = torch.ones(1, dtype=torch.float32, device=a8.device)
    if a8.dtype == E5M2:  # dgrad: b8 [N, E K], expert e's columns
        k = b8.shape[1] // E
        sl = (slice(None), slice(e * k, (e + 1) * k))
    else:  # forward: b8 [E Nb, K], expert e's rows
        n = b8.shape[0] // E
        sl = (slice(e * n, (e + 1) * n), slice(None))
    if not block:
        return a8[lo:hi], b8[sl], sa, sb
    return _dequant(a8, sa, "strip")[lo:hi], _dequant(b8, sb, "block")[sl], one, one


def ragged_gemm(a8, b8, offsets, sa, sb, E, native, block=False):
    """bf16 ``[R, N]``: ``out[r] = epi_store(sa sb a8[r] b8_e^T)`` for the expert ``e`` of row ``r`` (forward with an e4m3
    ``a8`` and ``b8 [E N, K]``; dgrad with an e5m2 ``a8`` and ``b8 [N, E K]``)."""
    if native:
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        return K.fp8_ragged_matmul(a8, b8, offsets, sa, sb, E, block=block)
    off = _host_segments(offsets)
    n = b8.shape[0] if a8.dtype == E5M2 else b8.shape[0] // E
    out = torch.zeros(a8.shape[0], n, dtype=torch.bfloat16, device=a8.device)
    for e in range(E):
        if off[e + 1] > off[e]:
            out[off[e]:off[e + 1]] = gemm(*_expert_operands(a8, b8, sa, sb, e, E, off[e], off[e + 1], block), False)
    return out


def ragged_gemm_swiglu(a8, b8, offsets, sa, sb, E, native, save_gate_up=True, block=False):
    """``(act [R, I], gate|up [R, 2I] or None)`` for the stacked ``[gate; up]`` weights ``b8 [E 2I, K]``.  ``act`` is zero
    on the rows outside the segments (its cast reads every row); gate|up is unspecified there."""
    R, I = a8.shape[0], b8.shape[0] // E // 2
    act = torch.zeros(R, I, dtype=torch.bfloat16, device=a8.device)
    gu = torch.empty(R, 2 * I, dtype=torch.bfloat16, device=a8.device) if save_gate_up else None
    if native:
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        K.fp8_ragged_matmul(a8, b8, offsets, sa, sb, E, out=act, epi=K.EPI_SWIGLU, out2=gu, block=block)
        return act, gu
    off = _host_segments(offsets)
    for e in range(E):
        lo, hi = off[e], off[e + 1]
        if hi > lo:
            act[lo:hi], gue = gemm_swiglu(*_expert_operands(a8, b8, sa, sb, e, E, lo, hi, block), False, save_gate_up)
            if save_gate_up:
                gu[lo:hi] = gue
    return act, gu


def ragged_gemm_dswiglu(a8, b8, offsets, sa, sb, gu, E, native, block=False):
    """dgate|dup ``[R, 2I]`` from the e5m2 ``a8 = dY`` and the transposed down weight ``b8 [I, E H]``; zero on the rows
    outside the segments (its cast reads every row)."""
    out2 = torch.zeros(gu.shape, dtype=torch.bfloat16, device=gu.device)
    if native:
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        K.fp8_ragged_matmul(a8, b8, offsets, sa, sb, E, epi=K.EPI_DSWIGLU, aux=gu, out2=out2, block=block)
        return out2
    off = _host_segments(offsets)
    for e in range(E):
        lo, hi = off[e], off[e + 1]
        if hi > lo:
            out2[lo:hi] = gemm_dswiglu(*_expert_operands(a8, b8, sa, sb, e, E, lo, hi, block), gu[lo:hi], False)
    return out2


def ragged_wgrad(a8t, b8t, offsets, sa, sb, E, native, out=None, accumulate=False, block=False):
    """``out [E, M, N]`` (bf16): ``out[e] (+)= sa sb a8t[:, rows of e] b8t[:, rows of e]^T`` for the transposed casts
    ``a8t [M, R]`` (e5m2) and ``b8t [N, R]`` (e4m3); an expert without rows gets zeros or keeps ``out[e]``."""
    if native:
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        return K.fp8_ragged_wgrad(a8t, b8t, offsets, sa, sb, E, out=out, accumulate=accumulate, block=block)
    off = _host_segments(offsets)
    if out is None:
        out = torch.empty(E, a8t.shape[0], b8t.shape[0], dtype=torch.bfloat16, device=a8t.device)
    for e in range(E):
        lo, hi = off[e], off[e + 1]
        if hi == lo:
            if not accumulate:
                out[e].zero_()
            continue
        sae = sa[lo // BLOCK:hi // BLOCK] if block else sa
        sbe = sb[:, lo // BLOCK:hi // BLOCK] if block else sb
        gemm(a8t[:, lo:hi], b8t[:, lo:hi], sae, sbe, False, out=out[e], accumulate=accumulate, block=block)
    return out
