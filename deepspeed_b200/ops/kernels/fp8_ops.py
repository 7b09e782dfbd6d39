"""Python face of ``csrc/cuda/fp8_cast.cu`` -- the tensorwise FP8 amax and cast(-transpose) kernels and the single-pass
blockwise cast.  The recipes they implement (and their torch references) are documented in :mod:`deepspeed_b200.ops.fp8`."""
import torch

from deepspeed_b200.ops import native as N

_FMT = {torch.float8_e4m3fn: N.F8E4M3, torch.float8_e5m2: N.F8E5M2}


def _check_x(x, what):
    if not (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1):
        raise N.NativeOpError(f"{what}: x must be a 2-D CUDA bf16 tensor with unit column stride, got "
                              f"{tuple(x.shape)} {x.dtype} strides {tuple(x.stride())} on {x.device}")


def fp8_amax(x, out=None):
    """``max |x|`` of the bf16 matrix ``x [R, C]`` into a one-element fp32 device tensor (NaN if ``x`` holds a NaN)."""
    _check_x(x, "fp8_amax")
    if out is None:
        out = torch.empty(1, dtype=torch.float32, device=x.device)
    rc = N.cuda().dsb_fp8_amax(N.ptr(x), N.c_i64(x.shape[0]), N.c_i64(x.shape[1]), N.c_i64(x.stride(0)), N.ptr(out),
                               N.stream())
    N.check(rc, "fp8_amax")
    return out


def fp8_cast(x, amax, fmt, rowwise=True, colwise=False, out=None, out_t=None, scale_inv=None):
    """Quantise the bf16 matrix ``x [R, C]`` with the power-of-two scale of ``amax`` (from :func:`fp8_amax`) to ``fmt``
    (``torch.float8_e4m3fn`` / ``float8_e5m2``).  Returns ``(q [R, C] or None, qt [C, R] or None, scale_inv [1])``;
    ``qt`` is the transpose of ``q`` (it needs ``R % 16 == 0``).  ``out`` / ``out_t`` may be strided views."""
    _check_x(x, "fp8_cast")
    if fmt not in _FMT or not (rowwise or colwise):
        raise N.NativeOpError(f"fp8_cast: format {fmt} (rowwise={rowwise}, colwise={colwise}) is not supported")
    R, C = x.shape
    q = qt = None
    if rowwise:
        q = out if out is not None else torch.empty(R, C, dtype=fmt, device=x.device)
        if q.dtype != fmt or tuple(q.shape) != (R, C) or q.stride(1) != 1:
            raise N.NativeOpError(f"fp8_cast: out must be [{R}, {C}] {fmt}")
    if colwise:
        qt = out_t if out_t is not None else torch.empty(C, R, dtype=fmt, device=x.device)
        if qt.dtype != fmt or tuple(qt.shape) != (C, R) or qt.stride(1) != 1:
            raise N.NativeOpError(f"fp8_cast: out_t must be [{C}, {R}] {fmt}")
    if scale_inv is None:
        scale_inv = torch.empty(1, dtype=torch.float32, device=x.device)
    rc = N.cuda().dsb_fp8_cast(N.ptr(x), N.c_i64(R), N.c_i64(C), N.c_i64(x.stride(0)), N.ptr(amax), _FMT[fmt], N.ptr(q),
                               N.c_i64(q.stride(0) if q is not None else 0), N.ptr(qt),
                               N.c_i64(qt.stride(0) if qt is not None else 0), N.ptr(scale_inv), N.stream())
    N.check(rc, "fp8_cast")
    return q, qt, scale_inv


_MODE = {None: 0, "strip": 1, "block": 2}


def fp8_cast_block(x, fmt, row="strip", col=None, out=None, out_scale=None, out_t=None, out_t_scale=None):
    """Blockwise-scaled cast of the bf16 matrix ``x [R, C]`` in one pass (``dsb_fp8_cast_block``): ``row`` / ``col`` say
    how the row-major copy ``q [R, C]`` / the transposed copy ``qt [C, R]`` is scaled -- ``"strip"`` (one scale per 1 x 128
    strip along the copy's columns), ``"block"`` (one per 128 x 128 block) or None (copy not made).  Returns
    ``(q, sq, qt, st)`` with the fp32 ``scale_inv`` tensors in the layouts of
    :func:`deepspeed_b200.ops.fp8.quantize_blockwise_reference`.  The outputs may be strided views."""
    _check_x(x, "fp8_cast_block")
    if fmt not in _FMT or row not in _MODE or col not in _MODE or (row is None and col is None):
        raise N.NativeOpError(f"fp8_cast_block: format {fmt} with row={row!r}, col={col!r} is not supported")
    R, C = x.shape
    rb, cb = -(-R // 128), -(-C // 128)

    def outputs(mode, data, scale, shape, strip_shape, block_shape, what):
        if mode is None:
            return None, None
        if data is None:
            data = torch.empty(shape, dtype=fmt, device=x.device)
        want = strip_shape if mode == "strip" else block_shape
        if scale is None:
            scale = torch.empty(want, dtype=torch.float32, device=x.device)
        if (data.dtype != fmt or tuple(data.shape) != shape or data.stride(1) != 1 or scale.dtype != torch.float32
                or tuple(scale.shape) != want or scale.stride(1) != 1):
            raise N.NativeOpError(f"fp8_cast_block: {what} must be {list(shape)} {fmt} with fp32 scales {list(want)}")
        return data, scale

    q, sq = outputs(row, out, out_scale, (R, C), (cb, R), (rb, cb), "out")
    qt, st = outputs(col, out_t, out_t_scale, (C, R), (rb, C), (cb, rb), "out_t")
    ld = lambda t: N.c_i64(t.stride(0) if t is not None else 0)
    rc = N.cuda().dsb_fp8_cast_block(N.ptr(x), N.c_i64(R), N.c_i64(C), N.c_i64(x.stride(0)), _FMT[fmt], _MODE[row], N.ptr(q),
                                     ld(q), N.ptr(sq), ld(sq), _MODE[col], N.ptr(qt), ld(qt), N.ptr(st), ld(st), N.stream())
    N.check(rc, "fp8_cast_block")
    return q, sq, qt, st
