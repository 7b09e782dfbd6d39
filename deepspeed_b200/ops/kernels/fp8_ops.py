"""Python face of ``csrc/cuda/fp8_cast.cu`` -- the tensorwise FP8 amax and cast(-transpose) kernels.  The recipe they
implement (and its torch reference) is documented in :mod:`deepspeed_b200.ops.fp8`."""
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
