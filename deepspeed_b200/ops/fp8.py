"""FP8 training recipe: tensorwise current scaling with power-of-two scales (torchao's "tensorwise", with Transformer
Engine's HYBRID formats).

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


def silu32(g):
    return g / (1 + torch.exp(-g))


def dsilu32(g):
    s = 1 / (1 + torch.exp(-g))
    return s * (1 + g * (1 - s))


# ---- the products of the two training nodes, on the kernels or in torch -------------------------------------------------
def gemm(a8, b8, sa, sb, native, out=None, accumulate=False):
    """bf16 ``[M, N]`` = ``sa sb a8 b8^T`` (``accumulate``: added to ``out`` before the one rounding)."""
    if native:
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        return K.fp8_matmul(a8, b8, sa, sb, out=out, epi=K.EPI_ACCUM if accumulate else K.EPI_STORE)
    c = matmul_reference(a8, b8, sa, sb)
    if accumulate:
        c = c + out.float()
    if out is None:
        return c.to(torch.bfloat16)
    return out.copy_(c)


def gemm_swiglu(a8, b8, sa, sb, native, save_gate_up=True):
    """``(act [M, I], gate|up [M, 2I] or None)`` for ``b8 = [gate; up] [2I, K]``: silu applied to the fp32 products."""
    if native:
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        I = b8.shape[0] // 2
        gu = torch.empty(a8.shape[0], 2 * I, dtype=torch.bfloat16, device=a8.device) if save_gate_up else None
        return K.fp8_matmul(a8, b8, sa, sb, epi=K.EPI_SWIGLU, out2=gu), gu
    gu = matmul_reference(a8, b8, sa, sb)
    g, u = gu.chunk(2, dim=1)
    return (silu32(g) * u).to(torch.bfloat16), (gu.to(torch.bfloat16) if save_gate_up else None)


def gemm_dswiglu(a8, b8, sa, sb, gu, native):
    """dgate|dup ``[M, 2I]`` (bf16) for the SwiGLU whose gate|up ``gu`` was saved: ``d = sa sb a8 b8^T`` in fp32, then
    ``dgate = d * u * silu'(g)`` and ``dup = d * silu(g)``."""
    if native:
        from deepspeed_b200.ops.kernels import gemm_sm100 as K
        out2 = torch.empty(gu.shape, dtype=torch.bfloat16, device=gu.device)
        K.fp8_matmul(a8, b8, sa, sb, epi=K.EPI_DSWIGLU, aux=gu, out2=out2)
        return out2
    d = matmul_reference(a8, b8, sa, sb)
    g, u = gu.float().chunk(2, dim=1)
    return torch.cat([d * u * dsilu32(g), d * silu32(g)], dim=1).to(torch.bfloat16)
