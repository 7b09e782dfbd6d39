"""Python face of ``csrc/cuda/gemm_sm90.cu`` -- the hand-written wgmma / TMA GEMM for sm_90a."""
import ctypes

import torch

from deepspeed_b200.ops import native as N

_checked = None


def supports(a, b, nt=True) -> bool:
    """Whether :func:`matmul_nt` takes these operands: bf16, 2-D, K-major (``a`` [M,K], ``b`` [N,K]), K % 8 == 0,
    16-byte aligned rows.  Only the NT form is answered here (``nt=False`` is always False); MN-major operands (NN / TN)
    go through :func:`matmul_2cta`, whose preconditions :func:`supports_2cta` checks."""
    if not nt:
        return False
    if a.dtype != torch.bfloat16 or b.dtype != torch.bfloat16 or a.dim() != 2 or b.dim() != 2:
        return False
    if a.stride(1) != 1 or b.stride(1) != 1 or a.shape[1] != b.shape[1]:
        return False
    K = a.shape[1]
    if K % 8 or a.stride(0) % 8 or b.stride(0) % 8 or a.data_ptr() % 16 or b.data_ptr() % 16:
        return False
    return a.shape[0] >= 128 and b.shape[0] >= 256 and K >= 64


def matmul_nt(a, b, out=None, sms=0):
    """``a [M,K] @ b[N,K]^T -> [M,N]`` bf16."""
    M, K = a.shape
    Nn = b.shape[0]
    if out is None:
        out = torch.empty(M, Nn, dtype=torch.bfloat16, device=a.device)
    rc = N.cuda().dsb_gemm_nt_bf16(N.ptr(a), N.ptr(b), N.ptr(out), M, Nn, K, a.stride(0), b.stride(0), out.stride(0), sms,
                                   N.stream())
    N.check(rc, "gemm_nt_bf16")
    return out


def supports_grouped(x, w, offsets) -> bool:
    """bf16 rows [R, K] (row stride % 8), stacked weights [E, N, K] contiguous, int32 device offsets [E + 1]."""
    return (x.is_cuda and x.dtype == torch.bfloat16 and torch.is_tensor(w) and w.dtype == torch.bfloat16 and w.dim() == 3
            and w.is_contiguous() and x.dim() == 2 and x.stride(1) == 1 and x.shape[1] == w.shape[2] and x.shape[1] % 8 == 0
            and w.shape[1] % 8 == 0 and x.stride(0) % 8 == 0 and w.shape[0] <= 256 and torch.is_tensor(offsets)
            and offsets.is_cuda and offsets.dtype == torch.int32 and x.data_ptr() % 16 == 0 and w.data_ptr() % 16 == 0
            and x.shape[1] >= 64)


def grouped_matmul_nt(x, w, offsets, out=None, sms=0):
    """Grouped (MoE) GEMM: ``out[r] = x[r] @ w[e]^T`` for ``offsets[e] <= r < offsets[e+1]`` in ONE persistent wgmma
    launch; ``offsets`` stays on the device (no host sync, CUDA-graph capturable)."""
    R, K = x.shape
    E, Nn, _ = w.shape
    if out is None:
        out = torch.empty(R, Nn, dtype=torch.bfloat16, device=x.device)
    rc = N.cuda().dsb_gemm_grouped_nt_bf16(N.ptr(x), N.ptr(w), N.ptr(out), N.ptr(offsets), R, E, Nn, K, x.stride(0), out.stride(0),
                                           sms, N.stream())
    N.check(rc, "gemm_grouped_nt_bf16")
    return out


RAGGED_ALIGN = 64  # rows per ragged segment granule: every expert offset is a multiple of it


def _ragged_rows_ok(t):
    return (t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 8 == 0
            and t.data_ptr() % 16 == 0 and t.shape[1] % 8 == 0)


def supports_ragged(x, w, offsets) -> bool:
    """Whether the ragged (dropless MoE) entry points take expert-sorted rows ``x [R, K]``, a stacked weight ``w [E, *, *]``
    (contiguous) and int32 device offsets ``[E + 1]``.  The shape conditions each form adds (``K % 64``, ``I % 128``) are
    checked by the kernel's host side, which refuses with :class:`NativeOpError`."""
    return (_ragged_rows_ok(x) and torch.is_tensor(w) and w.is_cuda and w.dtype == torch.bfloat16 and w.dim() == 3
            and w.is_contiguous() and w.data_ptr() % 16 == 0 and 1 <= w.shape[0] <= 256 and torch.is_tensor(offsets)
            and offsets.is_cuda and offsets.dtype == torch.int32 and offsets.is_contiguous()
            and offsets.numel() == w.shape[0] + 1)


def ragged_matmul(x, w, offsets, b_mn, out=None, epi=0, aux=None, out2=None, sms=0):
    """m-tiled ragged GEMM over expert-sorted rows (``dsb_gemm_ragged_bf16``; offsets stay on the device):

    * ``b_mn=False``: ``w [E, N, K]``, ``out[r] = x[r] @ w[e]^T``; with ``epi=EPI_SWIGLU`` ``w`` is ``[E, 2I, K]`` (gate
      rows, then up rows), ``out [R, I] = silu(gate) * up`` and ``out2`` (optional ``[R, 2I]``) receives gate|up;
    * ``b_mn=True``: ``w [E, K, N]``, ``out[r] = x[r] @ w[e]``; with ``epi=EPI_DSWIGLU`` ``aux`` is the saved gate|up
      ``[R, 2N]``, ``out2`` the ``[R, 2N]`` dgate|dup and ``out`` its left half.

    Segments are 64-row aligned and zero-padded (see the entry point); malformed device offsets make the kernel write
    nothing.  Rows of ``out`` outside ``[offsets[0], offsets[E])`` are not written.  Shapes that do not fit together raise
    :class:`NativeOpError` before anything is launched (the tensor maps are built from them)."""
    R, K = x.shape
    E = w.shape[0]
    if epi == EPI_SWIGLU:
        Nn = w.shape[1] // 2
    else:
        Nn = w.shape[2] if b_mn else w.shape[1]
    wk = w.shape[1] if b_mn else w.shape[2]
    bad = (w.dim() != 3 or wk != K or (epi == EPI_SWIGLU and w.shape[1] != 2 * Nn) or offsets.numel() != E + 1
           or (out is not None and tuple(out.shape) != (R, Nn)))
    if epi == EPI_SWIGLU and out2 is not None:
        bad = bad or tuple(out2.shape) != (R, 2 * Nn)
    if epi == EPI_DSWIGLU:
        bad = bad or aux is None or out2 is None or tuple(aux.shape) != (R, 2 * Nn) or tuple(out2.shape) != (R, 2 * Nn)
    if bad:
        raise N.NativeOpError(f"gemm_ragged_bf16: x {tuple(x.shape)}, w {tuple(w.shape)}, offsets {tuple(offsets.shape)} "
                              f"and the outputs do not fit together (b_mn={int(b_mn)}, epi={epi})")
    if out is None:
        out = torch.empty(R, Nn, dtype=torch.bfloat16, device=x.device)
    rc = N.cuda().dsb_gemm_ragged_bf16(N.ptr(x), N.ptr(w), N.ptr(out), N.ptr(offsets), R, E, Nn, K, x.stride(0),
                                       out.stride(0), int(b_mn), int(epi), N.ptr(aux),
                                       aux.stride(0) if aux is not None else 0, N.ptr(out2),
                                       out2.stride(0) if out2 is not None else 0, sms, N.stream())
    N.check(rc, "gemm_ragged_bf16")
    return out


def ragged_wgrad(a, b, offsets, E, out=None, accumulate=False, sms=0):
    """Variable-K grouped weight gradient (``dsb_gemm_ragged_wgrad_bf16``): ``out[e] = a[rows of e]^T @ b[rows of e]``
    (``accumulate``: added to ``out[e]``) for ``a [R, M]``, ``b [R, N]``, ``out [E, M, N]`` contiguous, in one launch.
    An expert without rows gets zeros (or keeps ``out[e]`` when accumulating)."""
    R, M = a.shape
    Nn = b.shape[1]
    if b.shape[0] != R or offsets.numel() != E + 1:
        raise N.NativeOpError(f"gemm_ragged_wgrad_bf16: a {tuple(a.shape)}, b {tuple(b.shape)} and offsets "
                              f"{tuple(offsets.shape)} do not share the rows of {E} experts")
    if out is None:
        assert not accumulate
        out = torch.empty(E, M, Nn, dtype=torch.bfloat16, device=a.device)
    if not out.is_contiguous() or tuple(out.shape) != (E, M, Nn):
        raise N.NativeOpError(f"gemm_ragged_wgrad_bf16: out must be a contiguous [{E}, {M}, {Nn}] tensor")
    if R == 0:
        return out if accumulate else out.zero_()
    rc = N.cuda().dsb_gemm_ragged_wgrad_bf16(N.ptr(a), N.ptr(b), N.ptr(out), N.ptr(offsets), R, E, M, Nn, a.stride(0),
                                             b.stride(0), int(bool(accumulate)), sms, N.stream())
    N.check(rc, "gemm_ragged_wgrad_bf16")
    return out


def matmul_nt_2cta(a, b, out=None, sms=0):
    """Same contract as :func:`matmul_nt` through the general entry point (grouped tile rasterisation)."""
    M, K = a.shape
    Nn = b.shape[0]
    if out is None:
        out = torch.empty(M, Nn, dtype=torch.bfloat16, device=a.device)
    rc = N.cuda().dsb_gemm_nt_bf16_2cta(N.ptr(a), N.ptr(b), N.ptr(out), M, Nn, K, a.stride(0), b.stride(0), out.stride(0),
                                        sms, N.stream())
    N.check(rc, "gemm_nt_bf16_2cta")
    return out


EPI_STORE, EPI_ACCUM, EPI_SWIGLU, EPI_DSWIGLU = 0, 1, 2, 3


def matmul_2cta(a, b, a_mn: bool, b_mn: bool, out=None, sms=0, epi=EPI_STORE, aux=None, out2=None, inter=0, group_m=8):
    """General kernel with selectable operand majorness and fused epilogue.

    ``a_mn=False``: ``a`` is [M, K];  ``a_mn=True``: ``a`` is [K, M] (the kernel multiplies by its transpose).
    ``b_mn=False``: ``b`` is [N, K];  ``b_mn=True``: ``b`` is [K, N].
    Result ``[M, N]`` bf16.  Rows may be strided (views of larger buffers).
    ``epi``: ``EPI_ACCUM`` adds into ``out``; ``EPI_SWIGLU`` -- ``b`` is ``[2*inter, K]`` (gate rows, then up rows), ``out``
    is ``[M, inter]`` = ``silu(gate) * up`` and ``out2`` (optional ``[M, 2*inter]``) receives gate|up; ``EPI_DSWIGLU`` --
    ``aux`` is the saved gate|up ``[M, 2*inter]``, ``out`` the dgate half and ``out2`` the whole ``[M, 2*inter]`` dgate|dup.
    ``group_m``: 128-row m-blocks per rasterisation super-group (L2 locality)."""
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    if epi == EPI_SWIGLU:
        Nn = inter
    else:
        Nn = b.shape[1] if b_mn else b.shape[0]
    if out is None:
        assert epi != EPI_ACCUM
        out = torch.empty(M, Nn, dtype=torch.bfloat16, device=a.device)
    rc = N.cuda().dsb_gemm_bf16_2cta_ex(N.ptr(a), N.ptr(b), N.ptr(out), M, Nn, K, a.stride(0), b.stride(0), out.stride(0),
                                        int(a_mn), int(b_mn), int(epi), N.ptr(aux), aux.stride(0) if aux is not None else 0,
                                        N.ptr(out2), out2.stride(0) if out2 is not None else 0, int(inter), int(group_m),
                                        sms, N.stream())
    N.check(rc, "gemm_bf16_2cta_ex")
    return out


def fp8_matmul(a, b, sa_inv, sb_inv, out=None, epi=EPI_STORE, aux=None, out2=None, group_m=8, sms=0):
    """Tensorwise-scaled FP8 GEMM (``dsb_gemm_fp8``): ``out [M, N] (bf16) = epi(sa_inv * sb_inv * a @ b^T)`` for K-major
    ``a [M, K]`` (``float8_e4m3fn`` or ``float8_e5m2``) and ``b [N, K]`` (``float8_e4m3fn``); ``sa_inv`` / ``sb_inv`` are
    one-element fp32 device tensors, read by the kernel (no host synchronisation).  Every 128 products are promoted into
    an fp32 accumulator: the tensor core's reduced-precision accumulation never carries the running sum, so it costs
    about 2**-14 of a block's magnitudes whatever K is, and nothing where a block sums exactly (small integers on a grid).

    ``epi``: ``EPI_ACCUM`` adds into ``out``; ``EPI_SWIGLU`` (``a`` e4m3) -- ``b`` is ``[2N, K]`` (gate rows, then up rows),
    ``out [M, N] = silu(g) * u`` and ``out2`` (optional ``[M, 2N]``) receives g|u; ``EPI_DSWIGLU`` (``a`` e5m2) -- ``aux`` is
    the saved gate|up ``[M, 2N]``, ``out2`` the ``[M, 2N]`` dgate|dup and ``out`` its left half (allocated as a view of
    ``out2`` when None).  Shapes that do not fit together raise :class:`NativeOpError` before a tensor map is built; the
    kernel's host side refuses the rest (see the entry point)."""
    fmt = {torch.float8_e4m3fn: N.F8E4M3, torch.float8_e5m2: N.F8E5M2}.get(a.dtype)
    M, K = a.shape if a.dim() == 2 else (0, 0)
    Nn = b.shape[0] // 2 if epi == EPI_SWIGLU else b.shape[0]
    bad = (fmt is None or b.dtype != torch.float8_e4m3fn or a.dim() != 2 or b.dim() != 2 or b.shape[1] != K
           or (epi == EPI_SWIGLU and b.shape[0] != 2 * Nn) or a.stride(1) != 1 or b.stride(1) != 1
           or sa_inv is None or sb_inv is None or sa_inv.dtype != torch.float32 or sb_inv.dtype != torch.float32
           or sa_inv.numel() != 1 or sb_inv.numel() != 1)
    if out is not None:
        bad = bad or tuple(out.shape) != (M, Nn) or out.dtype != torch.bfloat16 or out.stride(1) != 1
    if out2 is not None:
        bad = bad or tuple(out2.shape) != (M, 2 * Nn) or out2.dtype != torch.bfloat16 or out2.stride(1) != 1
    if aux is not None:
        bad = bad or tuple(aux.shape) != (M, 2 * Nn) or aux.dtype != torch.bfloat16 or aux.stride(1) != 1
    if epi == EPI_DSWIGLU:
        bad = bad or aux is None or out2 is None
    if epi == EPI_ACCUM:
        bad = bad or out is None
    if bad:
        raise N.NativeOpError(f"gemm_fp8: a {tuple(a.shape)} {a.dtype}, b {tuple(b.shape)} {b.dtype}, the scales and the "
                              f"outputs do not fit together (epi={epi})")
    if out is None:
        out = out2[:, :Nn] if epi == EPI_DSWIGLU else torch.empty(M, Nn, dtype=torch.bfloat16, device=a.device)
    rc = N.cuda().dsb_gemm_fp8(N.ptr(a), N.ptr(b), N.ptr(out), M, Nn, K, a.stride(0), b.stride(0), out.stride(0), fmt,
                               N.ptr(sa_inv), N.ptr(sb_inv), int(epi), N.ptr(aux), aux.stride(0) if aux is not None else 0,
                               N.ptr(out2), out2.stride(0) if out2 is not None else 0, int(group_m), sms, N.stream())
    N.check(rc, "gemm_fp8")
    return out


def fp8_matmul_block(a, b, sa_inv, sb_inv, out=None, epi=EPI_STORE, aux=None, out2=None, group_m=8, sms=0):
    """Blockwise-scaled FP8 GEMM (``dsb_gemm_fp8_block``): :func:`fp8_matmul` with ``sa_inv [ceil(K/128), M]`` (one scale
    per row of ``a`` and k-block of 128) and ``sb_inv [ceil(rows of b / 128), ceil(K/128)]`` (one per 128 x 128 block of
    ``b``) in place of the two scalars; each k-block's partial product is scaled as it is promoted,
    ``out = epi(sum_kb sa_inv[kb, m] * sb_inv[n // 128, kb] * a[m, kb] @ b[n, kb]^T)``.  Operands, epilogues and outputs
    are those of :func:`fp8_matmul`."""
    fmt = {torch.float8_e4m3fn: N.F8E4M3, torch.float8_e5m2: N.F8E5M2}.get(a.dtype)
    M, K = a.shape if a.dim() == 2 else (0, 0)
    Nn = b.shape[0] // 2 if epi == EPI_SWIGLU else b.shape[0]
    kb = -(-K // 128)
    bad = (fmt is None or b.dtype != torch.float8_e4m3fn or a.dim() != 2 or b.dim() != 2 or b.shape[1] != K
           or (epi == EPI_SWIGLU and b.shape[0] != 2 * Nn) or a.stride(1) != 1 or b.stride(1) != 1
           or sa_inv is None or sb_inv is None or sa_inv.dtype != torch.float32 or sb_inv.dtype != torch.float32
           or tuple(sa_inv.shape) != (kb, M) or tuple(sb_inv.shape) != (-(-b.shape[0] // 128), kb)
           or sa_inv.stride(1) != 1 or sb_inv.stride(1) != 1)
    if out is not None:
        bad = bad or tuple(out.shape) != (M, Nn) or out.dtype != torch.bfloat16 or out.stride(1) != 1
    if out2 is not None:
        bad = bad or tuple(out2.shape) != (M, 2 * Nn) or out2.dtype != torch.bfloat16 or out2.stride(1) != 1
    if aux is not None:
        bad = bad or tuple(aux.shape) != (M, 2 * Nn) or aux.dtype != torch.bfloat16 or aux.stride(1) != 1
    if epi == EPI_DSWIGLU:
        bad = bad or aux is None or out2 is None
    if epi == EPI_ACCUM:
        bad = bad or out is None
    if bad:
        raise N.NativeOpError(f"gemm_fp8_block: a {tuple(a.shape)} {a.dtype}, b {tuple(b.shape)} {b.dtype}, the scales and "
                              f"the outputs do not fit together (epi={epi})")
    if out is None:
        out = out2[:, :Nn] if epi == EPI_DSWIGLU else torch.empty(M, Nn, dtype=torch.bfloat16, device=a.device)
    rc = N.cuda().dsb_gemm_fp8_block(N.ptr(a), N.ptr(b), N.ptr(out), M, Nn, K, a.stride(0), b.stride(0), out.stride(0), fmt,
                                     N.ptr(sa_inv), sa_inv.stride(0), N.ptr(sb_inv), sb_inv.stride(0), int(epi), N.ptr(aux),
                                     aux.stride(0) if aux is not None else 0, N.ptr(out2),
                                     out2.stride(0) if out2 is not None else 0, int(group_m), sms, N.stream())
    N.check(rc, "gemm_fp8_block")
    return out


FP8_RAGGED_ALIGN = 128  # rows per FP8 ragged segment granule: the FP8 k-block, scale strip and scale block


def _fp8_scales_ok(s, shape, block):
    if s is None or s.dtype != torch.float32 or not s.is_cuda:
        return False
    if not block:
        return s.numel() == 1
    return tuple(s.shape) == shape and s.stride(1) == 1


def fp8_ragged_matmul(a, b, offsets, sa_inv, sb_inv, E, out=None, epi=EPI_STORE, aux=None, out2=None, block=False, sms=0):
    """m-tiled ragged FP8 GEMM over expert-sorted rows (``dsb_gemm_fp8_ragged``; offsets stay on the device, 128-row
    segments).  The format of ``a [R, K]`` picks the form:

    * ``float8_e4m3fn`` (forward): ``b`` is the stacked weight viewed ``[E * Nb, K]``; ``out[r] = a[r] @ b_e^T`` with
      ``b_e = b[e Nb:(e+1) Nb]`` (``Nb = N``), or with ``epi=EPI_SWIGLU`` (``Nb = 2N``, gate rows then up rows)
      ``out [R, N] = silu(gate) * up`` and ``out2`` (optional ``[R, 2N]``) the gate|up;
    * ``float8_e5m2`` (dgrad): ``b [N, E * K]`` is the transposed cast of that view; ``out[r] = a[r] @ b_e^T`` with
      ``b_e = b[:, e K:(e+1) K]``, or with ``epi=EPI_DSWIGLU`` ``aux`` the saved gate|up ``[R, 2N]``, ``out2`` the
      ``[R, 2N]`` dgate|dup and ``out`` its left half.

    Tensorwise (``block=False``): ``sa_inv`` / ``sb_inv`` one-element fp32 device tensors.  Blockwise: ``sa_inv
    [ceil(K/128), R]`` (strips of ``a``) and ``sb_inv`` the block scales of ``b`` (``[rows of b / 128, ceil(cols of b /
    128)]``).  Rows of ``out`` outside ``[offsets[0], offsets[E])`` are not written.  Shapes that do not fit together
    raise :class:`NativeOpError` before anything is launched."""
    fmt = {torch.float8_e4m3fn: N.F8E4M3, torch.float8_e5m2: N.F8E5M2}.get(a.dtype)
    dgrad = fmt == N.F8E5M2
    R, K = a.shape if a.dim() == 2 else (0, 0)
    bad = fmt is None or a.dim() != 2 or b.dim() != 2 or b.dtype != torch.float8_e4m3fn or a.stride(1) != 1
    bad = bad or b.stride(1) != 1 or not torch.is_tensor(offsets) or offsets.dtype != torch.int32
    bad = bad or offsets.numel() != E + 1 or not offsets.is_cuda or not offsets.is_contiguous() or E < 1
    Nn = 0
    if not bad:
        if dgrad:
            Nn = b.shape[0]
            bad = b.shape[1] != E * K or epi not in (EPI_STORE, EPI_DSWIGLU)
        else:
            Nb = b.shape[0] // E
            Nn = Nb // 2 if epi == EPI_SWIGLU else Nb
            bad = b.shape[0] != E * Nb or b.shape[1] != K or epi not in (EPI_STORE, EPI_SWIGLU)
            bad = bad or (epi == EPI_SWIGLU and Nb != 2 * Nn)
        kb = -(-K // 128)
        bad = bad or not _fp8_scales_ok(sa_inv, (kb, R), block)
        bad = bad or not _fp8_scales_ok(sb_inv, (-(-b.shape[0] // 128), -(-b.shape[1] // 128)), block)
    for t, shape in ((out, (R, Nn)), (out2, (R, 2 * Nn)), (aux, (R, 2 * Nn))):
        if t is not None:
            bad = bad or tuple(t.shape) != shape or t.dtype != torch.bfloat16 or t.stride(1) != 1
    if epi == EPI_DSWIGLU:
        bad = bad or aux is None or out2 is None
    if bad:
        raise N.NativeOpError(f"gemm_fp8_ragged: a {tuple(a.shape)} {a.dtype}, b {tuple(b.shape)} {b.dtype}, offsets, "
                              f"the scales and the outputs do not fit together (E={E}, epi={epi}, block={block})")
    if out is None:
        out = out2[:, :Nn] if epi == EPI_DSWIGLU else torch.empty(R, Nn, dtype=torch.bfloat16, device=a.device)
    ld = lambda t: t.stride(0) if t is not None else 0
    rc = N.cuda().dsb_gemm_fp8_ragged(N.ptr(a), N.ptr(b), N.ptr(out), N.ptr(offsets), R, E, Nn, K, a.stride(0),
                                      b.stride(0), out.stride(0), fmt, N.ptr(sa_inv), ld(sa_inv) if block else 0,
                                      N.ptr(sb_inv), ld(sb_inv) if block else 0, int(epi), N.ptr(aux), ld(aux),
                                      N.ptr(out2), ld(out2), int(bool(block)), sms, N.stream())
    N.check(rc, "gemm_fp8_ragged")
    return out


def fp8_ragged_wgrad(a, b, offsets, sa_inv, sb_inv, E, out=None, accumulate=False, block=False, sms=0):
    """Variable-K FP8 weight gradient (``dsb_gemm_fp8_ragged_wgrad``): ``out[e] (+)= a[:, rows of e] @ b[:, rows of
    e]^T`` for ``a [M, R]`` (``float8_e5m2``, the transposed gradient) and ``b [N, R]`` (``float8_e4m3fn``, the transposed
    input), ``out [E, M, N]`` contiguous bf16, in one launch over 128-row segments.  An expert without rows gets zeros
    (or keeps ``out[e]`` when accumulating).  Blockwise: ``sa_inv [ceil(R/128), M]`` (strips along the rows) and ``sb_inv
    [ceil(N/128), ceil(R/128)]``; tensorwise: one-element tensors."""
    M, R = a.shape if a.dim() == 2 else (0, 0)
    Nn = b.shape[0] if b.dim() == 2 else 0
    kb = -(-R // 128)
    bad = (a.dim() != 2 or b.dim() != 2 or a.dtype != torch.float8_e5m2 or b.dtype != torch.float8_e4m3fn
           or b.shape[1] != R or a.stride(1) != 1 or b.stride(1) != 1 or not torch.is_tensor(offsets)
           or offsets.dtype != torch.int32 or offsets.numel() != E + 1 or not offsets.is_cuda
           or not offsets.is_contiguous() or not _fp8_scales_ok(sa_inv, (kb, M), block)
           or not _fp8_scales_ok(sb_inv, (-(-Nn // 128), kb), block))
    if out is None and not bad:
        assert not accumulate
        out = torch.empty(E, M, Nn, dtype=torch.bfloat16, device=a.device)
    if bad or not out.is_contiguous() or tuple(out.shape) != (E, M, Nn) or out.dtype != torch.bfloat16:
        raise N.NativeOpError(f"gemm_fp8_ragged_wgrad: a {tuple(a.shape)} {a.dtype}, b {tuple(b.shape)} {b.dtype}, offsets, "
                              f"the scales and out do not fit together (E={E}, block={block})")
    ld = lambda t: t.stride(0) if block else 0
    rc = N.cuda().dsb_gemm_fp8_ragged_wgrad(N.ptr(a), N.ptr(b), N.ptr(out), N.ptr(offsets), R, E, M, Nn, a.stride(0),
                                            b.stride(0), N.ptr(sa_inv), ld(sa_inv), N.ptr(sb_inv), ld(sb_inv),
                                            int(bool(accumulate)), int(bool(block)), sms, N.stream())
    N.check(rc, "gemm_fp8_ragged_wgrad")
    return out


def supports_2cta(a, b, a_mn, b_mn, out=None) -> bool:
    ok = lambda t: (t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 8 == 0
                    and t.data_ptr() % 16 == 0 and t.shape[1] % 8 == 0)
    return ok(a) and ok(b) and (out is None or ok(out))


def matmul_nn(a, b, out=None):
    """a [M, K] @ b [K, N]."""
    return matmul_2cta(a, b, False, True, out=out)


def matmul_tn(a, b, out=None):
    """a[K, M]^T @ b[K, N]."""
    return matmul_2cta(a, b, True, True, out=out)


def matmul_nt_allgather(a, b_view, local_full, peers, flags, shard_bytes, chunk_bytes, b_offset_bytes, world, rank, epoch,
                        comm_ctas=16, out=None, sms=0):
    """Fused all-gather + GEMM (see kernel header).  ``b_view`` is the [N,K] view of the weight inside
    ``local_full`` (the unit's gathered buffer, being filled by this very kernel)."""
    M, K = a.shape
    Nn = b_view.shape[0]
    if out is None:
        out = torch.empty(M, Nn, dtype=torch.bfloat16, device=a.device)
    arr = (ctypes.c_void_p * world)(*[ctypes.c_void_p(p) for p in peers])
    rc = N.cuda().dsb_gemm_nt_bf16_allgather(N.ptr(a), N.ptr(b_view), N.ptr(out), M, Nn, K, a.stride(0), b_view.stride(0),
                                             out.stride(0), arr, N.ptr(local_full), N.ptr(flags),
                                             ctypes.c_int64(shard_bytes), ctypes.c_int64(chunk_bytes),
                                             ctypes.c_int64(b_offset_bytes), world, rank, comm_ctas,
                                             ctypes.c_uint32(epoch), sms, N.stream())
    N.check(rc, "gemm_nt_bf16_allgather")
    return out


def self_check() -> bool:
    """One-time numerical self test against torch.matmul on this device."""
    global _checked
    if _checked is not None:
        return _checked
    try:
        torch.manual_seed(0)
        a = torch.randn(384, 320, device="cuda", dtype=torch.bfloat16)
        b = torch.randn(768, 320, device="cuda", dtype=torch.bfloat16)
        c = matmul_nt(a, b)
        ref = (a.float() @ b.float().t())
        torch.cuda.synchronize()
        err = (c.float() - ref).abs().max().item()
        _checked = bool(err < 0.05 * ref.abs().max().item() + 0.5) and bool(torch.isfinite(c).all())
    except Exception:
        _checked = False
    return _checked
