"""Python face of ``csrc/cuda/attn_sm90.cu`` -- the wgmma training attention (head dim 64 or 128, bf16, GQA, causal).

``fwd`` / ``bwd`` work on 2-D ``[B*S, heads*d]`` views (row stride free), so the packed QKV projection output is consumed
in place: Q, K and V are column ranges of ONE buffer and the backward writes dQ | dK | dV into one packed buffer that the
QKV projection's backward GEMMs read directly (no transposes, no concatenation).

``window`` (every entry point, default ``None``): causal sliding-window attention -- query row ``i`` attends to key ``j``
only when ``i - window < j <= i`` (``window`` keys counting its own; flash-attn's ``window_size=(window - 1, 0)``), measured
inside each document for the varlen forms.  The kernels skip the key / query blocks outside the band, so the cost is
O(S * window) instead of O(S^2).

``head_dim`` (every entry point, default 128): 64 or 128.  It sizes the outputs and sets the default softmax scale
``1 / sqrt(head_dim)``.
"""
import math

import torch

from deepspeed_b200.ops import native as N

HEAD_DIM = 128
HEAD_DIMS = (64, 128)  # head dims of the training kernels
BLOCK = 128


def supports(qkv2d, hq, hkv, d, S) -> bool:
    return (qkv2d.is_cuda and qkv2d.dtype == torch.bfloat16 and d in HEAD_DIMS and S % BLOCK == 0 and hq % hkv == 0
            and qkv2d.stride(-1) == 1 and qkv2d.stride(0) % 8 == 0 and qkv2d.data_ptr() % 16 == 0)


def _window(window, causal):
    """The kernels' ``window`` argument: 0 for no window."""
    from deepspeed_b200.ops.attention import check_sliding_window
    if window is None:
        return 0
    if not causal:
        raise ValueError("a sliding window is defined only for causal attention")
    return check_sliding_window(window)


def supports_fwd(x2d, hq, hkv, d, B, S) -> bool:
    """Forward-only (inference prefill): any sequence length when one sequence is launched at a time."""
    return (x2d.is_cuda and x2d.dtype == torch.bfloat16 and d == HEAD_DIM and hq % hkv == 0 and x2d.stride(-1) == 1
            and x2d.stride(0) % 8 == 0 and x2d.data_ptr() % 16 == 0 and (B == 1 or S % BLOCK == 0))


def fwd(q, k, v, B, S, hq, hkv, causal=True, scale=None, out=None, need_lse=True, window=None, head_dim=HEAD_DIM):
    """``q [B*S, hq*d]``, ``k / v [B*S, hkv*d]`` (2-D views, any row stride, ``d = head_dim``) ->
    ``(o [B*S, hq*d], lse [B, hq, S])``.
    ``S`` may be any length when ``B == 1`` (a ragged last block is masked inside the kernel)."""
    T = B * S
    window = _window(window, causal)
    if out is None:
        out = torch.empty(T, hq * head_dim, dtype=torch.bfloat16, device=q.device)
    lse = torch.empty(B, hq, S, dtype=torch.float32, device=q.device) if need_lse else None
    scale = float(scale) if scale is not None else 1.0 / math.sqrt(head_dim)
    rc = N.cuda().dsb_attn_fwd_bf16(N.ptr(q), N.ptr(k), N.ptr(v), N.ptr(out), N.ptr(lse), B, S, hq, hkv, head_dim, q.stride(0),
                                    k.stride(0), v.stride(0), out.stride(0), q.shape[1], k.shape[1], v.shape[1],
                                    N.c_f(scale), int(bool(causal)), window, N.stream())
    N.check(rc, "attn_fwd_bf16")
    return out, lse


def supports_varlen(qkv2d, hq, hkv, d) -> bool:
    """Packed sequences (:func:`fwd_varlen` / :func:`bwd_varlen`): :func:`supports` without the length rule."""
    return (qkv2d.is_cuda and qkv2d.dtype == torch.bfloat16 and d in HEAD_DIMS and hq % hkv == 0 and qkv2d.stride(-1) == 1
            and qkv2d.stride(0) % 8 == 0 and qkv2d.data_ptr() % 16 == 0)


def _check_cu(cu_seqlens, dev):
    if not (cu_seqlens.dtype == torch.int32 and cu_seqlens.dim() == 1 and cu_seqlens.numel() >= 1
            and cu_seqlens.device == dev and cu_seqlens.is_contiguous()):
        raise ValueError("cu_seqlens must be a contiguous 1-D int32 tensor on the attention's device")
    return cu_seqlens.numel() - 1


def fwd_varlen(q, k, v, cu_seqlens, max_seqlen, hq, hkv, causal=True, scale=None, out=None, need_lse=True, window=None,
               head_dim=HEAD_DIM):
    """Document-masked attention over packed sequences: ``q [T, hq*d]``, ``k / v [T, hkv*d]`` (2-D views, any row
    stride, ``d = head_dim``), ``cu_seqlens`` int32 ``[n_docs + 1]`` on the device (offsets from 0 to T, non-decreasing, empty documents
    allowed), ``max_seqlen`` >= the longest document.  Each token attends only to tokens of its own document.
    Returns ``(o [T, hq*d], lse [hq, T])`` -- the LSE is indexed by absolute token row."""
    T = q.shape[0]
    n_docs = _check_cu(cu_seqlens, q.device)
    window = _window(window, causal)
    if out is None:
        out = torch.empty(T, hq * head_dim, dtype=torch.bfloat16, device=q.device)
    lse = torch.empty(hq, T, dtype=torch.float32, device=q.device) if need_lse else None
    scale = float(scale) if scale is not None else 1.0 / math.sqrt(head_dim)
    rc = N.cuda().dsb_attn_varlen_fwd_bf16(N.ptr(q), N.ptr(k), N.ptr(v), N.ptr(out), N.ptr(lse), N.ptr(cu_seqlens), n_docs,
                                           int(max_seqlen), T, hq, hkv, head_dim, q.stride(0), k.stride(0), v.stride(0),
                                           out.stride(0), q.shape[1], k.shape[1], v.shape[1], N.c_f(scale),
                                           int(bool(causal)), window, N.stream())
    N.check(rc, "attn_varlen_fwd_bf16")
    return out, lse


def split_packed(qkv2d, hq, hkv, d=HEAD_DIM):
    """Column views (no copies) of a packed ``[T, (hq + 2 hkv) * d]`` projection output."""
    return qkv2d[:, :hq * d], qkv2d[:, hq * d:(hq + hkv) * d], qkv2d[:, (hq + hkv) * d:]


def bwd(d_o, q, k, v, o, lse, B, S, hq, hkv, causal=True, scale=None, dq=None, dk=None, dv=None, window=None,
        head_dim=HEAD_DIM):
    """Gradients of :func:`fwd` (same ``window`` and ``head_dim``).  ``dq / dk / dv`` may be column views of one packed
    ``[T, (hq + 2 hkv) * d]`` buffer."""
    T = B * S
    dev = q.device
    window = _window(window, causal)
    if dq is None:
        dq = torch.empty(T, hq * head_dim, dtype=torch.bfloat16, device=dev)
    if dk is None:
        dk = torch.empty(T, hkv * head_dim, dtype=torch.bfloat16, device=dev)
    if dv is None:
        dv = torch.empty(T, hkv * head_dim, dtype=torch.bfloat16, device=dev)
    if d_o.stride(-1) != 1:
        d_o = d_o.contiguous()
    work = torch.empty(2 * B * hq * S, dtype=torch.float32, device=dev)
    scale = float(scale) if scale is not None else 1.0 / math.sqrt(head_dim)
    rc = N.cuda().dsb_attn_bwd_bf16(N.ptr(q), N.ptr(k), N.ptr(v), N.ptr(o), N.ptr(d_o), N.ptr(lse), N.ptr(dq), N.ptr(dk),
                                    N.ptr(dv), N.ptr(work), B, S, hq, hkv, head_dim, q.stride(0), k.stride(0), v.stride(0),
                                    o.stride(0), d_o.stride(0), dq.stride(0), dk.stride(0), dv.stride(0), q.shape[1],
                                    k.shape[1], v.shape[1], N.c_f(scale), int(bool(causal)), window, N.stream())
    N.check(rc, "attn_bwd_bf16")
    return dq, dk, dv


def bwd_varlen(d_o, q, k, v, o, lse, cu_seqlens, max_seqlen, hq, hkv, causal=True, scale=None, dq=None, dk=None, dv=None,
               window=None, head_dim=HEAD_DIM):
    """Gradients of :func:`fwd_varlen` (same ``cu_seqlens`` / ``max_seqlen`` / ``window`` / ``head_dim``, ``lse [hq, T]``
    from it).  ``dq / dk / dv`` may be column views of one packed ``[T, (hq + 2 hkv) * d]`` buffer."""
    T = q.shape[0]
    dev = q.device
    n_docs = _check_cu(cu_seqlens, dev)
    window = _window(window, causal)
    if dq is None:
        dq = torch.empty(T, hq * head_dim, dtype=torch.bfloat16, device=dev)
    if dk is None:
        dk = torch.empty(T, hkv * head_dim, dtype=torch.bfloat16, device=dev)
    if dv is None:
        dv = torch.empty(T, hkv * head_dim, dtype=torch.bfloat16, device=dev)
    if d_o.stride(-1) != 1:
        d_o = d_o.contiguous()
    work = torch.empty(2 * hq * T, dtype=torch.float32, device=dev)
    scale = float(scale) if scale is not None else 1.0 / math.sqrt(head_dim)
    rc = N.cuda().dsb_attn_varlen_bwd_bf16(N.ptr(q), N.ptr(k), N.ptr(v), N.ptr(o), N.ptr(d_o), N.ptr(lse), N.ptr(dq),
                                           N.ptr(dk), N.ptr(dv), N.ptr(work), N.ptr(cu_seqlens), n_docs, int(max_seqlen), T,
                                           hq, hkv, head_dim, q.stride(0), k.stride(0), v.stride(0), o.stride(0),
                                           d_o.stride(0), dq.stride(0), dk.stride(0), dv.stride(0), q.shape[1], k.shape[1],
                                           v.shape[1], N.c_f(scale), int(bool(causal)), window, N.stream())
    N.check(rc, "attn_varlen_bwd_bf16")
    return dq, dk, dv

