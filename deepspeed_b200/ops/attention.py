"""Causal self-attention on a packed QKV buffer.

``causal_attention(qkv2d, B, S, hq, hkv, d, rope, positions)``: rotates Q and K **in place** inside the
packed projection output (one launch, ``transformer.cu:rope_kernel``), runs the attention core and
returns ``[B*S, hq*d]``.  The backward produces one packed ``dqkv`` buffer and un-rotates it in place.

Attention-core backends (``backend=`` or ``DSB200_ATTN``):
  * ``cudnn`` / ``flash`` / ``efficient`` / ``math`` -- ``torch.nn.functional.scaled_dot_product_attention``
    with that SDPA backend (library path; cuDNN has a Hopper FMHA);
  * ``flash_attn`` -- the flash-attn package;
  * ``native`` -- the framework's own sm_90a kernel (``csrc/cuda/attn_sm90.cu``, bf16, head dim 64 or 128) when built;
  * ``auto`` -- native if available, else cudnn -> flash -> efficient -> math priority order.
Packed sequences (``cu_seqlens=``): the ``B*S`` token rows hold several documents at offsets ``cu_seqlens`` and every token
attends only within its own document (flash-attn's varlen semantics).  ``auto`` / ``native`` run the in-tree varlen
kernel; any other backend, dtype, a head dim other than 64 or 128, or a CPU tensor runs one SDPA call per document.
Sliding window (``sliding_window=W``, an int >= 1): query row ``i`` attends to key ``j`` only when ``i - W < j <= i`` -- W keys
counting its own position (HF's ``sliding_window``, flash-attn's ``window_size=(W - 1, 0)``), measured inside each document
with ``cu_seqlens``.  ``auto`` / ``native`` run the in-tree windowed kernel (head dim 64 or 128), which skips the tiles
outside the band; every other case runs SDPA with an explicit boolean band mask per sequence or document.  A window that covers the whole sequence
(or the longest document) is dropped, so such a call is exactly the unwindowed one.
Role parity: the reference has no training attention kernel of its own for HF models (it relies on
PyTorch / flash-attn, ``sequence/fpdt_layer.py:235``); the BERT-era fused layer is ``ops/transformer``.
"""
import numbers
import os

import torch
import torch.nn.functional as F

from deepspeed_b200.ops.kernels.transformer_ops import rope_qk_inplace

_ENV = os.environ.get("DSB200_ATTN", "").lower()


def check_sliding_window(sliding_window):
    """``None`` (no window) or the window as an int >= 1; anything else raises ``ValueError``."""
    if sliding_window is None:
        return None
    if isinstance(sliding_window, bool) or not isinstance(sliding_window, numbers.Integral) or sliding_window < 1:
        raise ValueError(f"sliding_window must be None or an int >= 1, got {sliding_window!r}")
    return int(sliding_window)


def _sdpa_band(q, k, v, window, scale=None):
    """Causal sliding-window SDPA through an explicit band mask.  SDPA has no window argument and rejects ``is_causal``
    together with ``attn_mask``, so causality is folded into the mask.  Flash takes no mask: a CUDA tensor runs one of
    the memory-efficient, cuDNN or math kernels."""
    i = torch.arange(q.shape[-2], device=q.device)
    diff = i[:, None] - i[None, :]
    mask = (diff >= 0) & (diff < window)  # True where query i may attend key j: i - window < j <= i
    if q.shape[1] != k.shape[1]:
        rep = q.shape[1] // k.shape[1]
        k, v = k.repeat_interleave(rep, dim=1), v.repeat_interleave(rep, dim=1)
    if not q.is_cuda:
        return F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=scale)
    from torch.nn.attention import SDPBackend, sdpa_kernel
    with sdpa_kernel([SDPBackend.EFFICIENT_ATTENTION, SDPBackend.CUDNN_ATTENTION, SDPBackend.MATH]):
        return F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=scale)


def _sdpa(q, k, v, backend, causal=True, scale=None, window=None):
    if window is not None and window < q.shape[-2]:
        return _sdpa_band(q, k, v, window, scale)
    gqa = q.shape[1] != k.shape[1]
    kw = dict(is_causal=causal, scale=scale)
    if gqa:
        kw["enable_gqa"] = True
    if not q.is_cuda or backend in ("math", ):
        if gqa:
            rep = q.shape[1] // k.shape[1]
            k, v = k.repeat_interleave(rep, dim=1), v.repeat_interleave(rep, dim=1)
            kw.pop("enable_gqa")
        return F.scaled_dot_product_attention(q, k, v, **kw)
    from torch.nn.attention import SDPBackend, sdpa_kernel
    table = {
        "cudnn": [SDPBackend.CUDNN_ATTENTION],
        "flash": [SDPBackend.FLASH_ATTENTION],
        "efficient": [SDPBackend.EFFICIENT_ATTENTION],
        "auto": [SDPBackend.CUDNN_ATTENTION, SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION,
                 SDPBackend.MATH],
    }
    order = table.get(backend, table["auto"])
    try:
        with sdpa_kernel(order, set_priority=True):
            return F.scaled_dot_product_attention(q, k, v, **kw)
    except TypeError:  # older signature without set_priority
        with sdpa_kernel(order):
            return F.scaled_dot_product_attention(q, k, v, **kw)


class _PackedCausalAttention(torch.autograd.Function):

    @staticmethod
    def forward(ctx, qkv, B, S, hq, hkv, d, rope, positions, backend, window):
        T = B * S
        if rope is not None:
            rope_qk_inplace(qkv, hq, hkv, d, rope, positions, S, backward=False)
        x = qkv.view(B, S, hq + 2 * hkv, d)
        q = x[:, :, :hq].transpose(1, 2)
        k = x[:, :, hq:hq + hkv].transpose(1, 2)
        v = x[:, :, hq + hkv:].transpose(1, 2)
        with torch.enable_grad():
            qd, kd, vd = (t.detach().requires_grad_(True) for t in (q, k, v))
            out = _sdpa(qd, kd, vd, backend, window=window)
        ctx.graph = (qd, kd, vd, out)
        ctx.meta = (B, S, hq, hkv, d, rope, positions)
        ctx.qkv_shape = qkv.shape
        return out.detach().transpose(1, 2).reshape(T, hq * d)

    @staticmethod
    def backward(ctx, dout):
        B, S, hq, hkv, d, rope, positions = ctx.meta
        qd, kd, vd, out = ctx.graph
        ctx.graph = None
        do = dout.view(B, S, hq, d).transpose(1, 2)
        dq, dk, dv = torch.autograd.grad(out, (qd, kd, vd), do)
        dqkv = torch.empty(ctx.qkv_shape, dtype=dout.dtype, device=dout.device)
        y = dqkv.view(B, S, hq + 2 * hkv, d)
        y[:, :, :hq].copy_(dq.transpose(1, 2))
        y[:, :, hq:hq + hkv].copy_(dk.transpose(1, 2))
        y[:, :, hq + hkv:].copy_(dv.transpose(1, 2))
        if rope is not None:
            rope_qk_inplace(dqkv, hq, hkv, d, rope, positions, S, backward=True)
        return dqkv, None, None, None, None, None, None, None, None, None


_TABLE = None


def _native_wins(B, S, hq, hkv, d) -> bool:
    """``auto``: the measured per-shape choice between the in-tree wgmma kernel and the cuDNN library kernel
    (``attention_table.json`` next to this file, written from ``scripts/bench_attention.py`` runs on an H100: fwd + bwd
    milliseconds of both).  Shapes not in the table use the library; no table has been measured on H100, so the in-tree
    kernel is opt-in there (``attention_backend="native"``)."""
    global _TABLE
    if _TABLE is None:
        import json
        try:
            with open(os.path.join(os.path.dirname(__file__), "attention_table.json")) as f:
                _TABLE = json.load(f).get("shapes", {})
        except (OSError, ValueError):
            _TABLE = {}
    e = _TABLE.get(f"B{B}_S{S}_hq{hq}_hkv{hkv}_d{d}")
    return bool(e and e.get("choice") == "native")


def document_positions(cu_seqlens, T):
    """int32 ``[T]`` position of every token inside its document (0 at each document start), built on ``cu_seqlens``'
    device without a host sync."""
    starts = cu_seqlens[:-1].long()
    lens = cu_seqlens[1:].long() - starts
    first = torch.repeat_interleave(starts, lens, output_size=T)
    return (torch.arange(T, device=cu_seqlens.device) - first).to(torch.int32)


def check_cu_seqlens(cu_seqlens, T, max_seqlen=None):
    """Validate document offsets into ``T`` token rows and return ``max_seqlen``.  A CPU tensor (the usual data-loader
    output) is checked in full: 1-D int32, starts at 0, ends at ``T``, non-decreasing; ``max_seqlen`` is derived from it
    when not given.  A device tensor is only checked for shape and dtype (no host sync) and needs ``max_seqlen``."""
    if not isinstance(cu_seqlens, torch.Tensor) or cu_seqlens.dim() != 1 or cu_seqlens.numel() < 1:
        raise ValueError("cu_seqlens must be a 1-D tensor of n_docs + 1 offsets")
    if cu_seqlens.dtype != torch.int32:
        raise ValueError(f"cu_seqlens must be int32, got {cu_seqlens.dtype}")
    if cu_seqlens.device.type != "cpu":
        if max_seqlen is None:
            raise ValueError("a device cu_seqlens needs max_seqlen (deriving it would sync with the host)")
        return int(max_seqlen)
    if int(cu_seqlens[0]) != 0:
        raise ValueError(f"cu_seqlens must start at 0, got {int(cu_seqlens[0])}")
    if int(cu_seqlens[-1]) != T:
        raise ValueError(f"cu_seqlens must end at the token count {T}, got {int(cu_seqlens[-1])}")
    lens = cu_seqlens[1:] - cu_seqlens[:-1]
    if bool((lens < 0).any()):
        raise ValueError("cu_seqlens must be non-decreasing")
    longest = int(lens.max()) if lens.numel() else 0
    if max_seqlen is not None and int(max_seqlen) < longest:
        raise ValueError(f"max_seqlen {int(max_seqlen)} is shorter than the longest document ({longest})")
    return longest if max_seqlen is None else int(max_seqlen)


def _doc_spans(cu_seqlens, T):
    """Host ``(start, end)`` pairs of the non-empty documents (syncs once for a device tensor)."""
    cu = cu_seqlens.tolist()
    if cu[0] != 0 or cu[-1] != T or any(b < a for a, b in zip(cu[:-1], cu[1:])):
        raise ValueError("cu_seqlens must be non-decreasing offsets from 0 to the token count")
    return [(a, b) for a, b in zip(cu[:-1], cu[1:]) if b > a]


def _split_doc(qkv, s, e, hq, hkv, d):
    x = qkv[s:e].view(1, e - s, hq + 2 * hkv, d)
    return x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2), x[:, :, hq + hkv:].transpose(1, 2)


class _PackedVarlenCausalAttention(torch.autograd.Function):
    """Packed documents through one SDPA call per document (the portable path and the reference for the varlen kernel):
    in-place RoPE with per-token positions, packed ``dqkv`` in the backward, un-rotated in place."""

    @staticmethod
    def forward(ctx, qkv, spans, hq, hkv, d, rope, positions, backend, causal, window):
        T = qkv.shape[0]
        if rope is not None:
            rope_qk_inplace(qkv, hq, hkv, d, rope, positions, T, backward=False)
        out = qkv.new_empty(T, hq * d)
        graphs = []
        for s, e in spans:
            parts = _split_doc(qkv, s, e, hq, hkv, d)  # views taken outside grad mode, like _PackedCausalAttention
            with torch.enable_grad():
                qd, kd, vd = (t.detach().requires_grad_(True) for t in parts)
                o = _sdpa(qd, kd, vd, backend, causal=causal, window=window)
            out[s:e] = o.detach().transpose(1, 2).reshape(e - s, hq * d)
            graphs.append((s, e, qd, kd, vd, o))
        ctx.graphs = graphs
        ctx.meta = (hq, hkv, d, rope, positions)
        ctx.qkv_shape = qkv.shape
        return out

    @staticmethod
    def backward(ctx, dout):
        hq, hkv, d, rope, positions = ctx.meta
        graphs, ctx.graphs = ctx.graphs, None
        T = ctx.qkv_shape[0]
        dqkv = torch.zeros(ctx.qkv_shape, dtype=dout.dtype, device=dout.device)
        for s, e, qd, kd, vd, o in graphs:
            do = dout[s:e].view(1, e - s, hq, d).transpose(1, 2)
            dq, dk, dv = torch.autograd.grad(o, (qd, kd, vd), do)
            y = dqkv[s:e].view(1, e - s, hq + 2 * hkv, d)
            y[:, :, :hq].copy_(dq.transpose(1, 2))
            y[:, :, hq:hq + hkv].copy_(dk.transpose(1, 2))
            y[:, :, hq + hkv:].copy_(dv.transpose(1, 2))
        if rope is not None:
            rope_qk_inplace(dqkv, hq, hkv, d, rope, positions, T, backward=True)
        return dqkv, None, None, None, None, None, None, None, None, None


def varlen_attention_sdpa(qkv2d, cu_seqlens, hq, hkv, d, rope=None, positions=None, backend="auto", causal=True,
                          sliding_window=None):
    """Per-document SDPA over packed documents (any device / dtype / head dim); ``positions`` as in
    :func:`causal_attention` (defaults to :func:`document_positions`).  ``sliding_window`` needs ``causal``; a document
    longer than the window runs with a boolean band mask."""
    window = check_sliding_window(sliding_window)
    if window is not None and not causal:
        raise ValueError("a sliding window is defined only for causal attention")
    T = qkv2d.shape[0]
    if rope is not None and positions is None:
        positions = document_positions(cu_seqlens, T)
    if positions is not None:
        positions = positions.reshape(-1).to(device=qkv2d.device, dtype=torch.int32)
    spans = _doc_spans(cu_seqlens, T)
    if torch.is_grad_enabled() and qkv2d.requires_grad:
        return _PackedVarlenCausalAttention.apply(qkv2d, spans, hq, hkv, d, rope, positions, backend, causal, window)
    if rope is not None:
        rope_qk_inplace(qkv2d, hq, hkv, d, rope, positions, T, backward=False)
    out = qkv2d.new_empty(T, hq * d)
    for s, e in spans:
        o = _sdpa(*_split_doc(qkv2d, s, e, hq, hkv, d), backend, causal=causal, window=window)
        out[s:e] = o.transpose(1, 2).reshape(e - s, hq * d)
    return out


def _varlen_causal_attention(qkv2d, T, hq, hkv, d, rope, positions, backend, cu_seqlens, max_seqlen, window):
    max_seqlen = check_cu_seqlens(cu_seqlens, T, max_seqlen)
    if window is not None and window >= max_seqlen:
        window = None  # no document is longer than the window: exactly the unwindowed call
    if backend in ("native", "auto") and qkv2d.is_cuda:
        from deepspeed_b200.ops.kernels import attention_sm100
        if attention_sm100.supports_varlen(qkv2d, hq, hkv, d):
            cu = cu_seqlens.to(qkv2d.device, non_blocking=True)
            if rope is not None:
                positions = (document_positions(cu, T) if positions is None else positions.reshape(-1).to(
                    device=qkv2d.device, dtype=torch.int32))
            if torch.is_grad_enabled() and qkv2d.requires_grad:
                return attention_sm100.packed_varlen_attention(qkv2d, cu, max_seqlen, hq, hkv, d, rope, positions, window)
            if rope is not None:
                rope_qk_inplace(qkv2d, hq, hkv, d, rope, positions, T, backward=False)
            q, k, v = attention_sm100.split_packed(qkv2d, hq, hkv, d)
            return attention_sm100.fwd_varlen(q, k, v, cu, max_seqlen, hq, hkv, causal=True, need_lse=False,
                                              window=window, head_dim=d)[0]
    if backend == "native":
        raise RuntimeError("native varlen attention kernel requested but unsupported for this input (needs a CUDA bf16 "
                           "tensor, head dim 64 or 128, 16-byte aligned rows)")
    return varlen_attention_sdpa(qkv2d, cu_seqlens, hq, hkv, d, rope, positions, backend, sliding_window=window)


def causal_attention(qkv2d, B, S, hq, hkv, d, rope=None, positions=None, backend="auto", cu_seqlens=None, max_seqlen=None,
                     sliding_window=None):
    """``qkv2d [B*S, (hq + 2 hkv) * d]`` -> ``[B*S, hq*d]``.  With ``cu_seqlens`` (int32 ``[n_docs + 1]`` offsets into the
    ``B*S`` rows, see :func:`check_cu_seqlens`) attention is masked to each document and ``positions`` defaults to
    :func:`document_positions`; a device ``cu_seqlens`` needs ``max_seqlen``.  ``sliding_window``: see the module
    docstring; a value that is not an int >= 1 raises ``ValueError``."""
    backend = _ENV or backend or "auto"
    window = check_sliding_window(sliding_window)
    if cu_seqlens is not None:
        return _varlen_causal_attention(qkv2d, B * S, hq, hkv, d, rope, positions, backend, cu_seqlens, max_seqlen, window)
    if window is not None and window >= S:
        window = None  # every row sees its whole causal prefix: exactly the unwindowed call
    # `auto` takes the in-tree kernel for a window whenever it can: it skips the tiles outside the band, the fallback masks
    if backend == "native" or (backend == "auto" and qkv2d.is_cuda and
                               (window is not None or _native_wins(B, S, hq, hkv, d))):
        from deepspeed_b200.ops.kernels import attention_sm100
        if attention_sm100.supports(qkv2d, hq, hkv, d, S):
            if torch.is_grad_enabled() and qkv2d.requires_grad:
                return attention_sm100.packed_causal_attention(qkv2d, B, S, hq, hkv, d, rope, positions, window)
            if rope is not None:
                rope_qk_inplace(qkv2d, hq, hkv, d, rope, positions, S, backward=False)
            q, k, v = attention_sm100.split_packed(qkv2d, hq, hkv, d)
            return attention_sm100.fwd(q, k, v, B, S, hq, hkv, causal=True, need_lse=False, window=window,
                                       head_dim=d)[0]
        if backend == "native":
            raise RuntimeError("native attention kernel requested but unsupported for this shape (needs bf16, head dim 64 "
                               "or 128, sequence length a multiple of 128)")
    if not (torch.is_grad_enabled() and qkv2d.requires_grad):
        if rope is not None:
            rope_qk_inplace(qkv2d, hq, hkv, d, rope, positions, S, backward=False)
        x = qkv2d.view(B, S, hq + 2 * hkv, d)
        out = _sdpa(x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2),
                    x[:, :, hq + hkv:].transpose(1, 2), backend, window=window)
        return out.transpose(1, 2).reshape(B * S, hq * d)
    return _PackedCausalAttention.apply(qkv2d, B, S, hq, hkv, d, rope, positions, backend, window)
