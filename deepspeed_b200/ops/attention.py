"""Causal self-attention on a packed QKV buffer.

``causal_attention(qkv2d, B, S, hq, hkv, d, rope, positions)``: rotates Q and K **in place** inside the
packed projection output (one launch, ``transformer.cu:rope_kernel``), runs the attention core and
returns ``[B*S, hq*d]``.  The backward produces one packed ``dqkv`` buffer and un-rotates it in place.  One autograd
node (``_PackedQKVAttention``) owns the rotation for each of the four cores: the in-tree kernel, dense or varlen, and
SDPA, dense or one call per document.

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
QK-norm (``qk_norm=(w_q, w_k, eps)``, Qwen3): every query head is RMS-normalised with its own ``[d]`` weight ``w_q`` and
every key head with ``w_k`` before RoPE, in the same in-place pass (``transformer.cu:qk_norm_rope_kernel``, see
``transformer_ops.qk_norm_rope_inplace``); the autograd node takes the two weights as inputs and returns their gradients.
``qk_norm=None`` runs exactly the calls it ran without the argument.
Role parity: the reference has no training attention kernel of its own for HF models (it relies on
PyTorch / flash-attn, ``sequence/fpdt_layer.py:235``); the BERT-era fused layer is ``ops/transformer``.
"""
import numbers
import os

import torch
import torch.nn.functional as F

from deepspeed_b200.ops.kernels import attention_sm100
from deepspeed_b200.ops.kernels.transformer_ops import qk_norm_rope_bwd_inplace, qk_norm_rope_inplace, rope_qk_inplace

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


def _heads(x, hq, hkv):
    """``q, k, v [B, heads, S, d]`` views of ``x [B, S, hq + 2 hkv, d]``."""
    return x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2), x[:, :, hq + hkv:].transpose(1, 2)


def _sdpa_graph(qkv, need_grad, *args, **kw):
    """:func:`_sdpa` on the views ``qkv = (q, k, v)`` -> ``(out, graph)``.  With ``need_grad`` the call runs on detached
    leaves under grad mode and ``graph`` keeps the leaves and the output, so :func:`_sdpa_grad` can differentiate this call
    alone; without it ``graph`` is ``None``.  ``out`` is detached either way."""
    if not need_grad:
        return _sdpa(*qkv, *args, **kw), None
    with torch.enable_grad():
        leaves = tuple(t.detach().requires_grad_(True) for t in qkv)
        out = _sdpa(*leaves, *args, **kw)
    return out.detach(), (leaves, out)


def _sdpa_grad(graph, do, y, hq, hkv):
    """Backward of one :func:`_sdpa_graph` call for the output gradient ``do``, written into ``y``, a
    ``[B, S, hq + 2 hkv, d]`` view of the packed ``dqkv``."""
    leaves, out = graph
    for dst, g in zip(_heads(y, hq, hkv), torch.autograd.grad(out, leaves, do)):
        dst.copy_(g)


# The four attention cores.  Each is built per call and carries ``hq, hkv, d`` and ``seq_len`` (the rotation's position
# modulus when ``positions`` is None).  ``forward(qkv, need_grad) -> (out [T, hq*d], tensors to save)`` reads the rotated
# packed buffer; ``backward(dout, saved) -> dqkv`` returns the packed gradient before the un-rotation.


class _NativeDense:
    """The in-tree kernel on ``B`` sequences of ``S`` tokens."""

    def __init__(self, B, S, hq, hkv, d, window):
        self.B, self.seq_len, self.hq, self.hkv, self.d, self.window = B, S, hq, hkv, d, window

    def forward(self, qkv, need_grad):
        q, k, v = attention_sm100.split_packed(qkv, self.hq, self.hkv, self.d)
        o, lse = attention_sm100.fwd(q, k, v, self.B, self.seq_len, self.hq, self.hkv, causal=True, need_lse=need_grad,
                                     window=self.window, head_dim=self.d)
        return o, (qkv, o, lse)

    def backward(self, dout, saved):
        qkv, o, lse = saved
        B, S, hq, hkv, d = self.B, self.seq_len, self.hq, self.hkv, self.d
        dqkv = torch.empty_like(qkv)
        dq, dk, dv = attention_sm100.split_packed(dqkv, hq, hkv, d)
        attention_sm100.bwd(dout.reshape(B * S, hq * d), *attention_sm100.split_packed(qkv, hq, hkv, d), o, lse, B, S, hq,
                            hkv, causal=True, dq=dq, dk=dk, dv=dv, window=self.window, head_dim=d)
        return dqkv


class _NativeVarlen:
    """The in-tree varlen kernel on ``T`` packed rows: documents at the device offsets ``cu_seqlens``, none longer than
    ``max_seqlen``."""

    def __init__(self, cu_seqlens, max_seqlen, T, hq, hkv, d, window):
        self.cu_seqlens, self.max_seqlen, self.seq_len = cu_seqlens, max_seqlen, T
        self.hq, self.hkv, self.d, self.window = hq, hkv, d, window

    def forward(self, qkv, need_grad):
        q, k, v = attention_sm100.split_packed(qkv, self.hq, self.hkv, self.d)
        o, lse = attention_sm100.fwd_varlen(q, k, v, self.cu_seqlens, self.max_seqlen, self.hq, self.hkv, causal=True,
                                            need_lse=need_grad, window=self.window, head_dim=self.d)
        return o, (qkv, o, lse, self.cu_seqlens)

    def backward(self, dout, saved):
        qkv, o, lse, cu_seqlens = saved
        hq, hkv, d = self.hq, self.hkv, self.d
        dqkv = torch.empty_like(qkv)
        dq, dk, dv = attention_sm100.split_packed(dqkv, hq, hkv, d)
        attention_sm100.bwd_varlen(dout.reshape(qkv.shape[0], hq * d), *attention_sm100.split_packed(qkv, hq, hkv, d), o,
                                   lse, cu_seqlens, self.max_seqlen, hq, hkv, causal=True, dq=dq, dk=dk, dv=dv,
                                   window=self.window, head_dim=d)
        return dqkv


class _SdpaDense:
    """SDPA with ``backend`` on ``B`` sequences of ``S`` tokens."""

    def __init__(self, B, S, hq, hkv, d, backend, window):
        self.B, self.seq_len, self.hq, self.hkv, self.d, self.backend, self.window = B, S, hq, hkv, d, backend, window

    def forward(self, qkv, need_grad):
        B, S, hq, hkv, d = self.B, self.seq_len, self.hq, self.hkv, self.d
        self.shape = qkv.shape
        out, self.graph = _sdpa_graph(_heads(qkv.view(B, S, hq + 2 * hkv, d), hq, hkv), need_grad, self.backend,
                                      window=self.window)
        return out.transpose(1, 2).reshape(B * S, hq * d), ()

    def backward(self, dout, saved):
        B, S, hq, hkv, d = self.B, self.seq_len, self.hq, self.hkv, self.d
        graph, self.graph = self.graph, None
        dqkv = torch.empty(self.shape, dtype=dout.dtype, device=dout.device)
        _sdpa_grad(graph, dout.view(B, S, hq, d).transpose(1, 2), dqkv.view(B, S, hq + 2 * hkv, d), hq, hkv)
        return dqkv


class _SdpaDocs:
    """One SDPA call with ``backend`` per document of ``T`` packed rows (the portable path and the reference for the
    varlen kernel); ``spans`` are the host ``(start, end)`` rows of the non-empty documents."""

    def __init__(self, spans, T, hq, hkv, d, backend, causal, window):
        self.spans, self.seq_len, self.hq, self.hkv, self.d = spans, T, hq, hkv, d
        self.backend, self.causal, self.window = backend, causal, window

    def forward(self, qkv, need_grad):
        hq, hkv, d = self.hq, self.hkv, self.d
        self.shape = qkv.shape
        out = qkv.new_empty(self.seq_len, hq * d)
        self.graphs = []
        for s, e in self.spans:
            o, graph = _sdpa_graph(_heads(qkv[s:e].view(1, e - s, hq + 2 * hkv, d), hq, hkv), need_grad, self.backend,
                                   causal=self.causal, window=self.window)
            out[s:e] = o.transpose(1, 2).reshape(e - s, hq * d)
            self.graphs.append(graph)
        return out, ()

    def backward(self, dout, saved):
        hq, hkv, d = self.hq, self.hkv, self.d
        graphs, self.graphs = self.graphs, None
        dqkv = torch.zeros(self.shape, dtype=dout.dtype, device=dout.device)
        for (s, e), graph in zip(self.spans, graphs):
            _sdpa_grad(graph, dout[s:e].view(1, e - s, hq, d).transpose(1, 2), dqkv[s:e].view(1, e - s, hq + 2 * hkv, d),
                       hq, hkv)
        return dqkv


def _rotate(qkv, core, rope, positions, w_q, w_k, eps, need_raw):
    """QK-norm + RoPE (or RoPE alone, or nothing) in place on the Q and K heads of ``qkv``; returns the pre-norm heads
    for the backward when ``need_raw`` and QK-norm is on, else ``None``."""
    if w_q is not None:
        return qk_norm_rope_inplace(qkv, core.hq, core.hkv, core.d, rope, w_q, w_k, eps, positions, core.seq_len,
                                    need_raw=need_raw)
    if rope is not None:
        rope_qk_inplace(qkv, core.hq, core.hkv, core.d, rope, positions, core.seq_len, backward=False)
    return None


class _PackedQKVAttention(torch.autograd.Function):
    """Attention on the packed QKV projection output through ``core``: Q and K rotated in place, then the core.  The
    backward takes the packed ``dqkv`` from the core -- the layout the QKV projection's backward GEMMs consume -- and
    un-rotates it in place; with QK-norm it also returns the gradients of ``w_q`` and ``w_k``."""

    @staticmethod
    def forward(ctx, qkv, core, rope, positions, w_q, w_k, eps):
        raw = _rotate(qkv, core, rope, positions, w_q, w_k, eps, need_raw=True)
        out, saved = core.forward(qkv, need_grad=True)
        ctx.save_for_backward(*saved, *(() if w_q is None else (raw, w_q, w_k)))
        ctx.core, ctx.n_core, ctx.rope, ctx.positions, ctx.eps = core, len(saved), rope, positions, eps
        return out

    @staticmethod
    def backward(ctx, dout):
        core, rope, positions, eps = ctx.core, ctx.rope, ctx.positions, ctx.eps
        saved = ctx.saved_tensors
        dqkv = core.backward(dout, saved[:ctx.n_core])
        dw_q = dw_k = None
        if eps is not None:
            raw, w_q, w_k = saved[ctx.n_core:]
            dw_q, dw_k = qk_norm_rope_bwd_inplace(dqkv, raw, core.hq, core.hkv, core.d, rope, w_q, w_k, eps, positions,
                                                  core.seq_len)
        elif rope is not None:
            rope_qk_inplace(dqkv, core.hq, core.hkv, core.d, rope, positions, core.seq_len, backward=True)
        return dqkv, None, None, None, dw_q, dw_k, None


def _attend(core, qkv2d, rope, positions, qk_norm):
    """Rotate and attend through ``core``: with the autograd node when grad mode is on and ``qkv2d`` or a QK-norm weight
    needs a gradient, else keeping nothing for a backward."""
    w_q, w_k, eps = qk_norm or (None, None, None)
    if torch.is_grad_enabled() and (qkv2d.requires_grad or (w_q is not None and (w_q.requires_grad or w_k.requires_grad))):
        return _PackedQKVAttention.apply(qkv2d, core, rope, positions, w_q, w_k, eps)
    _rotate(qkv2d, core, rope, positions, w_q, w_k, eps, need_raw=False)
    return core.forward(qkv2d, need_grad=False)[0]


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


def varlen_attention_sdpa(qkv2d, cu_seqlens, hq, hkv, d, rope=None, positions=None, backend="auto", causal=True,
                          sliding_window=None, qk_norm=None):
    """Per-document SDPA over packed documents (any device / dtype / head dim); ``positions`` and ``qk_norm`` as in
    :func:`causal_attention` (``positions`` defaults to :func:`document_positions`).  ``sliding_window`` needs ``causal``;
    a document longer than the window runs with a boolean band mask."""
    window = check_sliding_window(sliding_window)
    if window is not None and not causal:
        raise ValueError("a sliding window is defined only for causal attention")
    T = qkv2d.shape[0]
    if rope is not None and positions is None:
        positions = document_positions(cu_seqlens, T)
    if positions is not None:
        positions = positions.reshape(-1).to(device=qkv2d.device, dtype=torch.int32)
    return _attend(_SdpaDocs(_doc_spans(cu_seqlens, T), T, hq, hkv, d, backend, causal, window), qkv2d, rope, positions,
                   qk_norm)


def _varlen_causal_attention(qkv2d, T, hq, hkv, d, rope, positions, backend, cu_seqlens, max_seqlen, window, qk_norm):
    max_seqlen = check_cu_seqlens(cu_seqlens, T, max_seqlen)
    if window is not None and window >= max_seqlen:
        window = None  # no document is longer than the window: exactly the unwindowed call
    if backend in ("native", "auto") and qkv2d.is_cuda and attention_sm100.supports_varlen(qkv2d, hq, hkv, d):
        cu = cu_seqlens.to(qkv2d.device, non_blocking=True)
        if rope is not None:
            positions = (document_positions(cu, T) if positions is None else positions.reshape(-1).to(
                device=qkv2d.device, dtype=torch.int32))
        return _attend(_NativeVarlen(cu, max_seqlen, T, hq, hkv, d, window), qkv2d, rope, positions, qk_norm)
    if backend == "native":
        raise RuntimeError("native varlen attention kernel requested but unsupported for this input (needs a CUDA bf16 "
                           "tensor, head dim 64 or 128, 16-byte aligned rows)")
    return varlen_attention_sdpa(qkv2d, cu_seqlens, hq, hkv, d, rope, positions, backend, sliding_window=window,
                                 qk_norm=qk_norm)


def causal_attention(qkv2d, B, S, hq, hkv, d, rope=None, positions=None, backend="auto", cu_seqlens=None, max_seqlen=None,
                     sliding_window=None, qk_norm=None):
    """``qkv2d [B*S, (hq + 2 hkv) * d]`` -> ``[B*S, hq*d]``.  With ``cu_seqlens`` (int32 ``[n_docs + 1]`` offsets into the
    ``B*S`` rows, see :func:`check_cu_seqlens`) attention is masked to each document and ``positions`` defaults to
    :func:`document_positions`; a device ``cu_seqlens`` needs ``max_seqlen``.  ``sliding_window``: see the module
    docstring; a value that is not an int >= 1 raises ``ValueError``.  ``qk_norm``: ``None`` or ``(w_q, w_k, eps)``, the
    per-head RMSNorm of Q and K before RoPE (module docstring)."""
    backend = _ENV or backend or "auto"
    window = check_sliding_window(sliding_window)
    if cu_seqlens is not None:
        return _varlen_causal_attention(qkv2d, B * S, hq, hkv, d, rope, positions, backend, cu_seqlens, max_seqlen, window,
                                        qk_norm)
    if window is not None and window >= S:
        window = None  # every row sees its whole causal prefix: exactly the unwindowed call
    # `auto` takes the in-tree kernel for a window whenever it can: it skips the tiles outside the band, the fallback masks
    native = backend == "native" or (backend == "auto" and qkv2d.is_cuda and
                                     (window is not None or _native_wins(B, S, hq, hkv, d)))
    if native and not attention_sm100.supports(qkv2d, hq, hkv, d, S):
        if backend == "native":
            raise RuntimeError("native attention kernel requested but unsupported for this shape (needs bf16, head dim 64 "
                               "or 128, sequence length a multiple of 128)")
        native = False
    core = _NativeDense(B, S, hq, hkv, d, window) if native else _SdpaDense(B, S, hq, hkv, d, backend, window)
    return _attend(core, qkv2d, rope, positions, qk_norm)
