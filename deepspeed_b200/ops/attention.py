"""Causal self-attention on a packed QKV buffer.

``causal_attention(qkv2d, B, S, hq, hkv, d, rope, positions)``: rotates Q and K **in place** inside the
packed projection output (one launch, ``transformer.cu:rope_kernel``), runs the attention core and
returns ``[B*S, hq*d]``.  The backward produces one packed ``dqkv`` buffer and un-rotates it in place.

Attention-core backends (``backend=`` or ``DSB200_ATTN``):
  * ``cudnn`` / ``flash`` / ``efficient`` / ``math`` -- ``torch.nn.functional.scaled_dot_product_attention``
    with that SDPA backend (library path; cuDNN has a Hopper FMHA);
  * ``flash_attn`` -- the flash-attn package;
  * ``native`` -- the framework's own sm_90a kernel (``csrc/cuda/attn_sm90.cu``) when built;
  * ``auto`` -- native if available, else cudnn -> flash -> efficient -> math priority order.
Role parity: the reference has no training attention kernel of its own for HF models (it relies on
PyTorch / flash-attn, ``sequence/fpdt_layer.py:235``); the BERT-era fused layer is ``ops/transformer``.
"""
import os

import torch
import torch.nn.functional as F

from deepspeed_b200.ops.kernels.transformer_ops import rope_qk_inplace

_ENV = os.environ.get("DSB200_ATTN", "").lower()


def _sdpa(q, k, v, backend, causal=True, scale=None):
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
    def forward(ctx, qkv, B, S, hq, hkv, d, rope, positions, backend):
        T = B * S
        if rope is not None:
            rope_qk_inplace(qkv, hq, hkv, d, rope, positions, S, backward=False)
        x = qkv.view(B, S, hq + 2 * hkv, d)
        q = x[:, :, :hq].transpose(1, 2)
        k = x[:, :, hq:hq + hkv].transpose(1, 2)
        v = x[:, :, hq + hkv:].transpose(1, 2)
        with torch.enable_grad():
            qd, kd, vd = (t.detach().requires_grad_(True) for t in (q, k, v))
            out = _sdpa(qd, kd, vd, backend)
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
        return dqkv, None, None, None, None, None, None, None, None


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


def causal_attention(qkv2d, B, S, hq, hkv, d, rope=None, positions=None, backend="auto"):
    backend = _ENV or backend or "auto"
    if backend == "native" or (backend == "auto" and qkv2d.is_cuda and _native_wins(B, S, hq, hkv, d)):
        from deepspeed_b200.ops.kernels import attention_sm100
        if attention_sm100.supports(qkv2d, hq, hkv, d, S):
            if torch.is_grad_enabled() and qkv2d.requires_grad:
                return attention_sm100.packed_causal_attention(qkv2d, B, S, hq, hkv, d, rope, positions)
            if rope is not None:
                rope_qk_inplace(qkv2d, hq, hkv, d, rope, positions, S, backward=False)
            q, k, v = attention_sm100.split_packed(qkv2d, hq, hkv)
            return attention_sm100.fwd(q, k, v, B, S, hq, hkv, causal=True, need_lse=False)[0]
        if backend == "native":
            raise RuntimeError("native attention kernel requested but unsupported for this shape (needs bf16, head dim 128, "
                               "sequence length a multiple of 128)")
    if not (torch.is_grad_enabled() and qkv2d.requires_grad):
        if rope is not None:
            rope_qk_inplace(qkv2d, hq, hkv, d, rope, positions, S, backward=False)
        x = qkv2d.view(B, S, hq + 2 * hkv, d)
        out = _sdpa(x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2),
                    x[:, :, hq + hkv:].transpose(1, 2), backend)
        return out.transpose(1, 2).reshape(B * S, hq * d)
    return _PackedCausalAttention.apply(qkv2d, B, S, hq, hkv, d, rope, positions, backend)
