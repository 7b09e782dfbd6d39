"""Python face of the ragged-batch inference kernels (``csrc/cuda/moe_ragged.cu``, ``attention.cu``).

``ragged_embed``, ``kv_rotary_append`` (RoPE + paged KV write), ``paged_attention`` (decode / chunked prefill
against the blocked cache), ``row_gather`` (last-token logits gather).  Every op has a host (torch) path with
identical semantics so the scheduler / state-manager logic is testable without a GPU.  Reference counterparts:
``inference/v2/kernels/ragged_ops/{embed,linear_blocked_kv_rotary,blocked_flash,logits_gather}`` (N9b).
"""
import ctypes
import math
import os

import torch

from deepspeed_b200.ops import native as N
from deepspeed_b200.ops.quantizer.quantizer import _fma32


_ws = {}


def _decode_ws(device, n_acc, n_ml):
    """Persistent fp32 workspace for split-KV partials (persistent so CUDA-graph replays see stable addresses)."""
    ent = _ws.get(device)
    if ent is None or ent[0].numel() < n_acc or ent[1].numel() < n_ml:
        ent = (torch.empty(max(n_acc, 1 << 22), dtype=torch.float32, device=device),
               torch.empty(max(n_ml, 1 << 16), dtype=torch.float32, device=device))
        _ws[device] = ent
    return ent


def _decode_eligible(dtype, hq, hkv, d, q_stride):
    return (dtype in (torch.bfloat16, torch.float16) and d in (64, 128, 256) and hq % hkv == 0
            and hq // hkv in (1, 2, 4, 8) and q_stride % 8 == 0)


def paged_attention_path(dtype, hq, hkv, d, q_stride):
    """The CUDA kernel ``paged_attention`` runs for this problem: ``"mma"`` (tensor-core split-KV decode, d 64 / 128),
    ``"cuda_core"`` (split-KV decode, d 256 or with ``DSB200_PAGED_DECODE_MMA=0``) or ``"generic"`` (one CTA per query
    head: fp32, other head dims or head ratios, or ``DSB200_PAGED_V1=1``)."""
    if not _decode_eligible(dtype, hq, hkv, d, q_stride) or os.environ.get("DSB200_PAGED_V1", "0") == "1":
        return "generic"
    mma = not os.environ.get("DSB200_PAGED_DECODE_MMA", "1").startswith("0")
    return "mma" if mma and d in (64, 128) else "cuda_core"


def decode_splits(tokens, hkv, max_ctx):
    """KV splits of the decode kernels: enough that (tokens x kv_heads x splits) covers the 132 SMs a few times over, at
    most 32, and at least 256 cache positions per split.  It depends only on static shapes (graph-capturable: no
    device->host read of the positions)."""
    # the tensor-core kernel runs 2 CTAs per SM: one full wave (296 CTAs) is enough, every extra KV split costs a
    # partial-result round trip (measured: 118 us at 296 vs 130 us at 592 for 64 seqs x 2048 ctx)
    target = int(os.environ.get("DSB200_PAGED_CTA_TARGET", "296" if os.environ.get("DSB200_PAGED_DECODE_MMA", "1") != "0" else "592"))
    nsplit = 1
    while tokens * hkv * nsplit < target and nsplit < 32 and max_ctx // (nsplit * 2) >= 256:
        nsplit *= 2
    return nsplit


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def ragged_embed(ids, wte, pos_ids=None, wpe=None, pos_offset=0):
    T, H = ids.numel(), wte.shape[1]
    if wte.is_cuda:
        out = torch.empty(T, H, dtype=wte.dtype, device=wte.device)
        rc = N.cuda().dsb_ragged_embed(_p(ids), _p(pos_ids if wpe is not None else None), _p(wte), _p(wpe), _p(out), T, H,
                                       int(pos_offset), N.dt(wte), N.stream())
        N.check(rc, "ragged_embed")
        return out
    out = wte[ids.long()]
    if wpe is not None:
        out = out + wpe[pos_ids.long() + pos_offset]
    return out


def row_gather(h, idx):
    if h.is_cuda:
        out = torch.empty(idx.numel(), h.shape[1], dtype=h.dtype, device=h.device)
        rc = N.cuda().dsb_row_gather(_p(h), _p(idx), _p(out), idx.numel(), h.shape[1], N.dt(h), N.stream())
        N.check(rc, "row_gather")
        return out
    return h[idx.long()]


def kv_rotary_append(qkv, cache, cos, sin, seq_of, pos_of, block_table, hq, hkv, d, rot_dim, block_size):
    """In place: rotate q,k of packed ``qkv`` [T,(hq+2hkv)*d]; append k,v to ``cache``
    [blocks, block_size, 2, hkv, d].  ``rot_dim`` 0 disables the rotation (learned-position models)."""
    T = qkv.shape[0]
    max_blocks = block_table.shape[1]
    if qkv.is_cuda:
        rc = N.cuda().dsb_kv_rotary_append(_p(qkv), _p(cache), _p(cos), _p(sin), _p(seq_of), _p(pos_of), _p(block_table), T,
                                           hq, hkv, d, int(rot_dim), block_size, max_blocks, N.dt(qkv), N.stream())
        N.check(rc, "kv_rotary_append")
        return qkv
    v = qkv.view(T, hq + 2 * hkv, d)
    if rot_dim:
        half = rot_dim // 2
        c = cos[pos_of.long()][:, None, :].to(torch.float32)
        s = sin[pos_of.long()][:, None, :].to(torch.float32)
        rot = v[:, :hq + hkv].float()
        a, b = rot[..., :half].clone(), rot[..., half:rot_dim].clone()
        # the kernel's fmaf(a, c, -(b * s)) and fmaf(b, c, a * s), rounded the same way
        v[:, :hq + hkv, :half] = _fma32(a, c, -(b * s)).to(qkv.dtype)
        v[:, :hq + hkv, half:rot_dim] = _fma32(b, c, a * s).to(qkv.dtype)
    blk = block_table[seq_of.long(), (pos_of // block_size).long()].long()
    slot = (pos_of % block_size).long()
    cache[blk, slot] = v[:, hq:].reshape(T, 2, hkv, d)
    return qkv


def paged_attention(qkv, cache, seq_of, pos_of, block_table, hq, hkv, d, block_size, scale=None):
    """out [T, hq*d]: token t attends to cached keys [0, pos_of[t]] of sequence seq_of[t]."""
    T = qkv.shape[0]
    scale = scale if scale is not None else 1.0 / math.sqrt(d)
    max_blocks = block_table.shape[1]
    if qkv.is_cuda:
        out = torch.empty(T, hq * d, dtype=qkv.dtype, device=qkv.device)
        if paged_attention_path(qkv.dtype, hq, hkv, d, qkv.shape[1]) != "generic":
            nsplit = decode_splits(T, hkv, max_blocks * block_size)
            ws_acc, ws_ml = _decode_ws(qkv.device, T * hq * nsplit * d, T * hq * nsplit * 2) if nsplit > 1 else (None, None)
            rc = N.cuda().dsb_paged_decode(_p(qkv), _p(cache), _p(out), _p(ws_acc), _p(ws_ml), _p(seq_of), _p(pos_of),
                                           _p(block_table), T, hq, hkv, d, qkv.shape[1], block_size, max_blocks,
                                           ctypes.c_float(scale), nsplit, N.dt(qkv), N.stream())
            if rc == 0:
                return out
            if rc != -3:
                N.check(rc, "paged_decode")
        rc = N.cuda().dsb_paged_attention(_p(qkv), _p(cache), _p(out), _p(seq_of), _p(pos_of), _p(block_table), T, hq, hkv, d,
                                          qkv.shape[1], block_size, max_blocks, ctypes.c_float(scale), N.dt(qkv),
                                          N.stream())
        N.check(rc, "paged_attention")
        return out
    out = torch.empty(T, hq, d, dtype=torch.float32)
    q = qkv.view(T, hq + 2 * hkv, d)[:, :hq].float()
    rep = hq // hkv
    for t in range(T):
        n = int(pos_of[t]) + 1
        s = int(seq_of[t])
        nb = (n + block_size - 1) // block_size
        kv = cache[block_table[s, :nb].long()].reshape(nb * block_size, 2, hkv, d)[:n].float()
        k = kv[:, 0].repeat_interleave(rep, dim=1)  # [n, hq, d]
        v = kv[:, 1].repeat_interleave(rep, dim=1)
        att = torch.einsum("hd,nhd->hn", q[t], k) * scale
        out[t] = torch.einsum("hn,nhd->hd", att.softmax(-1), v)
    return out.reshape(T, hq * d).to(qkv.dtype)
