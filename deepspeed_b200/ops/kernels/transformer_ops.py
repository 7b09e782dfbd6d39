"""Autograd-aware python face of ``csrc/cuda/transformer.cu``.

``rms_norm`` / ``layer_norm`` / ``rope`` / ``gated_act`` (SwiGLU...) / ``softmax_cross_entropy`` /
``bias_act``.  CUDA tensors go to the sm_90a kernels (hard error if the native library is missing);
host tensors use an equivalent fp32 torch implementation so models run unchanged in the CPU tier.
Reference counterparts: ``ops/transformer/inference/op_binding/*`` (N8 wrappers) and the training
layer's norm / gelu ops (N7).
"""
import ctypes
from typing import Optional

import torch
import torch.nn.functional as F

from deepspeed_b200.ops import native as N

ACT_SILU, ACT_GELU_TANH, ACT_RELU, ACT_GELU = 0, 1, 2, 3
_ACT_NAMES = {"silu": 0, "swiglu": 0, "gelu_tanh": 1, "geglu": 1, "gelu_new": 1, "relu": 2, "reglu": 2, "gelu": 3}


def act_code(name) -> int:
    if isinstance(name, int):
        return name
    return _ACT_NAMES[name.lower()]


def _null():
    return ctypes.c_void_p(0)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else _null()


# ---------------------------------------------------------------------------------------------------
# norms
# ---------------------------------------------------------------------------------------------------
def _norm_fwd_native(x2, residual2, w, b, eps, kind):
    rows, hidden = x2.shape
    y = torch.empty_like(x2)
    res_out = torch.empty_like(x2) if residual2 is not None else None
    rstd = torch.empty(rows, dtype=torch.float32, device=x2.device)
    mean = torch.empty(rows, dtype=torch.float32, device=x2.device) if kind == 1 else None
    rc = N.cuda().dsb_norm_fwd(_p(x2), _p(residual2), _p(w), _p(b), _p(y), _p(res_out), _p(mean), _p(rstd), rows,
                               hidden, N.c_f(eps), kind, N.dt(x2), N.stream())
    N.check(rc, "norm_fwd")
    return y, res_out, mean, rstd


def _norm_bwd_native(dy2, x2, w, mean, rstd, dres2, kind, need_db):
    rows, hidden = x2.shape
    lib = N.cuda()
    grid = lib.dsb_norm_bwd_grid(rows)
    dx = torch.empty_like(x2)
    dw_part = torch.empty(grid, hidden, dtype=torch.float32, device=x2.device)
    db_part = torch.empty(grid, hidden, dtype=torch.float32, device=x2.device) if (kind == 1 and need_db) else None
    dw = torch.empty(hidden, dtype=w.dtype, device=x2.device)
    db = torch.empty(hidden, dtype=w.dtype, device=x2.device) if db_part is not None else None
    rc = lib.dsb_norm_bwd(_p(dy2), _p(x2), _p(w), _p(mean), _p(rstd), _p(dres2), _p(dx), _p(dw_part), _p(db_part),
                          _p(dw), _p(db), rows, hidden, kind, N.dt(x2), N.dt(w), 0, N.stream())
    N.check(rc, "norm_bwd")
    return dx, dw, db


def norm_bwd_path(rows, hidden, kind, dtype, aligned=True) -> str:
    """``"bulk"`` or ``"register"``: the kernel the CUDA norm backward runs for this problem (``kind`` 0 RMSNorm,
    1 LayerNorm; ``aligned``: dy, x, dres and dx start on 16-byte boundaries)."""
    return "bulk" if N.cuda().dsb_norm_bwd_path(rows, hidden, kind, N.dt(dtype), int(aligned)) == 1 else "register"


class _NormFn(torch.autograd.Function):
    """y = norm(x (+ residual)); returns (y, x+residual) when a residual is given."""

    @staticmethod
    def forward(ctx, x, residual, w, b, eps, kind):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1]).contiguous()
        r2 = residual.reshape(-1, shape[-1]).contiguous() if residual is not None else None
        if x.is_cuda:
            y, res_out, mean, rstd = _norm_fwd_native(x2, r2, w, b, eps, kind)
        else:
            xin = x2.float() + (r2.float() if r2 is not None else 0)
            res_out = xin.to(x.dtype) if r2 is not None else None
            xin = res_out.float() if res_out is not None else xin
            if kind == 1:
                mean = xin.mean(-1)
                var = xin.var(-1, unbiased=False)
                rstd = torch.rsqrt(var + eps)
                y = ((xin - mean[:, None]) * rstd[:, None] * w.float() + (b.float() if b is not None else 0)).to(x.dtype)
            else:
                mean = None
                rstd = torch.rsqrt(xin.pow(2).mean(-1) + eps)
                y = (xin * rstd[:, None] * w.float()).to(x.dtype)
        ctx.kind, ctx.has_res, ctx.has_b, ctx.shape = kind, residual is not None, b is not None, shape
        ctx.save_for_backward(res_out if res_out is not None else x2, w, mean, rstd)
        if residual is not None:
            return y.view(shape), res_out.view(shape)
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy, dres=None):
        xin, w, mean, rstd = ctx.saved_tensors
        hidden = ctx.shape[-1]
        dy2 = dy.reshape(-1, hidden).contiguous()
        dres2 = dres.reshape(-1, hidden).contiguous() if (ctx.has_res and dres is not None) else None
        if dy.is_cuda:
            dx, dw, db = _norm_bwd_native(dy2, xin, w, mean, rstd, dres2, ctx.kind, ctx.has_b)
        else:
            xf, df, wf = xin.float(), dy2.float(), w.float()
            mu = mean[:, None] if ctx.kind == 1 else 0.0
            xhat = (xf - mu) * rstd[:, None]
            g = df * wf
            m2 = (g * xhat).mean(-1, keepdim=True)
            m1 = g.mean(-1, keepdim=True) if ctx.kind == 1 else 0.0
            dx = rstd[:, None] * (g - m1 - xhat * m2)
            if dres2 is not None:
                dx = dx + dres2.float()
            dx = dx.to(dy.dtype)
            dw = (df * xhat).sum(0).to(w.dtype)
            db = df.sum(0).to(w.dtype) if (ctx.kind == 1 and ctx.has_b) else None
        dx = dx.view(ctx.shape)
        return dx, (dx if ctx.has_res else None), dw, db, None, None


def rms_norm(x, weight, eps=1e-6, residual=None):
    """RMSNorm.  With ``residual`` returns ``(norm(x + residual), x + residual)`` in one pass."""
    return _NormFn.apply(x, residual, weight, None, eps, 0)


def layer_norm(x, weight, bias=None, eps=1e-5, residual=None):
    return _NormFn.apply(x, residual, weight, bias, eps, 1)


# ---------------------------------------------------------------------------------------------------
# rotary embedding
# ---------------------------------------------------------------------------------------------------
class RotaryTable:
    """Precomputed fp32 cos/sin tables ``[max_pos, rot_dim/2]`` (no per-element powf/sincos at run
    time, unlike the reference kernel ``apply_rotary_pos_emb.cu:26``)."""

    def __init__(self, rot_dim, max_pos, base=10000.0, device="cpu", scaling=None):
        inv = 1.0 / (base**(torch.arange(0, rot_dim, 2, dtype=torch.float64) / rot_dim))
        if scaling is not None and scaling.get("rope_type", scaling.get("type")) == "llama3":
            inv = _llama3_scale(inv, scaling)
        t = torch.arange(max_pos, dtype=torch.float64)
        if scaling is not None and scaling.get("rope_type", scaling.get("type")) == "linear":
            t = t / scaling["factor"]
        f = torch.outer(t, inv)
        self.cos = f.cos().float().contiguous().to(device)
        self.sin = f.sin().float().contiguous().to(device)
        self.rot_dim = rot_dim
        self.max_pos = max_pos

    def to(self, device):
        self.cos, self.sin = self.cos.to(device), self.sin.to(device)
        return self


def _llama3_scale(inv_freq, sc):
    import math
    factor, lo, hi = sc["factor"], sc.get("low_freq_factor", 1.0), sc.get("high_freq_factor", 4.0)
    old = sc.get("original_max_position_embeddings", 8192)
    wavelen = 2 * math.pi / inv_freq
    smooth = ((old / wavelen) - lo) / (hi - lo)
    out = torch.where(wavelen > old / lo, inv_freq / factor, inv_freq)
    mid = (wavelen <= old / lo) & (wavelen >= old / hi)
    return torch.where(mid, (1 - smooth) * inv_freq / factor + smooth * inv_freq, out)


def _rope_apply(x, table: RotaryTable, positions, seq_len, backward):
    """In place on ``x`` viewed as [tokens, heads, head_dim] with arbitrary token stride."""
    tokens, heads, hd = x.shape
    if x.is_cuda:
        assert x.stride(2) == 1 and x.stride(1) == hd
        rc = N.cuda().dsb_rope(_p(x), _p(table.cos), _p(table.sin), _p(positions), N.c_i64(tokens), heads, hd,
                               table.rot_dim, N.c_i64(x.stride(0)), seq_len, int(backward), N.dt(x), N.stream())
        N.check(rc, "rope")
        return x
    half = table.rot_dim // 2
    pos = positions.long() if positions is not None else (torch.arange(tokens, device=x.device) % seq_len)
    c = table.cos[pos][:, None, :]
    s = table.sin[pos][:, None, :] * (-1.0 if backward else 1.0)
    a, b = x[..., :half].float(), x[..., half:2 * half].float()
    o1, o2 = (a * c - b * s).to(x.dtype), (b * c + a * s).to(x.dtype)  # both before either store (a/b may alias x)
    x[..., :half] = o1
    x[..., half:2 * half] = o2
    return x


class _RopeFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, table, positions, seq_len):
        ctx.table, ctx.seq_len = table, seq_len
        ctx.save_for_backward(positions) if positions is not None else None
        ctx.has_pos = positions is not None
        ctx.mark_dirty(x)
        _rope_apply(x, table, positions, seq_len, False)
        return x

    @staticmethod
    def backward(ctx, dy):
        pos = ctx.saved_tensors[0] if ctx.has_pos else None
        dy = dy.contiguous() if not _rope_ok(dy) else dy
        dx = dy.clone() if not dy.is_contiguous() else dy.clone()
        _rope_apply(dx, ctx.table, pos, ctx.seq_len, True)
        return dx, None, None, None


def _rope_ok(t):
    return t.stride(-1) == 1 and t.stride(-2) == t.shape[-1]


def rope_(x, table: RotaryTable, positions=None, seq_len=None):
    """Apply rotary embedding **in place** to ``x`` of shape [tokens, heads, head_dim] (a strided view
    into a packed QKV buffer is fine).  Differentiable."""
    return _RopeFn.apply(x, table, positions, seq_len or x.shape[0])


def rope_qk_inplace(qkv, n_q, n_kv, head_dim, table, positions=None, seq_len=None, backward=False):
    """Rotate the Q and K heads of a packed ``[tokens, (n_q + 2 n_kv) * head_dim]`` buffer with ONE
    launch (Q and K heads are contiguous in the packed layout).  Not autograd-tracked: used inside
    fused attention functions that call it again with ``backward=True``."""
    tokens = qkv.shape[0]
    view = qkv.as_strided((tokens, n_q + n_kv, head_dim), (qkv.stride(0), head_dim, 1))
    return _rope_apply(view, table, positions, seq_len or tokens, backward)


# ---------------------------------------------------------------------------------------------------
# QK-norm + rotary embedding (Qwen3 attention)
# ---------------------------------------------------------------------------------------------------
def _qk_norm_native(qkv, head_dim, table):
    """Whether ``transformer.cu``'s fused QK-norm kernels take this buffer: CUDA bf16 / fp16 / fp32, head dim 64 or 128,
    a full rotary table, unit column stride and 16-byte aligned rows."""
    per = 4 if qkv.dtype == torch.float32 else 8
    return (qkv.is_cuda and qkv.dtype in (torch.bfloat16, torch.float16, torch.float32) and head_dim in (64, 128)
            and table is not None and table.rot_dim == head_dim and qkv.stride(-1) == 1 and qkv.stride(0) % per == 0
            and qkv.data_ptr() % 16 == 0)


def _qk_heads(qkv, n_q, n_kv, head_dim):
    return qkv.as_strided((qkv.shape[0], n_q + n_kv, head_dim), (qkv.stride(0), head_dim, 1))


def _qk_weights(w_q, w_k, n_q, n_kv):
    """fp32 ``[n_q + n_kv, head_dim]``: ``w_q`` for every query head, then ``w_k`` for every key head."""
    return torch.cat([w_q.float().expand(n_q, -1), w_k.float().expand(n_kv, -1)])


def _rotate_f32(x, table, positions, seq_len, sign):
    """Rotate-half RoPE (``sign`` -1: the transpose) of fp32 ``x [tokens, heads, head_dim]``, out of place; the dims past
    ``table.rot_dim`` pass through."""
    if table is None:
        return x
    half = table.rot_dim // 2
    pos = positions.long() if positions is not None else torch.arange(x.shape[0], device=x.device) % seq_len
    c = table.cos.to(x.device)[pos][:, None, :]
    s = table.sin.to(x.device)[pos][:, None, :] * sign
    a, b = x[..., :half], x[..., half:2 * half]
    return torch.cat([a * c - b * s, b * c + a * s, x[..., 2 * half:]], dim=-1)


def qk_norm_rope_inplace(qkv, n_q, n_kv, head_dim, table, w_q, w_k, eps, positions=None, seq_len=None, need_raw=True):
    """Qwen3's QK-norm followed by RoPE, **in place** on the Q and K heads of a packed
    ``[tokens, (n_q + 2 n_kv) * head_dim]`` buffer (any row stride): every query head becomes
    ``rope(w_q * q * rsqrt(mean(q^2) + eps))`` and every key head the same with ``w_k``; V is untouched.  ``positions`` /
    ``seq_len`` as in :func:`rope_qk_inplace`; ``table=None`` normalises without rotating.

    All arithmetic is fp32 and each result is rounded to the buffer's dtype once.  (HF's ``Qwen3RMSNorm`` rounds the
    normalised value to the input dtype before the weight multiply and RoPE rounds again, so a bf16 HF model differs
    from this in the last bits; in fp32 the two agree.)

    Returns the pre-norm Q|K heads ``[tokens, (n_q + n_kv) * head_dim]`` (contiguous, the buffer's dtype), which
    :func:`qk_norm_rope_bwd_inplace` takes, or ``None`` with ``need_raw=False`` (no backward follows).  Not
    autograd-tracked.  CUDA bf16 / fp16 / fp32 buffers with head dim 64 or
    128 and a full rotary table run one fused kernel; every other case (another head dim, a partial rotary table, a CPU
    tensor) an fp32 torch composition with the same semantics."""
    tokens = qkv.shape[0]
    seq_len = seq_len or tokens
    heads = _qk_heads(qkv, n_q, n_kv, head_dim)
    if _qk_norm_native(qkv, head_dim, table):
        raw = torch.empty(tokens, (n_q + n_kv) * head_dim, dtype=qkv.dtype, device=qkv.device) if need_raw else None
        w_q, w_k = w_q.to(qkv.dtype).contiguous(), w_k.to(qkv.dtype).contiguous()
        rc = N.cuda().dsb_qk_norm_rope(_p(qkv), _p(raw), _p(table.cos), _p(table.sin), _p(positions), _p(w_q), _p(w_k),
                                       N.c_i64(tokens), n_q, n_kv, head_dim, N.c_i64(qkv.stride(0)), seq_len,
                                       N.c_f(eps), N.dt(qkv), N.stream())
        N.check(rc, "qk_norm_rope")
        return raw
    return _qk_norm_rope_torch(heads, n_q, table, w_q, w_k, eps, positions, seq_len, need_raw)


def _qk_norm_rope_torch(heads, n_q, table, w_q, w_k, eps, positions, seq_len, need_raw=True):
    """The fp32 torch composition of :func:`qk_norm_rope_inplace`, on its ``[tokens, n_q + n_kv, head_dim]`` view."""
    tokens, n, head_dim = heads.shape
    raw = heads.reshape(tokens, n * head_dim).clone() if need_raw else None
    x = heads.float()
    y = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * _qk_weights(w_q, w_k, n_q, n - n_q)
    heads.copy_(_rotate_f32(y, table, positions, seq_len, 1.0).to(heads.dtype))
    return raw


def qk_norm_rope_bwd_inplace(dqkv, raw, n_q, n_kv, head_dim, table, w_q, w_k, eps, positions=None, seq_len=None):
    """Backward of :func:`qk_norm_rope_inplace`, **in place** on the dQ and dK heads of the packed gradient ``dqkv`` (same
    layout as the forward's buffer; dV untouched), given the ``raw`` pre-norm heads the forward returned.  Returns
    ``(dw_q, dw_k)`` in the weights' dtypes: fp32 sums over tokens and over the heads of each kind, in a fixed order (the
    CUDA kernel reduces per-CTA partials with the column-sum kernel), so they are bit-reproducible from run to run."""
    tokens = dqkv.shape[0]
    seq_len = seq_len or tokens
    heads = _qk_heads(dqkv, n_q, n_kv, head_dim)
    if _qk_norm_native(dqkv, head_dim, table):
        assert raw.is_contiguous() and raw.dtype == dqkv.dtype and raw.shape == (tokens, (n_q + n_kv) * head_dim)
        lib = N.cuda()
        grid = lib.dsb_qk_norm_rope_bwd_grid(N.c_i64(tokens), n_q + n_kv, head_dim, N.dt(dqkv))
        dw_part = torch.empty(grid, 2 * head_dim, dtype=torch.float32, device=dqkv.device)
        dw = torch.empty(2 * head_dim, dtype=w_q.dtype, device=dqkv.device)
        wq, wk = w_q.to(dqkv.dtype).contiguous(), w_k.to(dqkv.dtype).contiguous()
        rc = lib.dsb_qk_norm_rope_bwd(_p(dqkv), _p(raw), _p(table.cos), _p(table.sin), _p(positions), _p(wq), _p(wk),
                                      _p(dw_part), _p(dw), N.c_i64(tokens), n_q, n_kv, head_dim,
                                      N.c_i64(dqkv.stride(0)), seq_len, N.c_f(eps), N.dt(dqkv), N.dt(w_q), N.stream())
        N.check(rc, "qk_norm_rope_bwd")
        return dw[:head_dim].to(w_q.dtype), dw[head_dim:].to(w_k.dtype)
    return _qk_norm_rope_bwd_torch(heads, raw, n_q, table, w_q, w_k, eps, positions, seq_len)


def _qk_norm_rope_bwd_torch(heads, raw, n_q, table, w_q, w_k, eps, positions, seq_len):
    """The fp32 torch composition of :func:`qk_norm_rope_bwd_inplace`, on its ``[tokens, n_q + n_kv, head_dim]`` view."""
    tokens, n, head_dim = heads.shape
    r = _rotate_f32(heads.float(), table, positions, seq_len, -1.0)
    x = raw.view(tokens, n, head_dim).float()
    rstd = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    xhat = x * rstd
    g = r * _qk_weights(w_q, w_k, n_q, n - n_q)
    dw = r * xhat  # before the store below: without a table r is a view of the fp32 buffer
    heads.copy_((rstd * (g - xhat * (g * xhat).mean(-1, keepdim=True))).to(heads.dtype))
    return dw[:, :n_q].sum((0, 1)).to(w_q.dtype), dw[:, n_q:].sum((0, 1)).to(w_k.dtype)


# ---------------------------------------------------------------------------------------------------
# embedding backward
# ---------------------------------------------------------------------------------------------------
def embedding_bwd_(dy, ids, out):
    """``out[v] += sum of dy[t] over the tokens t with ids[t] == v``, **in place** on ``out [V, H]``; returns ``out``.
    ``dy`` is ``[..., H]`` with one row per id.  Deterministic: each id's rows are summed in fp32 in token order, added to
    the out row and rounded to ``out``'s dtype once.  Rows whose id does not occur are not read or written, so ``out``
    may already hold another contribution (a tied LM head's dW).

    CUDA bf16 / fp16 / fp32 operands with ``H % 8 == 0`` and 16-byte aligned buffers run ``transformer.cu``'s
    ``embedding_bwd_kernel`` (ids sorted on the device, no host sync); anything else runs :func:`_embedding_bwd_torch`."""
    H = out.shape[-1]
    dy2 = dy.reshape(-1, H)
    ids1 = ids.reshape(-1)
    floats = (torch.bfloat16, torch.float16, torch.float32)
    if dy2.is_cuda and out.is_cuda and out.is_contiguous() and dy2.dtype in floats and out.dtype in floats:
        dy2 = dy2.contiguous()
        sid, order = torch.sort(ids1.long(), stable=True)
        lib = N.cuda()
        part = torch.empty(lib.dsb_embedding_bwd_part_rows(N.c_i64(ids1.numel())), H, dtype=torch.float32,
                           device=out.device)
        rc = lib.dsb_embedding_bwd(_p(dy2), _p(sid), _p(order), _p(part), _p(out), N.c_i64(ids1.numel()), H, N.dt(dy2),
                                   N.dt(out), N.stream())
        if rc != -2:
            N.check(rc, "embedding_bwd")
            return out
    return _embedding_bwd_torch(dy2, ids1, out)


def _embedding_bwd_torch(dy2, ids1, out):
    """The torch form of :func:`embedding_bwd_` with the same semantics: an fp32 ``index_add_`` over the rows in sorted
    (stable, so token) order, one rounding per touched row."""
    sid, order = torch.sort(ids1.long(), stable=True)
    uniq, seg = torch.unique_consecutive(sid, return_inverse=True)
    acc = torch.zeros(uniq.numel(), out.shape[-1], dtype=torch.float32, device=out.device)
    acc.index_add_(0, seg.to(out.device), dy2[order].float().to(out.device))
    uniq = uniq.to(out.device)
    out[uniq] = (out[uniq].float() + acc).to(out.dtype)
    return out


# ---------------------------------------------------------------------------------------------------
# gated activation (SwiGLU & friends)
# ---------------------------------------------------------------------------------------------------
def gated_act_fwd_raw(gu, act=ACT_SILU, out=None):
    """``act(gate) * up`` of a contiguous packed ``[T, 2I]`` tensor (into the contiguous ``out [T, I]`` when given), no
    autograd."""
    if isinstance(act, str):
        act = act_code(act)
    inter = gu.shape[-1] // 2
    if gu.is_cuda:
        if out is None:
            out = torch.empty(gu.shape[0], inter, dtype=gu.dtype, device=gu.device)
        rc = N.cuda().dsb_gated_act_fwd(_p(gu), _p(out), N.c_i64(gu.shape[0]), inter, act, N.dt(gu), N.stream())
        N.check(rc, "gated_act_fwd")
        return out
    g, u = gu[:, :inter].float(), gu[:, inter:].float()
    y = (_act_torch(g, act) * u).to(gu.dtype)
    return y if out is None else out.copy_(y)


def gated_act_bwd(dout, gu, act=ACT_SILU, act_out=None):
    """Gradient of :func:`gated_act` w.r.t. the packed ``[T, 2I]`` input: ``[d * up * act'(gate) | d * act(gate)]``.
    ``act_out`` (contiguous ``[T, I]``, optional) also receives the forward output ``act(gate) * up`` from the same pass,
    bit-identical to :func:`gated_act_fwd_raw` of ``gu``: a caller need not keep the forward's output for backward."""
    if isinstance(act, str):
        act = act_code(act)
    inter = gu.shape[-1] // 2
    d2 = dout.reshape(-1, inter)
    if not d2.is_contiguous():
        d2 = d2.contiguous()
    if gu.is_cuda:
        dgu = torch.empty_like(gu)
        if act_out is not None:
            assert act_out.is_contiguous() and act_out.shape == (gu.shape[0], inter) and act_out.dtype == gu.dtype
        rc = N.cuda().dsb_gated_act_bwd(_p(d2), _p(gu), _p(dgu), _p(act_out), N.c_i64(gu.shape[0]), inter, act, N.dt(gu),
                                        N.stream())
        N.check(rc, "gated_act_bwd")
        return dgu
    g = gu[:, :inter].float().requires_grad_(True)
    u = gu[:, inter:].float()
    with torch.enable_grad():
        a = _act_torch(g, act)
        (da, ) = torch.autograd.grad(a, g, torch.ones_like(a))
    a = a.detach()
    if act_out is not None:
        act_out.copy_((a * u).to(gu.dtype))
    return torch.cat([d2.float() * u * da, d2.float() * a], dim=-1).to(gu.dtype)


class _GatedActFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, gate_up, act):
        inter = gate_up.shape[-1] // 2
        gu = gate_up.reshape(-1, 2 * inter)
        if not gu.is_contiguous():
            gu = gu.contiguous()
        out = gated_act_fwd_raw(gu, act)
        ctx.act, ctx.inter, ctx.shape = act, inter, gate_up.shape
        ctx.save_for_backward(gu)
        return out.view(*gate_up.shape[:-1], inter)

    @staticmethod
    def backward(ctx, dout):
        (gu, ) = ctx.saved_tensors
        return gated_act_bwd(dout, gu, ctx.act).view(ctx.shape), None


def _act_torch(g, act):
    if act == ACT_SILU:
        return F.silu(g)
    if act == ACT_GELU_TANH:
        return F.gelu(g, approximate="tanh")
    if act == ACT_RELU:
        return F.relu(g)
    return F.gelu(g)


def gated_act(gate_up, act="silu"):
    """``act(gate) * up`` for a packed ``[..., 2*I]`` tensor (gate first)."""
    return _GatedActFn.apply(gate_up, act_code(act))


swiglu = gated_act


# ---------------------------------------------------------------------------------------------------
# bias + activation (+ residual)
# ---------------------------------------------------------------------------------------------------
class _BiasActFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, bias, residual, act):
        cols = x.shape[-1]
        x2 = x.reshape(-1, cols).contiguous()
        r2 = residual.reshape(-1, cols).contiguous() if residual is not None else None
        if x2.is_cuda:
            y = torch.empty_like(x2)
            rc = N.cuda().dsb_bias_act(_p(x2), _p(bias), _p(r2), _p(y), N.c_i64(x2.shape[0]), cols, act, N.dt(x2),
                                       N.stream())
            N.check(rc, "bias_act")
        else:
            f = x2.float() + (bias.float() if bias is not None else 0)
            if act >= 0:
                f = _act_torch(f, act)
            if r2 is not None:
                f = f + r2.float()
            y = f.to(x.dtype)
        ctx.act, ctx.has_bias, ctx.has_res, ctx.shape = act, bias is not None, residual is not None, x.shape
        ctx.save_for_backward(x2, bias)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, bias = ctx.saved_tensors
        cols = ctx.shape[-1]
        d2 = dy.reshape(-1, cols).contiguous()
        if ctx.act < 0:
            dx = d2
        elif d2.is_cuda:
            dx = torch.empty_like(d2)
            rc = N.cuda().dsb_bias_act_bwd(_p(d2), _p(x2), _p(bias), _p(dx), N.c_i64(d2.shape[0]), cols, ctx.act,
                                           N.dt(d2), N.stream())
            N.check(rc, "bias_act_bwd")
        else:
            f = (x2.float() + (bias.float() if bias is not None else 0)).requires_grad_(True)
            with torch.enable_grad():
                a = _act_torch(f, ctx.act)
                (da, ) = torch.autograd.grad(a, f, torch.ones_like(a))
            dx = (d2.float() * da).to(dy.dtype)
        db = dx.float().sum(0).to(bias.dtype) if ctx.has_bias else None
        return dx.view(ctx.shape), db, (dy if ctx.has_res else None), None


def bias_act(x, bias=None, act: Optional[str] = "gelu", residual=None):
    return _BiasActFn.apply(x, bias, residual, -1 if act is None else act_code(act))


def bias_gelu(x, bias):
    return bias_act(x, bias, "gelu")


def bias_residual(x, bias, residual):
    return bias_act(x, bias, None, residual)


# ---------------------------------------------------------------------------------------------------
# softmax cross entropy
# ---------------------------------------------------------------------------------------------------
def xent_valid(labels, vocab, ignore_index=-100):
    """Rows that contribute to the loss: the label is in ``[0, vocab)`` and is not ``ignore_index``.  Every other row
    (including a label out of range) is ignored like ``ignore_index``: zero loss, zero gradient, not counted in a mean."""
    return (labels != ignore_index) & (labels >= 0) & (labels < vocab)


def softmax_xent_fwd_bwd(logits, labels, gscale=1.0, d_gscale=None, ignore_index=-100, inplace_grad=True):
    """Per-row loss (fp32) and, written **in place over ``logits``** when ``inplace_grad``, the gradient
    ``(softmax - onehot) * gscale``.  Rows that :func:`xent_valid` rejects get loss 0 and gradient 0.
    Returns ``(loss_rows, grad_or_None)``.  Not an autograd function: callers (``chunked_linear_xent``) wire the
    gradient manually."""
    rows, vocab = logits.shape
    loss = torch.empty(rows, dtype=torch.float32, device=logits.device)
    if logits.is_cuda:
        grad = logits if inplace_grad else None
        rc = N.cuda().dsb_softmax_xent(_p(logits), _p(labels), _p(loss), _null(), _p(grad), N.c_i64(rows), vocab,
                                       N.c_i64(logits.stride(0)), N.c_i64(ignore_index), N.c_f(gscale),
                                       _p(d_gscale), N.dt(logits), N.stream())
        N.check(rc, "softmax_xent")
        return loss, grad
    lf = logits.float()
    lse = torch.logsumexp(lf, dim=-1)
    valid = xent_valid(labels, vocab, ignore_index)
    safe = torch.where(valid, labels, 0)
    loss = torch.where(valid, lse - lf.gather(1, safe[:, None]).squeeze(1), torch.zeros_like(lse))
    grad = None
    if inplace_grad:
        p = torch.exp(lf - lse[:, None])
        p.scatter_add_(1, safe[:, None], -torch.ones_like(p[:, :1]))
        gs = gscale * (float(d_gscale.item()) if d_gscale is not None else 1.0)
        p = p * gs * valid[:, None]
        logits.copy_(p.to(logits.dtype))
        grad = logits
    return loss, grad


class _XentFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, logits, labels, ignore_index):
        l2 = logits.reshape(-1, logits.shape[-1])
        work = l2.clone()  # gradient is produced in place on the clone
        lab = labels.reshape(-1).contiguous()
        loss, grad = softmax_xent_fwd_bwd(work, lab, 1.0, None, ignore_index, True)
        n = xent_valid(lab, l2.shape[-1], ignore_index).sum().clamp(min=1)
        ctx.save_for_backward(grad, n)
        ctx.shape = logits.shape
        return loss.sum() / n

    @staticmethod
    def backward(ctx, dloss):
        grad, n = ctx.saved_tensors
        return (grad.float() * (dloss / n)).to(grad.dtype).view(ctx.shape), None, None


def cross_entropy(logits, labels, ignore_index=-100):
    """Mean token cross entropy via the fused kernel (drop-in for ``F.cross_entropy``)."""
    return _XentFn.apply(logits, labels, ignore_index)


def fused_add(a, b, c=None, d=None, scale=1.0):
    if a.is_cuda:
        y = torch.empty_like(a)
        rc = N.cuda().dsb_fused_add(_p(a), _p(b), _p(c), _p(d), _p(y), N.c_i64(a.numel()), N.c_f(scale), N.dt(a),
                                    N.stream())
        N.check(rc, "fused_add")
        return y
    out = a.float() + b.float()
    if c is not None:
        out = out + c.float()
    if d is not None:
        out = out + d.float()
    return (out * scale).to(a.dtype)
