"""RMSNorm forward and backward at the shapes the Llama training step runs, against float64.

A bf16 RMSNorm backward with ``hidden % 1024 == 0``, ``hidden <= 8192`` and at least 1024 rows runs the bulk-async kernel
(one template instantiation per ``hidden / 1024``, two CTAs per SM up to hidden 4096 and one above); fewer rows run the
register-cached kernel.  Every bulk case asserts which kernel the library picks, so a changed threshold cannot turn these
into register-path tests unnoticed.  Bounds are per element, in the terms of ``tests/numerics.py``.
"""
import math

import pytest
import torch

from tests.numerics import U, assert_within, ulp

pytestmark = pytest.mark.gpu

EPS = 1e-5
# forward rstd: <= 32 fp32 fma per thread and a block reduction of <= 10 levels (42 U on the sum of squares, halved by the
# square root), the divide and the eps add, rsqrtf's 2 ulp
RSTD_REL = 32 * U
# backward row reduction sum(dy * w * xhat): <= 64 fma per thread (VPT * 8 in the bulk kernel, 4 * 8 in the register
# one), <= 16 reduction levels
N_ROW_SUM = 80


def _inputs(rows, hidden, dtype, with_res, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda *s: torch.randn(*s, generator=g, device="cuda")
    x = mk(rows, hidden).to(dtype)
    r = mk(rows, hidden).to(dtype) if with_res else None
    w = (1 + 0.1 * mk(hidden)).to(dtype)
    return x, r, w, mk(rows, hidden).to(dtype), (mk(rows, hidden).to(dtype) if with_res else None)


def _forward_reference(xin, w):
    xin = xin.double()
    rstd = torch.rsqrt(xin.pow(2).mean(-1) + EPS)
    return xin * rstd[:, None] * w.double(), rstd


# ---------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("hidden", [3072, 5120, 7168])  # 96 / 160 / 224 threads per row in 16-bit types
def test_rms_norm_forward(hidden, dtype, with_res):
    from deepspeed_b200.ops.kernels.transformer_ops import _norm_fwd_native
    rows = 300
    x, r, w, _, _ = _inputs(rows, hidden, dtype, with_res, seed=hidden)
    y, res_out, _, rstd = _norm_fwd_native(x, r, w, None, EPS, 0)
    if with_res:
        # the residual stream is x + r rounded once to the storage type, exactly what torch computes
        assert torch.equal(res_out, x + r)
    xin = res_out if with_res else x
    y_ref, rstd_ref = _forward_reference(xin, w)
    assert_within(rstd, rstd_ref, RSTD_REL * rstd_ref, "rstd")
    # y = (x * rstd) * w: two fp32 roundings on top of rstd's error
    assert_within(y, y_ref, ulp(y_ref, dtype) + (RSTD_REL + 2 * U) * y_ref.abs(), "y")


# ---------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------
def _backward(x, r, w, gy, gres):
    """dx, d(residual), dw through the public autograd function, as the model calls it."""
    from deepspeed_b200.ops.kernels import transformer_ops as T
    x = x.clone().requires_grad_(True)
    w = w.clone().requires_grad_(True)
    if r is None:
        torch.autograd.backward([T.rms_norm(x, w, EPS)], [gy])
        return x.grad, None, w.grad
    r = r.clone().requires_grad_(True)
    y, s = T.rms_norm(x, w, EPS, residual=r)
    torch.autograd.backward([y, s], [gy, gres])
    return x.grad, r.grad, w.grad


def _check_backward(x, r, w, gy, gres, dx, dr, dw):
    rows, hidden = x.shape
    xin = ((x + r) if r is not None else x).double()  # the forward saves the rounded residual stream
    dy, w64 = gy.double(), w.double()
    rstd = torch.rsqrt(xin.pow(2).mean(-1, keepdim=True) + EPS)
    xhat = xin * rstd
    g = dy * w64
    m2 = (g * xhat).mean(-1, keepdim=True)
    t = xhat * m2
    dx_ref = rstd * (g - t)
    if gres is not None:
        dx_ref = dx_ref + gres.double()
    dw_ref = (dy * xhat).sum(0)

    # dx = rstd * (dy * w - x * rstd * m2) (+ dres): dy * w is exact in fp32; m2 carries N_ROW_SUM roundings and rstd's
    # error over sum|g * xhat| / hidden; t and the difference round three times; rstd enters up to three times
    m2_err = (N_ROW_SUM + 1 + RSTD_REL / U) * U * (g * xhat).abs().mean(-1, keepdim=True)
    pre = rstd * ((g.abs() + t.abs()) * (4 * U + 3 * RSTD_REL) + xin.abs() * rstd * m2_err)
    if gres is not None:
        pre = pre + U * gres.double().abs()
    assert_within(dx, dx_ref, ulp(dx_ref, dx.dtype) + pre, "dx")
    if r is not None:
        assert_within(dr, dx_ref, ulp(dx_ref, dr.dtype) + pre, "d(residual)")
    # dw: one fp32 fma per row into a per-CTA partial (<= ceil(rows / 132) rows per CTA), then a column sum over <= 528
    # partials (<= 66 sequential adds plus an 8-way tree); xhat rounds once and carries rstd's error
    n_dw = math.ceil(rows / 132) + 66 + 8 + 1 + RSTD_REL / U
    dw_pre = n_dw * U * (dy * xhat).abs().sum(0)
    assert_within(dw, dw_ref, ulp(dw_ref, dw.dtype) + dw_pre, "dw")


def _bulk_cases():
    for hidden in range(1024, 8193, 1024):  # every VPT instantiation; 2 CTAs per SM up to 4096, 1 above
        for rows in (1024, 1024 + 37):  # 1061 rows: CTAs own 4 or 5 rows, so the 4-stage ring wraps unevenly
            yield hidden, rows
    for hidden in (3072, 8192):  # 8192 rows = the training step's 2 x 4096 tokens: ~31-62 rows per CTA
        yield hidden, 8192


@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("hidden,rows", list(_bulk_cases()))
def test_rms_norm_backward_bulk(hidden, rows, with_res):
    from deepspeed_b200.ops.kernels import transformer_ops as T
    x, r, w, gy, gres = _inputs(rows, hidden, torch.bfloat16, with_res, seed=hidden * 7 + rows)
    assert all(t.data_ptr() % 16 == 0 for t in (x, gy) + ((r, gres) if with_res else ()))
    assert T.norm_bwd_path(rows, hidden, 0, torch.bfloat16) == "bulk"
    dx, dr, dw = _backward(x, r, w, gy, gres)
    _check_backward(x, r, w, gy, gres, dx, dr, dw)


def test_rms_norm_backward_path_boundary():
    """1023 rows run the register kernel and 1024 the bulk kernel; both agree with float64 on the same leading rows."""
    from deepspeed_b200.ops.kernels import transformer_ops as T
    hidden = 3072
    x, r, w, gy, gres = _inputs(1024, hidden, torch.bfloat16, True, seed=1023)
    for rows, path in ((1023, "register"), (1024, "bulk")):
        assert T.norm_bwd_path(rows, hidden, 0, torch.bfloat16) == path
        xs, rs, gys, gress = (t[:rows].contiguous() for t in (x, r, gy, gres))
        dx, dr, dw = _backward(xs, rs, w, gys, gress)
        _check_backward(xs, rs, w, gys, gress, dx, dr, dw)
