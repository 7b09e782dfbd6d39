"""Float64 references and per-element error bounds shared by the kernel tests.

A bound has two parts:
* one ulp of the output type at |reference|: the final rounding is at most half an ulp of the computed value, and that
  value may sit one binade above the reference;
* the error the computation accumulates before that rounding, written as a multiple of the fp32 unit roundoff ``U``
  times the magnitudes that enter it.
"""
import math

import torch

U = 2.0**-24  # fp32 unit roundoff
_MANT = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}
_EMIN = {torch.float32: -126, torch.bfloat16: -126, torch.float16: -14}


def ulp(x, dtype):
    """Spacing of ``dtype`` values at |x| (float64 result); the subnormal spacing below the normal range."""
    x = x.double().abs()
    _, e = torch.frexp(x)  # x = m * 2**e, m in [0.5, 1)
    e = torch.where(x > 0, e - 1, _EMIN[dtype]).clamp(min=_EMIN[dtype])
    return torch.ldexp(torch.ones_like(x), e - _MANT[dtype])


def assert_within(out, ref, bound, what):
    """|out - ref| <= bound element by element; non-finite reference entries must be matched exactly."""
    out, ref = out.double(), ref.double()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(ref)
    fin = torch.isfinite(ref)
    if not bool(fin.all()):
        assert torch.equal(out[~fin], ref[~fin]), f"{what}: non-finite reference entries differ"
    err = (out - ref).abs()
    bad = fin & ~(err <= bound)  # a NaN output fails
    if bool(bad.any()):
        ratio = torch.where(bad, err.nan_to_num(math.inf) / bound.clamp_min(1e-300), -1.0).reshape(-1)
        k = int(ratio.argmax())
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(k), ref.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} elements outside the bound; worst at {idx}: "
                             f"got {out.reshape(-1)[k].item()!r}, want {ref.reshape(-1)[k].item()!r} "
                             f"+- {bound.reshape(-1)[k].item():.3g}")


# ---------------------------------------------------------------------------------------------------------------------
# softmax cross entropy
# ---------------------------------------------------------------------------------------------------------------------
def xent_reference(logits, labels, ignore_index=-100, gscale=1.0):
    """Float64 per-row loss and gradient ``(softmax - onehot) * gscale``.  A row counts when its label is in
    ``[0, vocab)`` and is not ``ignore_index``; every other row has loss 0 and gradient 0.
    Returns ``(loss, grad, lse, p, valid)``."""
    lf = logits.double()
    vocab = lf.shape[1]
    valid = (labels != ignore_index) & (labels >= 0) & (labels < vocab)
    safe = torch.where(valid, labels, 0)[:, None]
    lse = torch.logsumexp(lf, -1)
    p = torch.exp(lf - lse[:, None])
    loss = torch.where(valid, lse - lf.gather(1, safe).squeeze(1), 0.0)
    grad = p.scatter_add(1, safe, -torch.ones_like(p[:, :1])) * (gscale * valid[:, None])
    return loss, grad, lse, p, valid


def xent_kernel_error(lf, lse):
    """Error of the fused softmax-xent kernel before its output rounding, for float64 logits ``lf`` (what the kernel
    read) and their float64 ``lse``.  Returns ``(lse_err [rows], p_rel [rows, vocab])``: the absolute error of the
    kernel's log-sum-exp and the relative error of each ``exp(x - lse)`` it forms.

    The kernel sums ``__expf(x - running_max)`` in fp32: at most ``ceil(vocab / threads)`` adds per thread, then two
    block reductions of at most 10 levels each.  ``__expf`` is exact to 2 ulp plus ``|arg| U`` from rounding the argument
    times log2(e); the running-max rescales of a thread add up to at most the row's span.  ``__logf`` is exact to
    ``2**-21`` absolute, and ``max + log(sum)`` rounds once more."""
    vocab = lf.shape[1]
    threads = 1024 if vocab >= 8192 else 128  # (256 threads for 2048 <= vocab < 8192: 128 over-counts the adds)
    fin = torch.isfinite(lf)
    mx = lf.max(-1).values
    span = mx - torch.where(fin, lf, mx[:, None]).min(-1).values
    rel_sum = (math.ceil(vocab / threads) + 24 + 3 * span) * U
    lse_err = rel_sum + 2.0**-21 + 2 * U * lse.abs()
    p_rel = lse_err[:, None] + ((lf - lse[:, None]).abs() + 4) * U
    return lse_err, p_rel


def xent_bounds(logits, loss_ref, grad_ref, lse, p, gscale, dtype):
    """Per-element bounds for the kernel's row loss (fp32) and its gradient written in ``dtype``."""
    lf = logits.double()
    lse_err, p_rel = xent_kernel_error(lf, lse)
    loss_bound = lse_err + U * (lse.abs() + loss_ref.abs())
    # p * p_rel is the error of exp(x - lse); the label's "- 1", the gscale product and the scaling round once each;
    # exp results below the normal range flush to zero
    pre = torch.where(p > 0, p * p_rel, 0.0) + 2.0**-126
    grad_bound = ulp(grad_ref, dtype) + abs(gscale) * pre + 3 * U * grad_ref.abs()
    return loss_bound, grad_bound


# ---------------------------------------------------------------------------------------------------------------------
# LM head + cross entropy over token chunks
# ---------------------------------------------------------------------------------------------------------------------
def chunked_xent_reference(h, w, labels, chunk, ignore_index=-100):
    """Float64 mean cross entropy of ``softmax(h w^T)`` against ``labels`` and its gradients ``dh`` and ``dW`` for a unit
    upstream gradient, with per-element bounds for the pipeline ``chunked_linear_xent`` runs in ``h.dtype``:

    1. the logits GEMM accumulates ``H`` products in fp32 (at most ``H U sum|h||w|``) and rounds to ``h.dtype``;
    2. the fused kernel forms ``(softmax - onehot) / n`` from those logits and writes it in ``h.dtype``; a logit error
       ``dz`` moves ``p_j`` by the factor ``exp(dz_j - d lse)`` with ``|d lse| <= log sum_k p_k exp(dz_k)``;
    3. ``dh = grad @ w`` accumulates ``V`` products and rounds once;
    4. ``dW`` accumulates ``grad^T h`` chunk by chunk and rounds to ``h.dtype`` after every chunk.

    Returns ``(loss, dh, dW, loss_bound, dh_bound, dW_bound)``; the references are float64 tensors on ``h.device``."""
    dtype = h.dtype
    T, H = h.shape
    V = w.shape[0]
    w64 = w.double()
    valid = (labels != ignore_index) & (labels >= 0) & (labels < V)
    n = max(int(valid.sum()), 1)
    dh = torch.empty(T, H, dtype=torch.float64, device=h.device)
    dh_bound = torch.empty_like(dh)
    dW = torch.zeros(V, H, dtype=torch.float64, device=h.device)
    dW_bound = torch.zeros_like(dW)
    loss_sum = loss_abs = loss_err = 0.0
    n_chunks = 0
    for s in range(0, T, chunk):
        e = min(s + chunk, T)
        n_chunks += 1
        hc = h[s:e].double()
        z = hc @ w64.t()
        acc = H * U * (hc.abs() @ w64.abs().t())
        dz = 0.5 * ulp(z.abs() + acc, dtype) + acc
        del acc
        loss_c, g, lse, p, vc = xent_reference(z, labels[s:e], ignore_index, 1.0 / n)
        shift = torch.logsumexp(torch.log(p) + dz, -1)  # bound on |d lse| (log p = -inf where p underflowed: fine)
        lse_err, p_rel = xent_kernel_error(z, lse)
        safe = torch.where(vc, labels[s:e], 0)[:, None]
        loss_sum += float(loss_c.sum())
        loss_abs += float(loss_c.abs().sum())
        loss_err += float(((shift + dz.gather(1, safe).squeeze(1) + lse_err) * vc).sum())
        pre = torch.where(p > 0, p * torch.expm1(dz + shift[:, None] + p_rel), 0.0)
        del z, dz, p_rel
        pre = (pre + 2.0**-126) * vc[:, None] / n  # rows that do not count are written as exact zeros
        eg = pre + ulp(g.abs() + pre, dtype) + 3 * U * g.abs()
        del pre
        dh[s:e] = g @ w64
        dh_bound[s:e] = (eg + V * U * g.abs()) @ w64.abs()
        dW += g.t() @ hc
        dW_bound += (eg + (e - s) * U * g.abs()).t() @ hc.abs()
        dW_bound += ulp(dW.abs() + dW_bound, dtype)
        del g, eg, p
    dh_bound += ulp(dh.abs() + dh_bound, dtype)
    loss = loss_sum / n
    # row losses are summed in fp32 within a chunk (at most ``chunk`` adds), then chunk by chunk
    loss_bound = (loss_err + (chunk + n_chunks + 2) * U * loss_abs) / n + U * abs(loss)
    return loss, dh, dW, loss_bound, dh_bound, dW_bound
