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


def assert_bits_equal(out, ref, what):
    """``out`` and ``ref`` (same dtype) hold the same bit patterns, NaN payloads and signed zeros included."""
    assert out.dtype == ref.dtype and out.shape == ref.shape, (what, out.dtype, ref.dtype, out.shape, ref.shape)
    view = {1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[out.element_size()]
    bad = out.contiguous().view(view) != ref.contiguous().view(view)
    if bool(bad.any()):
        k = int(bad.reshape(-1).nonzero()[0])
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(k), ref.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} elements differ; first at {idx}: "
                             f"got {out.reshape(-1)[k].item()!r}, want {ref.reshape(-1)[k].item()!r}")


# ---------------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------------
def exact_grid(rows, cols, gen, emin=-12, emax=12, ints=4):
    """bf16 ``[rows, cols]``: integers in ``[-ints, ints]`` times ``2**e_r``, one exponent per row.  Returns
    ``(tensor, e)`` with ``e`` the int32 exponents ``[rows]``.

    Used as ``A [M, K]`` and ``B [N, K]`` of ``A @ B^T``, every term of the dot product of row i and column j is an integer
    times ``2**(e_i + f_j)``.  While ``sum_k |a_ik| |b_jk| < 2**22`` (``16 K < 2**22``: any K up to 262143) every product
    and every partial sum is exactly representable in fp32, so an fp32 accumulation is exact in any order and the
    product rounds to bf16 exactly once.  Each row and column of C gets its own scale, so a value written to the wrong
    row, column or tile cannot match."""
    dev = gen.device
    v = torch.randint(-ints, ints + 1, (rows, cols), generator=gen, device=dev, dtype=torch.int32).float()
    e = torch.randint(emin, emax + 1, (rows, ), generator=gen, device=dev, dtype=torch.int32)
    return torch.ldexp(v, e[:, None]).bfloat16(), e


def exact_addend(e_rows, e_cols, gen, ints=128):
    """bf16 ``C_old [M, N]`` on the grid of ``A @ B^T`` for row exponents ``e_rows`` of A and ``e_cols`` of B: integers in
    ``[-ints, ints]`` (exact in bf16 up to 256) times ``2**(e_i + f_j)``, so ``C_old + A @ B^T`` stays exact in fp32."""
    v = torch.randint(-ints, ints + 1, (e_rows.numel(), e_cols.numel()), generator=gen, device=gen.device,
                      dtype=torch.int32).float()
    return torch.ldexp(v, e_rows[:, None] + e_cols[None, :]).bfloat16()


def _gemm_blocks(M, N, K, budget=2**24):
    """Row and column blocks of an [M, N] product whose float64 operand and result blocks hold at most ``budget``
    (or one 128-row / 128-column strip) elements each: 128 MB in float64, whatever the problem."""
    cb = min(N, max(128, budget // max(K, 1)))
    rb = min(M, max(128, min(budget // cb, budget // max(K, 1))))
    for r in range(0, M, rb):
        for c in range(0, N, cb):
            yield slice(r, min(r + rb, M)), slice(c, min(c + cb, N))


def gemm_reference(a, b, c_old=None, magnitudes=False):
    """Float64 ``a @ b^T (+ c_old)`` block by block: yields ``(rows, cols, ref, mag)`` with ``mag = |a| @ |b|^T`` when
    ``magnitudes`` else None.  ``a`` [M, K] and ``b`` [N, K] may be any strided views (transposes included)."""
    M, K = a.shape
    N = b.shape[0]
    for rs, cs in _gemm_blocks(M, N, K):
        a64, b64 = a[rs].double(), b[cs].double()
        ref = a64 @ b64.t()
        if c_old is not None:
            ref += c_old[rs, cs].double()
        mag = a64.abs() @ b64.abs().t() if magnitudes else None
        del a64, b64
        yield rs, cs, ref, mag


def assert_gemm_exact(c, a, b, c_old=None, what="C"):
    """``c`` is bit-equal to ``bf16(a @ b^T + c_old)`` rounded once from the exact sum; valid for :func:`exact_grid`
    operands (and a ``c_old`` on the same grid), where that sum is exactly representable in fp32."""
    for rs, cs, ref, _ in gemm_reference(a, b, c_old):
        assert_bits_equal(c[rs, cs], ref.to(torch.bfloat16), f"{what}[{rs.start}:{rs.stop}, {cs.start}:{cs.stop}]")


def gemm_accum_error(mag, K):
    """Error of an fp32 accumulator that sums ``K`` bf16 products of magnitudes ``mag = |A| @ |B|^T``.

    bf16 products are exact in fp32.  Summing K of them in any order, each add rounding to nearest, errs by at most
    ``K U sum_k |a_k||b_k|`` (``U = 2**-24``); the tensor core's adder may truncate instead of rounding, which at most
    doubles the per-add error, hence ``2 K U |A| |B|^T``.  An accumulation in any format with fewer than 23 fraction bits
    cannot meet it."""
    return 2 * K * U * mag


def gemm_bound(ref, mag, K, c_old=None):
    """Per-element bound on a bf16 GEMM output that accumulates ``K`` products in fp32 (:func:`gemm_accum_error`).
    ``EPI_ACCUM`` adds ``c_old`` in fp32 (one more rounding, ``U`` times the sum) before the bf16 rounding, which costs
    at most one :func:`ulp` of the computed value."""
    acc = gemm_accum_error(mag, K)
    if c_old is not None:
        acc = acc + U * (ref.abs() + acc)
    return ulp(ref.abs() + acc, torch.bfloat16) + acc


def assert_gemm_bounded(c, a, b, c_old=None, what="C"):
    """``|c - (a @ b^T + c_old)| <= gemm_bound`` element by element, in float64."""
    K = a.shape[1]
    for rs, cs, ref, mag in gemm_reference(a, b, c_old, magnitudes=True):
        assert_within(c[rs, cs], ref, gemm_bound(ref, mag, K, c_old), f"{what}[{rs.start}:{rs.stop}, {cs.start}:{cs.stop}]")


# ---------------------------------------------------------------------------------------------------------------------
# SwiGLU
# ---------------------------------------------------------------------------------------------------------------------
SILU_LIP = 1.1  # max |silu'(x)| = 1.0998...: silu moves by at most 1.1 |dx|


def swiglu_reference(g, u, g_err=0.0, u_err=0.0):
    """Float64 ``act = silu(g) * u`` and its bound for a kernel that forms ``silu(g) = g / (1 + __expf(-g))`` in fp32 from
    fp32 inputs within ``g_err`` / ``u_err`` of ``g`` / ``u``, multiplies once and rounds to bf16.

    ``__expf`` is exact to 2 ulp plus ``|g| U`` from rounding its scaled argument; the add and the IEEE divide round once
    each, so silu carries ``(|g| + 6) U`` relative error and the product one more ``U``.  Below ``g = -80`` ``__expf(-g)``
    may overflow and the kernel writes 0, which is within ``|act|`` of the truth.  An input error moves ``act`` by at most
    ``1.1 g_err (|u| + u_err) + |silu(g)| u_err``.

    Which ``g`` and ``u`` to pass depends on the path.  The fused GEMM epilogue applies silu to the fp32 accumulators: pass
    the float64 sums, with the accumulation bound (:func:`gemm_bound` without its final rounding) as the input error, or
    none on :func:`exact_grid` data, where the accumulators are exact.  The library path applies silu to the gate|up it
    stored in bf16: pass those bf16 values, which is what it read, without an input error.  Measured against the float64
    sums instead, the library path would need an extra ``ulp(g) / 2`` and ``ulp(u) / 2`` of input error for that
    rounding, so its bound is looser than the fused epilogue's."""
    g, u = g.double(), u.double()
    silu = g * torch.sigmoid(g)
    act = silu * u
    moved = SILU_LIP * g_err * (u.abs() + u_err) + silu.abs() * u_err
    mag = act.abs() + moved
    bound = ulp(mag, torch.bfloat16) + moved + (g.abs() + g_err + 8) * U * mag + torch.where(g < -80, mag, 0.0)
    return act, bound


def dswiglu_reference(d, g, u, d_fp32=False, d_err=0.0):
    """Float64 ``(dgate, dup)`` of ``act = silu(g) * u`` for the upstream gradient ``d``, and their bounds for a kernel
    that computes ``dgate = (d * u) * s (1 + g (1 - s))`` and ``dup = d * silu(g)`` in fp32 (``s = 1 / (1 + __expf(-g))``,
    silu as in :func:`swiglu_reference`) from bf16 ``g`` and ``u`` and rounds each to bf16.  Returns
    ``(dgate, dgate_bound, dup, dup_bound)``.

    With ``d`` in bf16 the product ``d * u`` is exact in fp32 (8 x 8 significant bits).  ``d_fp32=True`` is the dSwiGLU
    GEMM epilogue, whose ``d`` is an fp32 accumulator: ``d * u`` then rounds once, one more ``U |dgate|``; ``d_err`` is
    that accumulator's error, which the two products carry as ``|u dsilu(g)| d_err`` and ``|silu(g)| d_err``."""
    d, g, u = d.double(), g.double(), u.double()
    s = torch.sigmoid(g)
    silu = g * s
    inner = 1 + g * (1 - s)
    s_err = s * (g.abs() + 6) * U  # sigmoid carries (|g| + 6) U relative, as silu does
    dact = s * inner
    # s's error enters through s and 1 - s; the products of s (1 + g (1 - s)) round once each
    dact_err = s_err * (inner.abs() + s * g.abs()) + s * U * (2 * g.abs() * (1 - s).abs() + inner.abs()) + U * dact.abs()
    dgate = d * u * dact
    moved = (u * dact).abs() * d_err
    mag = dgate.abs() + moved
    dgate_bound = ulp(mag, torch.bfloat16) + moved + ((d.abs() + d_err) * u.abs()) * (dact_err + U * dact.abs())
    if d_fp32:
        dgate_bound = dgate_bound + U * mag
    dup = d * silu
    moved = silu.abs() * d_err
    mag = dup.abs() + moved
    dup_bound = ulp(mag, torch.bfloat16) + moved + (g.abs() + 8) * U * mag
    return dgate, dgate_bound, dup, dup_bound


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


# ---------------------------------------------------------------------------------------------------------------------
# training attention (csrc/cuda/attn_sm90.cu)
# ---------------------------------------------------------------------------------------------------------------------
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
U_BF16 = 2.0**-8  # bf16 unit roundoff: 8 significant bits, round to nearest
ATTN_BLOCK = 64  # keys per block of the forward and dQ kernels, query rows per block of the dK / dV kernel
ATTN_ROWS = 1024  # query rows per float64 chunk: a [1024, 4096] float64 matrix is 32 MB


def _rel(n):
    """``|prod (1 + d_k) - 1|`` for ``n`` fp32 roundings ``|d_k| <= U``."""
    return math.expm1(n * math.log1p(U))


def attention_documents(T, cu_seqlens=None):
    """Non-empty ``(start, end)`` token spans: the documents of ``cu_seqlens`` or one sequence of ``T`` rows."""
    cu = [0, T] if cu_seqlens is None else [int(c) for c in cu_seqlens]
    return [(s, e) for s, e in zip(cu[:-1], cu[1:]) if e > s]


def attention_visible(L, causal=True, window=None, device=None):
    """bool ``[L, L]``: query row i sees key j -- ``j <= i`` when causal, and ``i - window < j`` with a window."""
    i = torch.arange(L, device=device)
    diff = i[:, None] - i[None, :]
    vis = diff >= 0 if causal else torch.ones(L, L, dtype=torch.bool, device=device)
    if window is not None:
        vis = vis & (diff < window)
    return vis


def _attention(q, k, v, do, cu_seqlens, causal, window, scale, mask, kv_heads, bounds):
    """Float64 attention one (document, query head, chunk of query rows) at a time, and the bounds of
    :func:`attention_bounds` when ``bounds``.  Heads outside ``kv_heads`` keep reference 0 and bound inf."""
    T, Hq, d = q.shape
    Hkv = k.shape[1]
    rep = Hq // Hkv
    c = 1.0 / math.sqrt(d) if scale is None else float(scale)
    cl = c * LOG2E
    f64 = dict(dtype=torch.float64, device=q.device)
    ref = {"o": torch.zeros(T, Hq, d, **f64), "lse": torch.zeros(Hq, T, **f64)}
    if do is not None:
        ref.update(dq=torch.zeros(T, Hq, d, **f64), dk=torch.zeros(T, Hkv, d, **f64), dv=torch.zeros(T, Hkv, d, **f64))
    bnd = {n: torch.full_like(r, math.inf) for n, r in ref.items()} if bounds else None
    R2, R3, R4 = _rel(2), _rel(3), _rel(4)
    for s0, e0 in attention_documents(T, cu_seqlens):
        L = e0 - s0
        vis = mask[s0:e0, s0:e0] if mask is not None else attention_visible(L, causal, window, q.device)
        n_b = -(-L // ATTN_BLOCK)  # key blocks (forward, dQ) or query blocks per head (dK / dV) a kernel visits at most
        for g in (range(Hkv) if kv_heads is None else kv_heads):
            K, V = k[s0:e0, g].double(), v[s0:e0, g].double()
            aK, aV = K.abs(), V.abs()
            if do is not None:
                dK, dV = torch.zeros(L, d, **f64), torch.zeros(L, d, **f64)
                if bounds:
                    eK, mK, eV, mV = (torch.zeros(L, d, **f64) for _ in range(4))
            for h in range(g * rep, (g + 1) * rep):
                for r0 in range(0, L, ATTN_ROWS):
                    r1 = min(r0 + ATTN_ROWS, L)
                    rows = slice(s0 + r0, s0 + r1)
                    vm = vis[r0:r1]
                    Q = q[rows, h].double()
                    sc = Q @ K.t()
                    t = (sc * c).masked_fill(~vm, -math.inf)
                    lse = torch.logsumexp(t, -1)
                    P = torch.exp(t - lse[:, None]).nan_to_num(0.0)  # a row that sees nothing: P = 0
                    O = P @ V
                    ref["o"][rows, h] = O
                    ref["lse"][h, rows] = lse
                    if do is not None:
                        dO = do[rows, h].double()
                        dP = dO @ V.t()
                        delta = (dO * O).sum(-1)
                        dS = P * (dP - delta[:, None]) * c
                        ref["dq"][rows, h] = dS @ K
                        dK += dS.t() @ Q
                        dV += P.t() @ dO
                    if not bounds:
                        continue
                    # ---- forward ----
                    zero = torch.zeros((), **f64)
                    e_s = gemm_accum_error(Q.abs() @ aK.t(), d)
                    err_x = torch.where(vm, cl * (e_s * (1 + R4) + R4 * sc.abs()), zero)
                    t2 = torch.where(vm, sc * cl, zero)
                    t2max = torch.where(vm, t2, -math.inf).max(-1).values
                    emax = err_x.max(-1).values
                    dist = t2max[:, None] - t2 + err_x + emax[:, None]
                    span = t2max - torch.where(vm, t2, math.inf).min(-1).values + 2 * emax
                    lnrel = LN2 * (err_x + U * (dist + span[:, None])) + (5 * n_b + 4) * U
                    Pe = torch.where(vm, P * torch.expm1(lnrel) + 2.0**-125, zero)
                    Pw = P + Pe  # bound on |p~| / l
                    num = (Pe + U_BF16 * Pw) @ aV + gemm_accum_error((Pw * (1 + U_BF16)) @ aV, ATTN_BLOCK * n_b)
                    rho = Pe.sum(-1) + (16 * n_b + 2) * U * Pw.sum(-1)
                    e_pre = (num + O.abs() * rho[:, None]) / (1 - rho)[:, None]
                    e_o = e_pre + R2 * (O.abs() + e_pre)
                    b_o = ulp(O.abs() + e_o, torch.bfloat16) + e_o
                    bnd["o"][rows, h] = b_o
                    a = -torch.log1p(-rho) * LOG2E + 2 * U * torch.log2(vm.sum(-1).double() + 1)
                    e2 = a + U * (lse.abs() * LOG2E + a)
                    b_lse = LN2 * e2 + R2 * (lse.abs() + LN2 * e2)
                    bnd["lse"][h, rows] = b_lse
                    if do is None:
                        continue
                    # ---- backward ----
                    e_l2 = LOG2E * b_lse * (1 + R2) + R2 * LOG2E * lse.abs()
                    e_xc = cl * (e_s * (1 + R3) + R3 * sc.abs())
                    y = (t2 - lse[:, None] * LOG2E).abs()
                    err_y = e_xc + e_l2[:, None] + U * (y + e_xc + e_l2[:, None])
                    Pbe = torch.where(vm, P * torch.expm1(LN2 * err_y + 4 * U) + 2.0**-126, zero)
                    e_dp = gemm_accum_error(dO.abs() @ aV.t(), d)
                    aOh = O.abs() + b_o
                    e_delta = (dO.abs() * b_o).sum(-1) + 8 * U * (dO.abs() * aOh).sum(-1)
                    e_g = e_dp + e_delta[:, None]
                    gabs = (dP - delta[:, None]).abs()
                    e_dS = c * (Pbe * (gabs + e_g) + P * e_g) + R4 * c * (P + Pbe) * (dP.abs() + delta.abs()[:, None] + e_g)
                    e_dS = torch.where(vm, e_dS + U_BF16 * (dS.abs() + e_dS), zero)
                    aS = dS.abs() + e_dS
                    e_P = Pbe + U_BF16 * (P + Pbe)
                    aP = P + e_P
                    e_q = e_dS @ aK + gemm_accum_error(aS @ aK, ATTN_BLOCK * n_b)
                    bnd["dq"][rows, h] = ulp(ref["dq"][rows, h].abs() + e_q, torch.bfloat16) + e_q
                    eK += e_dS.t() @ Q.abs()
                    mK += aS.t() @ Q.abs()
                    eV += e_P.t() @ dO.abs()
                    mV += aP.t() @ dO.abs()
            if do is None:
                continue
            ref["dk"][s0:e0, g] = dK
            ref["dv"][s0:e0, g] = dV
            if bounds:
                K_kv = rep * ATTN_BLOCK * n_b  # products each dK / dV accumulator sums: every query row of every head
                for name, R, e, m in (("dk", dK, eK, mK), ("dv", dV, eV, mV)):
                    e = e + gemm_accum_error(m, K_kv)
                    bnd[name][s0:e0, g] = ulp(R.abs() + e, torch.bfloat16) + e
    return ref, bnd


def attention_reference(q, k, v, do=None, cu_seqlens=None, causal=True, window=None, scale=None, mask=None,
                        kv_heads=None):
    """Float64 training attention from explicit formulas.  ``q [T, Hq, d]``, ``k / v [T, Hkv, d]`` and ``do [T, Hq, d]``
    (any dtype or strides); query head h reads kv head ``h // (Hq / Hkv)``.  Each document of ``cu_seqlens`` (one
    sequence of T rows when None) is attended on its own; row i of a document sees key j when ``j <= i`` (causal) and
    ``i - window < j`` (a window).  ``mask`` (bool ``[T, T]``) replaces that rule inside each document.

    With ``t = scale * q k^T`` over the visible keys: ``P = softmax(t)``, ``O = P V``, ``LSE = logsumexp(t)`` (natural
    log) and for the upstream ``do``: ``dP = do V^T``, ``delta = rowsum(do * O)``, ``dS = P (dP - delta) scale``,
    ``dQ = dS K``, ``dK = dS^T Q`` and ``dV = P^T do``, with dK and dV summed over the query heads of a group.

    Returns a dict of float64 tensors ``o [T, Hq, d]``, ``lse [Hq, T]`` and, with ``do``, ``dq``, ``dk``, ``dv``.
    Only the kv heads in ``kv_heads`` (all when None) and their query heads are computed; the rest stay 0."""
    return _attention(q, k, v, do, cu_seqlens, causal, window, scale, mask, kv_heads, False)[0]


def attention_bounds(q, k, v, do=None, cu_seqlens=None, causal=True, window=None, scale=None, kv_heads=None):
    """``(ref, bound)``: :func:`attention_reference` and per-element bounds on the outputs of ``attn_sm90.cu``, as dicts
    with the same keys.  Heads left out by ``kv_heads`` get bound inf.  Every term is a magnitude times unit roundoffs
    (``U = 2**-24`` for fp32, ``U_BF16 = 2**-8`` for bf16); ``n_b = ceil(L / 64)`` blocks bound the keys (or query
    rows per head) a kernel visits, and ``_rel(n)`` is ``n`` fp32 roundings compounded.

    Forward, per (query row, head), with ``t`` in the log2 domain and ``P`` relative to the kernel's running max:

    1. ``S = Q K^T`` sums d bf16 products in fp32: :func:`gemm_accum_error`.
    2. ``x = s * scale_log2``: ``scale_log2`` is ``fp32(fp32(scale) * fp32(log2 e))``, three roundings, and the product
       one more: ``_rel(4) |s|`` on top of the accumulation error.
    3. ``p = ex2.approx(x - m)``: 2 ulp (``4U`` relative) plus ``ln2 U |x - m|`` from rounding the argument (the model
       :func:`swiglu_reference` uses for ``__expf``); results below ``2**-126`` flush to zero.  ``|x - m|`` for any
       running max is at most the row's max minus x.
    4. Each key block rescales o and l by the same ``alpha = ex2(m_old - m_new)``.  The common factor cancels in
       ``o / l``, but blocks seen earlier carry more factors than later ones, so per block the ex2's ``4U`` and its
       argument's ``ln2 U |m_old - m_new|`` weigh p unevenly; the increments of the running max add up to the row's span.
       The two products round once each per block: ``5U`` per block in all, as a relative error of p.
    5. l sums the *unrounded* fp32 p: at most ``16 n_b + 2`` adds per thread (16 keys per block, two quad shuffles).
    6. ``O += P V`` uses p rounded to bf16: ``U_BF16 P |V|``.  This mismatch with l does not cancel and dominates.
       The fp32 accumulation runs over ``64 n_b`` keys.
    7. ``1 / l`` (IEEE) and the multiply round once each, then the bf16 rounding of O (one :func:`ulp`).
    8. ``LSE = (m + log2f(l)) ln2``: l's relative error ``rho`` becomes ``-log2(1 - rho)``; log2f is exact to 1 ulp
       (``2U |log2 l|``, ``l <= n_visible + 1``), the add rounds once and the product with ``fp32(ln 2)`` twice.

    Backward:

    9. The prep pass forms ``delta`` from the bf16 O the forward wrote: ``|O_bf16 - O| |dO|`` against the float64 delta,
       plus 8 roundings (three fmaf after an exact first product, five warp-tree adds) of ``|O_bf16| |dO|``.
    10. ``lse2 = lse * fp32(log2 e)`` rounds twice, on top of the forward's LSE error.
    11. ``p = ex2(fmaf(s, scale_log2, -lse2))``: the score error as in 1-2 with one fewer rounding (fmaf fuses the
        product), the lse2 error, the fmaf's rounding of its result, and ex2's ``4U``; an LSE error is a relative
        error of P.
    12. ``dP = dO V^T`` sums d products in fp32.
    13. ``dS = p (dP - delta) scale`` rounds at the subtraction, both products and ``fp32(scale)``: ``_rel(4)`` of
        ``p (|dP| + |delta|)`` -- the subtraction's rounding scales with its operands, not with ``|dP - delta|``.
    14. P and dS are rounded to bf16 before their MMAs.
    15. dV and dK accumulate ``rep * 64 n_b`` products in fp32 (every query row of every head of the group), dQ
        ``64 n_b`` (every key); each output rounds to bf16 once."""
    return _attention(q, k, v, do, cu_seqlens, causal, window, scale, None, kv_heads, True)


def assert_attention_bounded(got, q, k, v, do=None, cu_seqlens=None, causal=True, window=None, scale=None,
                             kv_heads=None, what="attention"):
    """Every output in ``got`` (a dict with any of ``o [T, Hq, d]``, ``lse [Hq, T]``, ``dq``, ``dk``, ``dv``) lies inside
    :func:`attention_bounds`.  Returns the worst ``err / bound`` per output."""
    ref, bnd = attention_bounds(q, k, v, do, cu_seqlens, causal, window, scale, kv_heads)
    worst = {}
    for name, out in got.items():
        out = out.to(ref[name].device).double()
        assert_within(out, ref[name], bnd[name], f"{what}: {name}")
        worst[name] = float(((out - ref[name]).abs() / bnd[name]).nan_to_num(0.0).max())
    return worst


def attention_emulation(q, k, v, do=None, cu_seqlens=None, causal=True, window=None, scale=None, mask=None):
    """The kernels' algorithm in torch fp32, with the same arguments and outputs as :func:`attention_reference`: scores
    in fp32 scaled by the fp32 ``scale * log2 e`` and exponentiated with exp2, P rounded to bf16 before ``P V`` while l
    sums the fp32 p, ``LSE = (m + log2 l) ln 2``; the backward recomputes P from the LSE, forms delta from the bf16 O,
    rounds dS and P to bf16 and accumulates in fp32.  O, dQ, dK and dV are bf16, the LSE fp32."""
    T, Hq, d = q.shape
    Hkv = k.shape[1]
    rep = Hq // Hkv
    c = torch.tensor(1.0 / math.sqrt(d) if scale is None else float(scale), dtype=torch.float32)
    c2 = c * torch.tensor(LOG2E, dtype=torch.float32)
    ln2 = torch.tensor(LN2, dtype=torch.float32)
    l2e = torch.tensor(LOG2E, dtype=torch.float32)
    f32 = dict(dtype=torch.float32, device=q.device)
    c, c2, ln2, l2e = (x.to(q.device) for x in (c, c2, ln2, l2e))
    o = torch.zeros(T, Hq, d, **f32)
    lse = torch.zeros(Hq, T, **f32)
    if do is not None:
        dq = torch.zeros(T, Hq, d, **f32)
        dk = torch.zeros(T, Hkv, d, **f32)
        dv = torch.zeros(T, Hkv, d, **f32)
    bf = lambda x: x.bfloat16().float()  # noqa: E731
    for s0, e0 in attention_documents(T, cu_seqlens):
        L = e0 - s0
        vm = mask[s0:e0, s0:e0] if mask is not None else attention_visible(L, causal, window, q.device)
        for h in range(Hq):
            g = h // rep
            Q, K, V = q[s0:e0, h].float(), k[s0:e0, g].float(), v[s0:e0, g].float()
            S = Q @ K.t()
            x = (S * c2).masked_fill(~vm, -math.inf)
            m = x.max(-1, keepdim=True).values
            m = torch.where(torch.isfinite(m), m, 0.0)
            p = torch.exp2(x - m)
            l = p.sum(-1, keepdim=True)
            oh = bf((bf(p) @ V) * torch.where(l > 0, 1 / l, 0.0))
            o[s0:e0, h] = oh
            lh = ((m + torch.log2(l)) * ln2).squeeze(-1)
            lse[h, s0:e0] = lh
            if do is None:
                continue
            dO = do[s0:e0, h].float()
            pb = torch.where(vm, torch.exp2(S * c2 - (lh * l2e)[:, None]), 0.0)
            dP = dO @ V.t()
            delta = (oh * dO).sum(-1, keepdim=True)
            dS = bf(pb * (dP - delta) * c)
            dq[s0:e0, h] = dS @ K
            dk[s0:e0, g] += dS.t() @ Q
            dv[s0:e0, g] += bf(pb).t() @ dO
    out = {"o": o.bfloat16(), "lse": lse}
    if do is not None:
        out.update(dq=dq.bfloat16(), dk=dk.bfloat16(), dv=dv.bfloat16())
    return out


ATTN_FAMILIES = ("diffuse", "peaked", "rescale", "uniform")


def attention_data(family, T, hq, hkv, d, gen):
    """bf16 ``(q [T, hq, d], k / v [T, hkv, d], do [T, hq, d])`` on ``gen``'s device for one data family:

    * ``diffuse``: ``randn * 0.7`` -- logits of std 0.5, a flat softmax;
    * ``peaked``: q and k ``randn * 2.4`` -- logits of std 5.8, a few keys carry each row;
    * ``rescale``: column 0 of k rises from -88 to 88 along the rows and q's column 0 is 88, so the scores rise along
      the keys (about +-1000 in the log2 domain at d = 128), the running max moves in every 64-key block, and the
      other columns add ``randn * 0.5``;
    * ``uniform``: K = 0, every visible key weighs the same and O is the mean of the visible V."""
    dev = gen.device
    rn = lambda *s: torch.randn(*s, generator=gen, device=dev)  # noqa: E731
    v, do = rn(T, hkv, d), rn(T, hq, d)
    if family == "diffuse":
        q, k, v = rn(T, hq, d) * 0.7, rn(T, hkv, d) * 0.7, v * 0.7
    elif family == "peaked":
        q, k = rn(T, hq, d) * 2.4, rn(T, hkv, d) * 2.4
    elif family == "rescale":
        q, k = rn(T, hq, d) * 0.5, rn(T, hkv, d) * 0.5
        q[:, :, 0] = 88.0
        k[:, :, 0] = torch.linspace(-88.0, 88.0, T, device=dev)[:, None]
    elif family == "uniform":
        q, k = rn(T, hq, d), torch.zeros(T, hkv, d, device=dev)
    else:
        raise ValueError(family)
    return tuple(x.bfloat16() for x in (q, k, v, do))


# ---------------------------------------------------------------------------------------------------------------------
# optimizers and gradient utilities (csrc/cuda/optim.cu, csrc/cpu/cpu_optim.cpp)
# ---------------------------------------------------------------------------------------------------------------------
# The kernels are built without fast-math: IEEE division and square root, and fp32 subnormals are kept (no flush to
# zero).  nvcc and g++ may contract ``a * b + c`` into one fma, and the host tier writes some of the kernels' explicit
# fmas as a product and a sum; every bound below counts the product's rounding too, so it holds either way.  Each rounding errs by at most ``U`` times its result plus ``TINY`` (half the
# smallest fp32 subnormal), which covers results in the subnormal range.
TINY = 2.0**-150


def f32(x):
    """``x`` rounded to fp32 (the value a ``float`` kernel argument carries), as a Python float."""
    return float(torch.tensor(float(x), dtype=torch.float32))


def adam_hyper(lr, beta1, beta2, eps, weight_decay, step, bias_correction=True, grad_scale=1.0, d_gscale=None,
               adamw=True):
    """The Adam hyperparameters as ``adam_math`` sees them: every argument rounded to fp32, the bias corrections
    ``1 - beta**step`` formed in float64 by the wrapper and rounded to fp32, ``1 - beta`` in fp32 (exact by Sterbenz for
    ``beta`` in [0.5, 1]) and the gradient scale ``fp32(grad_scale) * d_gscale`` rounded once."""
    b1, b2 = f32(beta1), f32(beta2)
    gs = f32(grad_scale)
    if d_gscale is not None:
        gs = f32(gs * f32(d_gscale))
    return dict(lr=f32(lr), b1=b1, b2=b2, b1m=f32(1.0 - b1), b2m=f32(1.0 - b2), eps=f32(eps), wd=f32(weight_decay),
                bc1=f32(1.0 - beta1**step) if bias_correction else 1.0,
                bc2=f32(1.0 - beta2**step) if bias_correction else 1.0, gs=gs, adamw=bool(adamw))


def _sqrt_err(x, e):
    """Bound on ``|sqrt(x') - sqrt(x)|`` for ``|x' - x| <= e``, ``x >= 0``."""
    lo = (x - e).clamp_min(0.0)
    return torch.minimum(e.sqrt(), e / (x.sqrt() + lo.sqrt()).clamp_min(1e-300))


def adam_reference(p, g, m, v, h, dtypes=None, update=False):
    """Float64 one Adam/AdamW step of ``adam_math`` from the state the kernel starts from (any dtypes), with the
    hyperparameters ``h`` of :func:`adam_hyper`.  Returns ``(p, m, v)`` and their bounds ``(bp, bm, bv)`` for outputs
    stored in ``dtypes = (param dtype, state dtype)`` (fp32 when None).

    The operation sequence and the error each step adds before the final rounding (absolute, ``e_x`` for value ``x``):

    1. ``g1 = g * gs``: one rounding.
    2. L2 (``adamw`` off): ``g2 = fma(wd, p, g1)``: one rounding.
    3. ``m' = fma(b1, m, fp32(b1m * g2))``: the product rounds, plus ``b1m e_g2``; the fma's rounding is the stored
       value's.
    4. ``v' = fma(b2, v, fp32(fp32(b2m * g2) * g2))``: two product roundings, plus ``b2m (2 |g2| e_g2 + e_g2^2)``.
    5. ``mh = m' / bc1`` and ``vh = v' / bc2`` round once each (twice each on the host tier's SIMD paths, which
       multiply by the rounded reciprocal; the bound counts two); ``sqrt`` once more, with the input error carried by
       ``min(sqrt(e), e / (sqrt(x) + sqrt(x - e)))``; ``+ eps`` once.
    6. ``u = mh / d``: ``(e_mh + |u| e_d) / (d - e_d)`` and one rounding.
    7. AdamW: ``u2 = fma(wd, p, u)``: one rounding.
    8. ``p' = fma(-lr, u2, p)``: ``lr e_u2``, then the stored rounding.

    Each stored value gets one :func:`ulp` of its dtype at ``|ref| + err`` on top (the header's convention).
    ``update=True`` also returns the update ``u2`` and its error (LAMB's trust ratio is formed from it)."""
    pd, sd = dtypes if dtypes is not None else (torch.float32, torch.float32)
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    R = lambda x: U * x.abs() + TINY  # noqa: E731  one rounding of a result of magnitude |x|
    g1 = g * h["gs"]
    e = R(g1)
    if not h["adamw"]:
        g1 = g1 + h["wd"] * p
        e = e + R(h["wd"] * p) + R(g1.abs() + e)
    t1 = h["b1m"] * g1
    m1 = h["b1"] * m + t1
    em = h["b1m"] * e + R(t1.abs() + h["b1m"] * e) + R(h["b1"] * m)
    t2 = h["b2m"] * g1 * g1
    v1 = h["b2"] * v + t2
    ev = h["b2m"] * (2 * g1.abs() * e + e * e) + 2.0001 * R(t2.abs() + h["b2m"] * (2 * g1.abs() * e + e * e)) \
        + R(h["b2"] * v)
    bm = ulp(m1.abs() + em, sd) + em
    bv = ulp(v1.abs() + ev, sd) + ev
    # the moments the update uses are the kernel's fp32 values before the state's rounding: only em, ev
    mh = m1 / h["bc1"]
    emh = em / h["bc1"] + 2.0001 * R(mh.abs() + em / h["bc1"])
    vh = v1 / h["bc2"]
    evh = ev / h["bc2"] + 2.0001 * R(vh + ev / h["bc2"])
    s = vh.sqrt()
    es = _sqrt_err(vh, evh) + R(s + _sqrt_err(vh, evh))
    d = s + h["eps"]
    ed = es + R(d + es)
    u = mh / d
    eu = (emh + u.abs() * ed) / (d - ed).clamp_min(1e-300)
    eu = eu + R(u.abs() + eu)
    if h["adamw"]:
        u = u + h["wd"] * p
        eu = eu + R(h["wd"] * p) + R(u.abs() + eu)
    p1 = p - h["lr"] * u
    ep = h["lr"] * eu + R(h["lr"] * u)
    bp = ulp(p1.abs() + ep, pd) + ep
    if update:
        return p1, m1, v1, bp, bm, bv, u, eu
    return p1, m1, v1, bp, bm, bv


def lion_reference(p, g, m, lr, beta1, beta2, weight_decay, gs, dtypes=None, fused=True):
    """Float64 Lion step of ``lion_flat_kernel`` / ``dsb_cpu_lion`` from the kernel's state, ``gs`` the fp32 gradient
    scale the kernel uses.  Returns ``(p, m, sign, bp, bm)``.

    The sign is exact: ``g1 = fp32(g * gs)`` and ``t = fp32(fp32(1 - b1) * g1)`` are fp32 products (emulated bit for bit
    in fp32), ``b1 m`` is exact in float64 (24 x 24 bits) and the float64 sum ``b1 m + t`` has the sign of the exact sum.
    The fma rounds that sum once to fp32, which keeps its sign unless it underflows to zero (magnitude at most
    ``2**-150``).  ``p' = p (1 - lr wd) - lr sign``: ``1 - lr wd`` rounds up to twice (``U (lr wd + |decay|)``), the
    product once; the subtraction's rounding is the stored one.  ``m' = fma(b2, m, fp32((1 - b2) g1))``: one product
    rounding, then the stored rounding.

    ``fused=False`` is the host tier, which may round ``b1 m`` and ``b2 m`` before the sum: there the sign is only known
    where ``|c|`` exceeds that rounding, elsewhere the bound on p widens by ``2 lr``, and m's bound gets one more ``U``."""
    pd, sd = dtypes if dtypes is not None else (torch.float32, torch.float32)
    b1, b2, lr, wd = f32(beta1), f32(beta2), f32(lr), f32(weight_decay)
    g1 = g.float() * torch.tensor(f32(gs), dtype=torch.float32, device=g.device)
    t = g1 * torch.tensor(f32(1.0 - b1), dtype=torch.float32, device=g.device)
    c = b1 * m.double() + t.double()
    sign = torch.where(c.abs() > TINY, torch.sign(c), 0.0)
    p64 = p.double()
    decay = 1.0 - lr * wd
    p1 = p64 * decay - lr * sign
    e_dec = U * (lr * wd + abs(decay))
    ep = p64.abs() * e_dec + U * (p64 * decay).abs() + 2 * TINY
    t2 = f32(1.0 - b2) * g1.double()
    m1 = b2 * m.double() + t2
    em = U * t2.abs() + TINY
    if not fused:
        ep = ep + torch.where(c.abs() <= U * (b1 * m.double()).abs() + TINY, 2 * lr, 0.0)
        em = em + U * (b2 * m.double()).abs() + TINY
    return p1, m1, sign, ulp(p1.abs() + ep, pd) + ep, ulp(m1.abs() + em, sd) + em


def adagrad_reference(p, g, hsum, lr, eps, weight_decay, gs, pd=torch.float32):
    """Float64 Adagrad step with ``torch.optim.Adagrad``'s formula (``lr_decay = 0``, no initial accumulator):
    ``g' = g gs + wd p``, ``h' = h + g'^2``, ``p' = p - lr g' / (sqrt(h') + eps)``.  Returns ``(p, h, bp, bh)``.

    The kernel rounds ``g gs`` and the fma with ``wd p`` once each, ``h + g'^2`` up to twice (the stored rounding is the
    second), ``lr g'``, the sqrt, ``+ eps`` and the division once each; the subtraction is the stored rounding."""
    lr, eps, wd = f32(lr), f32(eps), f32(weight_decay)
    p, g, hsum = p.double(), g.double(), hsum.double()
    g1 = g * f32(gs)
    e = U * g1.abs() + TINY
    g1 = g1 + wd * p
    e = e + U * (wd * p).abs() + U * (g1.abs() + e) + 2 * TINY
    h1 = hsum + g1 * g1
    eh = 2 * g1.abs() * e + e * e + U * g1 * g1 + TINY
    s = h1.sqrt()
    es = _sqrt_err(h1, eh + U * h1) + U * s + TINY
    d = s + eps
    ed = es + U * (d + es) + TINY
    q = lr * g1 / d
    eq = (lr * e + q.abs() * ed) / (d - ed).clamp_min(1e-300) + 2.0001 * U * q.abs() + 2 * TINY
    p1 = p - q
    return p1, h1, ulp(p1.abs() + eq, pd) + eq, ulp(h1 + eh, torch.float32) + eh


def sgd_reference(p, g, buf, lr, momentum, dampening, weight_decay, nesterov, first, gs, pd=torch.float32):
    """Float64 SGD step with ``torch.optim.SGD``'s semantics: ``d = g gs + wd p``; with momentum the buffer is ``d`` on
    the first step and ``momentum buf + (1 - dampening) d`` after, and the direction is ``d + momentum buf`` (nesterov)
    or ``buf``; ``p' = p - lr d``.  Returns ``(p, buf, bp, bbuf)``; every operation of the kernel rounds at most once
    (``2U`` for ``(1 - dampening) d`` and the fma)."""
    lr, mom, damp, wd = f32(lr), f32(momentum), f32(dampening), f32(weight_decay)
    p, g, buf = p.double(), g.double(), buf.double()
    d = g * f32(gs)
    e = U * d.abs() + TINY
    d = d + wd * p
    e = e + U * (wd * p).abs() + U * (d.abs() + e) + 2 * TINY
    b1, eb = buf, torch.zeros_like(buf)
    if mom != 0.0:
        if first:
            b1, eb = d, e
        else:
            b1 = mom * buf + f32(1.0 - damp) * d
            eb = f32(1.0 - damp) * e + U * f32(1.0 - damp) * (d.abs() + e) + U * (mom * buf).abs() + 2 * TINY
        if nesterov:
            d, e = d + mom * b1, e + mom * eb + U * (mom * b1).abs() + U * (d + mom * b1).abs() + 2 * TINY
        else:
            d, e = b1, eb
    p1 = p - lr * d
    ep = lr * e + U * lr * d.abs() + TINY
    return p1, b1, ulp(p1.abs() + ep, pd) + ep, ulp(b1.abs() + eb, torch.float32) + eb


def sumsq_depth(n, dtype, grid_cap=132 * 4, threads=512):
    """Longest chain of fp32 additions behind ``dsb_sumsq``'s result for ``n`` elements: a thread's grid-stride fma chain
    (vector path, then the scalar tail, or all scalar when misaligned), the block tree (5 warp levels twice), the
    partials' per-thread sum and tree, and the accumulate."""
    per = 4 if dtype == torch.float32 else 8
    grid = max(1, min(-(-(n // 8 + 1) // threads), grid_cap))
    chain = per * -(-(n // per) // (grid * threads)) + -(-n // (grid * threads))
    return chain + 10 + -(-grid // 1024) + 10 + 1


def sumsq_bound(total, n, dtype):
    """Bound on ``|dsb_sumsq(x) - sum(x^2)|`` for a sum of squares ``total`` of ``n`` elements: every term and partial
    sum is non-negative, so ``L`` roundings along the longest chain err by at most ``_rel(L)`` of the total."""
    return _rel(sumsq_depth(n, dtype)) * total + 2 * TINY


def clip_coeff_reference(sumsq, inv_loss_scale, max_norm):
    """Float64 ``(gscale, norm)`` of ``clip_coeff_kernel`` for a finite fp32 ``sumsq``:
    ``norm = sqrt(ss) inv_ls`` and ``gscale = inv_ls min(1, max_norm / (norm + 1e-6))`` (with the fp32 arguments), and
    their relative bounds: sqrt and product round once each (2U), ``norm + 1e-6f``, the division and the last product
    once each, plus ``1e-6f``'s distance from 1e-6."""
    inv, mx = f32(inv_loss_scale), f32(max_norm)
    norm = math.sqrt(sumsq) * inv
    c = inv
    if mx > 0:
        c = inv * min(1.0, mx / (norm + 1e-6))
    rel_norm = 2.0001 * U
    eps_err = abs(f32(1e-6) - 1e-6) / (norm + 1e-6)
    rel_c = (rel_norm + 3.0001 * U + eps_err) if mx > 0 else 0.0
    return c, norm, rel_c, rel_norm


def round_bf16_truncate(x):
    """fp32 -> bf16 by dropping the low 16 bits (round toward zero): the wrong cast a bound check must reject."""
    return (x.float().contiguous().view(torch.int32) & -65536).view(torch.float32).bfloat16()


# ---------------------------------------------------------------------------------------------------------------------
# group quantization (csrc/cuda/quant.cu)
# ---------------------------------------------------------------------------------------------------------------------
# Exact emulations of the kernels' fp32 arithmetic, in numpy float32 (IEEE, subnormals kept, like the kernels built
# without fast-math): a group's scale is ``span / 2^k`` (at least the smallest fp32 subnormal, 1 for an empty range,
# NaN when the group holds a NaN or an inf), codes are ``rint(x * (1/scale))`` through the fp32 reciprocal (a division
# when that overflows), clamped; dequantization is ``fmaf(code, scale, offset)``.  The minifloat formats are defined
# independently: each grid is enumerated from its codes and values are rounded to the nearest grid point in float64.
import numpy as np  # noqa: E402

F32_TINY = np.float32(2.0**-149)  # smallest fp32 subnormal


def _np32(x):
    return x.detach().cpu().float().numpy() if torch.is_tensor(x) else np.asarray(x, dtype=np.float32)


def fmaf(a, b, c):
    """fp32 ``a * b + c`` rounded once (``__fmaf_rn``).  The float64 product of two fp32 values is exact; the float64
    sum is corrected with its exact rounding error (TwoSum) where it lands on an fp32 rounding midpoint."""
    a, b, c = (np.asarray(t, dtype=np.float32).astype(np.float64) for t in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    with np.errstate(invalid="ignore", over="ignore"):
        r = s.astype(np.float32)
        d = s - r.astype(np.float64)
        up = np.nextafter(r, np.float32(np.inf))
        dn = np.nextafter(r, np.float32(-np.inf))
        half_up = (up.astype(np.float64) - r) / 2
        half_dn = (r.astype(np.float64) - dn.astype(np.float64)) / 2
        fix_up = (err > 0) & (d > 0) & (d == half_up)
        fix_dn = (err < 0) & (d < 0) & (-d == half_dn)
    return np.where(fix_up, up, np.where(fix_dn, dn, r)).astype(np.float32)


def to_grid(x, scale):
    """``x / scale`` as the kernels compute it: ``x * (1/scale)`` in fp32, or the division when ``1/scale`` overflows."""
    x, scale = np.asarray(x, np.float32), np.asarray(scale, np.float32)
    with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
        inv = np.float32(1) / scale
        return np.where(np.isfinite(inv), x * inv, x / scale).astype(np.float32)


def group_scale(span, finite, steps):
    """Scale of a group whose range is ``span`` (fp32) over ``steps`` quantization steps."""
    span = np.asarray(span, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        sc = np.where(span > 0, np.maximum(span / np.float32(steps), F32_TINY), np.float32(1)).astype(np.float32)
    return np.where(finite, sc, np.float32(np.nan)).astype(np.float32)


def int_quant_reference(x, groups, bits, sym, rint=np.rint):
    """Emulation of ``quantize_kernel`` / ``fake_quant_kernel``: ``(codes int64 [groups, gs], scale, offset)`` with
    codes in ``[-2^(b-1), 2^(b-1)-1]`` (symmetric) or ``[0, 2^b - 1]`` (asymmetric, before the int8 bias of -128)."""
    g = _np32(x).reshape(groups, -1)
    with np.errstate(invalid="ignore", over="ignore"):
        if sym:
            lo_q, hi_q, steps = -2**(bits - 1), 2**(bits - 1) - 1, 2**(bits - 1)
            span = np.abs(g).max(axis=1)
            offset = np.zeros(groups, np.float32)
        else:
            lo_q, hi_q, steps = 0, 2**bits - 1, 2**bits
            offset = g.min(axis=1)
            span = (g.max(axis=1) - offset).astype(np.float32)
        finite = np.isfinite(span)  # a NaN or an inf in the group, or an asymmetric range beyond fp32
        scale = group_scale(span, finite, steps)
        v = rint(to_grid(g - offset[:, None], scale[:, None]))
        v = np.where(finite[:, None], np.clip(v, lo_q, hi_q), lo_q)  # a non-finite group: its NaN quotient clamps low
    return v.astype(np.int64), scale, offset


def int_dequant_reference(codes, scale, offset=None):
    """fp32 ``fmaf(code, scale, offset)`` per element, like ``dequant_one``."""
    off = np.zeros_like(scale) if offset is None else offset
    return fmaf(codes.astype(np.float32), scale[:, None], off[:, None])


def pack_int(codes, bits, sym):
    """Byte layout of ``quantize``'s codes: int8 (asymmetric biased by -128), or 4-bit nibbles, low nibble first."""
    c = codes.reshape(codes.shape[0], -1)
    if bits == 8:
        return (c if sym else c - 128).astype(np.int8)
    n = c & 0xF
    return (n[:, 0::2] | (n[:, 1::2] << 4)).astype(np.uint8).view(np.int8)


# ---- minifloats ----
FP_FORMATS = {"e4m3": (8, 3), "e5m2": (8, 2), "e3m2": (6, 2), "e2m1": (4, 1), "e4m7": (12, 7)}


def fp_grid(fmt):
    """``(values float64, codes int64)`` of every finite non-negative value of ``fmt``, ascending, by enumerating the
    codes: the hardware FP8 formats through torch's float8 dtypes, the software formats (no inf / NaN codes) from the
    sign / exponent / mantissa fields."""
    bits, m = FP_FORMATS[fmt]
    if bits == 8:
        dt = torch.float8_e4m3fn if m == 3 else torch.float8_e5m2
        vals = torch.arange(128, dtype=torch.uint8).view(dt).double().numpy()
        codes = np.arange(128)
        ok = np.isfinite(vals)
        return vals[ok], codes[ok]
    e = bits - 1 - m
    bias = 2**(e - 1) - 1
    codes = np.arange(2**(bits - 1))
    ef, mf = codes >> m, codes & (2**m - 1)
    vals = np.where(ef == 0, mf * 2.0**(1 - bias - m), (1 + mf * 2.0**-m) * 2.0**(ef.astype(np.float64) - bias))
    return vals, codes


def fp_round(v, fmt, ties_even=None):
    """Codes of fp32 values ``v`` (already divided by the scale) rounded to the nearest ``fmt`` value, saturating at
    the format's maximum: ties to even for FP8 (the hardware conversion), away from zero for the software formats
    (``ties_even`` overrides that).
    The sign bit is the sign of ``v`` (FP8) or ``v < 0`` (software formats, whose encoder never writes -0 for a zero);
    a NaN gives the FP8 NaN code or the maximum."""
    bits, m = FP_FORMATS[fmt]
    vals, codes = fp_grid(fmt)
    v = np.asarray(v, np.float32).astype(np.float64)
    a = np.abs(v)
    nan = np.isnan(a)
    a = np.where(nan, vals[-1], np.minimum(a, vals[-1]))
    lo = np.clip(np.searchsorted(vals, a, side="right") - 1, 0, len(vals) - 1)
    hi = np.minimum(lo + 1, len(vals) - 1)
    dlo, dhi = a - vals[lo], vals[hi] - a
    if ties_even is None:
        ties_even = bits == 8
    tie_hi = (codes[hi] & 1) == 0 if ties_even else np.ones_like(dlo, dtype=bool)
    c = np.where((dhi < dlo) | ((dhi == dlo) & tie_hi & (hi != lo)), codes[hi], codes[lo])
    neg = np.signbit(v) if bits == 8 else (v < 0)
    c = np.where(neg, c | (1 << (bits - 1)), c)
    if bits == 8:
        c = np.where(nan, 0x7F, c)
    return c.astype(np.int64)


def fp_decode(codes, fmt):
    """float64 value of every code (NaN for the FP8 NaN codes)."""
    bits, m = FP_FORMATS[fmt]
    if bits == 8:
        dt = torch.float8_e4m3fn if m == 3 else torch.float8_e5m2
        return torch.from_numpy(np.asarray(codes, np.uint8)).view(dt).double().numpy()
    vals, _ = fp_grid(fmt)
    codes = np.asarray(codes)
    mag = vals[codes & (2**(bits - 1) - 1)]
    return np.where(codes >> (bits - 1), -mag, mag)


def fp_max(fmt):
    return fp_grid(fmt)[0][-1]


def fp_quant_reference(x, groups, fmt):
    """Emulation of ``fp_quantize_kernel`` (round to nearest): ``(codes int64 [groups, gs], scale fp32 [groups])``."""
    g = _np32(x).reshape(groups, -1)
    with np.errstate(invalid="ignore"):
        amax = np.abs(g).max(axis=1)
        scale = group_scale(amax, np.isfinite(amax), np.float32(fp_max(fmt)))
    return fp_round(to_grid(g, scale[:, None]), fmt), scale


def fp_dequant_reference(codes, scale, fmt):
    """fp32 ``decode(code) * scale`` per element."""
    return (fp_decode(codes, fmt).astype(np.float32) * np.asarray(scale, np.float32)[:, None]).astype(np.float32)


def pack_bits(codes, bits):
    """Codes of ``bits`` width written little-endian into one byte stream per group (rows), padded to whole bytes."""
    c = np.asarray(codes, np.int64).reshape(codes.shape[0], -1)
    rows, n = c.shape
    bitarr = ((c[:, :, None] >> np.arange(bits)) & 1).reshape(rows, n * bits)
    pad = (-bitarr.shape[1]) % 8
    bitarr = np.concatenate([bitarr, np.zeros((rows, pad), np.int64)], axis=1)
    return (bitarr.reshape(rows, -1, 8) << np.arange(8)).sum(axis=2).astype(np.uint8)


def quant_cases(groups, gs, dtype, bits, sym, gen, tiny=True):
    """``groups`` groups of ``gs`` values in ``dtype``, the first ones the edges where codecs go wrong, the rest random
    with group magnitudes across 2^-20 .. 2^20 (2^-10 .. 2^10 in fp16):
    0. every value on an exact ``x / scale = k + 1/2`` tie, with +-amax (symmetric) or lo / hi (asymmetric) present;
    1. a constant group (hi == lo); 2. an all-zero group; 3. a negative-only group;
    4. a tiny group (amax about 1e-38, so ``1/scale`` overflows to inf; zeros among it) unless ``tiny`` is false;
    5. a group with a huge (finite) range."""
    x = torch.randn(groups, gs, generator=gen, dtype=torch.float64)
    e = 10 if dtype == torch.float16 else 20
    x *= torch.exp2(torch.randint(-e, e + 1, (groups, 1), generator=gen).double())
    huge = x[min(5, groups - 1)] / x[min(5, groups - 1)].abs().max() * (6e4 if dtype == torch.float16 else 1e36)
    s = 2.0**-3
    half = 2**(bits - 1)
    if sym:
        k = torch.randint(-half, half - 1, (gs, ), generator=gen).double()
        ties = (k + 0.5) * s
        ties[0], ties[-1] = half * s, -half * s
    else:
        k = torch.randint(0, 2 * half - 1, (gs, ), generator=gen).double()
        ties = (k - half + 0.5) * s
        ties[0], ties[-1] = -half * s, half * s
    rows = [ties, torch.full((gs, ), -0.3), torch.zeros(gs), -x[min(3, groups - 1)].abs() - 1.0]
    if tiny:
        t = x[min(4, groups - 1)] / x[min(4, groups - 1)].abs().max() * 1e-38
        t[::3] = 0.0
        rows.append(t)
    rows.append(huge)
    for i, r in enumerate(rows[:groups]):
        x[i] = r
    # + 0 turns the -0s of underflowed values into +0: which of two equal zeros a min reduction keeps is unspecified
    return (x.to(dtype) + 0.0).reshape(-1)


def loco_reference(x, err, groups, bits, beta, reset):
    """Emulation of ``loco_quantize_kernel``: ``comp = x + err``; codes of ``comp``; the error slice becomes
    ``fmaf(beta, err, (1 - beta) * fmaf(-code, scale, comp))`` (0 on reset), and stays as it was in a non-finite
    group.  Returns ``(codes, scale, new err [groups, gs])``."""
    e = _np32(err).reshape(groups, -1)
    comp = (_np32(x).reshape(groups, -1) + e).astype(np.float32)
    codes, scale, _ = int_quant_reference(comp, groups, bits, True)
    b = np.float32(beta)
    if reset:
        upd = np.zeros_like(comp)
    else:
        upd = fmaf(b, e, ((np.float32(1) - b) * fmaf(-codes.astype(np.float32), scale[:, None], comp)).astype(np.float32))
    return codes, scale, np.where(np.isfinite(scale)[:, None], upd, e).astype(np.float32)


def reduce_reference(codes, scale, offset, peers, bits, sym, err=None, err_beta=0.0):
    """Emulation of ``dequant_reduce_kernel`` over input groups ``[peers * out_groups]``: the dequantized chunks summed
    in peer order in fp32, ``fmaf(err_beta, err, sum)``, requantized; the error slice becomes
    ``sum - fmaf(code, scale, offset)`` unless the group is non-finite.  Returns ``(codes, scale, offset, new err)``."""
    deq = int_dequant_reference(codes, scale, offset)
    out_groups = deq.shape[0] // peers
    deq = deq.reshape(peers, out_groups, -1)
    acc = np.zeros(deq.shape[1:], np.float32)
    for k in range(peers):
        acc = (acc + deq[k]).astype(np.float32)
    if err is not None:
        acc = fmaf(np.float32(err_beta), _np32(err).reshape(acc.shape), acc)
    c2, s2, o2 = int_quant_reference(acc, out_groups, bits, sym)
    new = None
    if err is not None:
        new = (acc - int_dequant_reference(c2, s2, o2)).astype(np.float32)
        new = np.where(np.isfinite(s2)[:, None], new, _np32(err).reshape(acc.shape))
    return c2, s2, o2, new


def fp_cases(fmt, groups, gs, gen):
    """Group 0 holds, in units of the scale (its amax is the format maximum, so the scale is 1), every grid value,
    every midpoint (ties), values one fp32 ulp either side of them (the subnormal band and each mantissa rollover into
    the next binade included); group 1 is all zeros, group 2 tiny (amax 1e-38, zeros among it), the rest random
    across 2^-24 .. 2^4 of their amax."""
    vals, _ = fp_grid(fmt)
    mids = ((vals[:-1] + vals[1:]) / 2).astype(np.float32)
    special = np.concatenate([vals.astype(np.float32), mids, np.nextafter(mids, np.float32(0)),
                              np.nextafter(mids, np.float32(np.inf))])
    special = np.concatenate([special, -special])
    x = torch.randn(groups, gs, generator=gen, dtype=torch.float64)
    x *= torch.exp2(torch.randint(-24, 5, (groups, gs), generator=gen).double())
    sp = torch.from_numpy(special).double()
    take = sp[torch.randint(0, sp.numel(), (gs, ), generator=gen)]
    take[:min(gs, sp.numel())] = sp[torch.randperm(sp.numel(), generator=gen)[:gs]]
    take[0] = vals[-1]
    x[0] = take
    x[1] = 0.0
    if groups > 2:
        x[2] = x[2] / x[2].abs().max() * 1e-38
        x[2, ::3] = 0.0
    return x.float().reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------
# ragged inference: paged attention, MoE gating, weight-only quantized GEMMs (csrc/cuda/attention.cu, moe_ragged.cu,
# wq_gemm.cu, wq_tc_gemm.cu)
# ---------------------------------------------------------------------------------------------------------------------
U_OUT = {torch.bfloat16: 2.0**-8, torch.float16: 2.0**-11, torch.float32: U}  # unit roundoff of each storage type


def paged_rows(cache, block_table, seq, n, block_size):
    """``(k, v)`` ``[n, hkv, d]`` in the stored dtype: the first ``n`` cached positions of sequence ``seq``, read through
    its block table (position j lives in block ``block_table[seq, j // block_size]``, slot ``j % block_size``)."""
    j = torch.arange(n, device=cache.device)
    blk = block_table[seq].to(cache.device).long()[j // block_size]
    kv = cache[blk, j % block_size]  # [n, 2, hkv, d]
    return kv[:, 0], kv[:, 1]


def paged_problem(ctx, hq, hkv, d, block_size, dtype, gen, peak=20.0, max_blocks=None, chunk=None):
    """``(qkv, cache, seq_of, pos_of, block_table)`` on ``gen``'s device: a packed qkv batch and a paged cache.  Sequence i
    has ``ctx[i]`` cached positions and one decode token at the last one (with ``chunk[i] = c`` its last c positions are
    query tokens of one prefill chunk, each with its own causal limit).  The blocks are a random permutation of a pool
    with spare blocks, so block tables are permuted and non-contiguous; table entries past a sequence point at real
    blocks but are never read.  q and k are scaled so the largest ``|q.k| / sqrt(d)`` of a token is about ``peak``
    (the max over ~1e3 keys of N(0, a^4) scores is ~3.5 a^2); values are N(0, 1)."""
    dev = gen.device
    need = [-(-c // block_size) for c in ctx]
    pool = sum(need) + 3
    perm = torch.randperm(pool, generator=gen, device=dev).to(torch.int32)
    bt = torch.zeros(len(ctx), max(need) if max_blocks is None else max_blocks, dtype=torch.int32, device=dev)
    o = 0
    for i, n in enumerate(need):
        bt[i, :n] = perm[o:o + n]
        bt[i, n:] = perm[(o + n) % pool]
        o += n
    a = math.sqrt(peak / 3.5)
    cache = torch.randn(pool, block_size, 2, hkv, d, generator=gen, device=dev) * a
    cache[:, :, 1] /= a
    seq_of, pos_of = [], []
    for i, c in enumerate(ctx):
        for p in range(c - (1 if chunk is None else chunk[i]), c):
            seq_of.append(i)
            pos_of.append(p)
    qkv = torch.randn(len(seq_of), (hq + 2 * hkv) * d, generator=gen, device=dev) * a
    i32 = dict(dtype=torch.int32, device=dev)
    return qkv.to(dtype), cache.to(dtype), torch.tensor(seq_of, **i32), torch.tensor(pos_of, **i32), bt


def paged_attention_bounds(q, cache, seq_of, pos_of, block_table, block_size, scale, dtype, nsplit=1, mma=False):
    """``(ref, bound)`` float64 ``[T, hq, d]``: decode attention over the paged cache and a per-element bound on the
    paged-attention kernels' output.  ``q [T, hq, d]`` holds the stored query rows; token t sees the cached keys
    ``[0, pos_of[t]]`` of sequence ``seq_of[t]``; query head h reads kv head ``h // (hq / hkv)``.  ``scale`` is used as
    the fp32 value the kernels receive.  ``nsplit``: KV splits merged at the end; ``mma``: the tensor-core kernel, which
    rounds P to ``dtype`` before ``P V``.

    Per (token, head), with ``x = scale q.k`` over the n visible keys and ``n_s = ceil(n / 4) + nsplit + 8`` bounding the
    sequential fp32 updates any one accumulator sees (each of 4 warps walks a quarter of a split's keys, then the warps and
    the splits are merged):

    1. The score sums d exact products in fp32 (the tensor core may truncate): :func:`gemm_accum_error`.  The CUDA-core
       kernels round ``q * scale`` to fp32 first and the tensor-core kernel rounds ``s * scale`` once: ``2 U scale |q||k|``
       and ``U |x|`` cover either.
    2. ``p = __expf(x - m)`` for a running max m: ex2.approx errs by 2 ulp (``4U``); the subtraction, the product with
       ``log2 e`` and that constant's rounding each move the argument by ``U |x - m|``: ``3U (x_max - x + 2 e_max)``.
       Results below ``2**-126`` flush to zero.
    3. The running max is common to every p and cancels in ``o / l``, but each rescale ``alpha = __expf(m_old - m_new)``
       and the warp and split merges weigh the keys seen before it: ``4U`` and ``3U |dm|`` per factor, the increments of
       the max adding up to the row's span, and the rounding of ``acc * alpha`` and ``l * alpha``: ``(6 n_s + 30) U +
       9U span`` as a relative error of p.
    4. ``o`` and ``l`` sum at most ``n_s + 16`` terms each in fp32 (16 keys per MMA inside the tensor core): ``2 (n_s + 16)
       U`` of ``sum p |v|`` and ``(n_s + 16) U`` of ``sum p``.
    5. The tensor-core kernel rounds p to ``dtype`` for ``P V`` while ``l`` sums the fp32 p: ``u_dtype p |v|``.
    6. ``o / l`` (or ``o * (1 / l)``) rounds at most three times, then once more to ``dtype`` (one :func:`ulp`)."""
    T, hq, d = q.shape
    hkv = cache.shape[3]
    rep = hq // hkv
    c = float(np.float32(scale))
    dev = q.device
    ref = torch.zeros(T, hq, d, dtype=torch.float64, device=dev)
    bnd = torch.zeros_like(ref)
    u_p = U_OUT[dtype] if mma else 0.0
    for t in range(T):
        n = int(pos_of[t]) + 1
        k, v = paged_rows(cache, block_table, int(seq_of[t]), n, block_size)
        n_s = -(-n // 4) + nsplit + 8
        for g in range(hkv):
            K, V = k[:, g].to(dev).double(), v[:, g].to(dev).double()
            Q = q[t, g * rep:(g + 1) * rep].double()  # [rep, d]
            s = Q @ K.t()
            x = c * s
            e_x = c * (gemm_accum_error(Q.abs() @ K.abs().t(), d) + 2 * U * (Q.abs() @ K.abs().t())) + U * x.abs()
            xmax = x.max(-1, keepdim=True).values
            emax = e_x.max(-1, keepdim=True).values
            span = xmax - x.min(-1, keepdim=True).values + 2 * emax
            dist = xmax - x + 2 * emax
            lnrel = e_x + 3 * U * dist + (6 * n_s + 30) * U + 9 * U * span
            P = torch.softmax(x, -1)
            O = P @ V
            Pe = P * torch.expm1(lnrel) + 2.0**-125
            Pw = P + Pe
            aV = V.abs()
            num = Pe @ aV + (u_p + 2 * (n_s + 16) * U) * (Pw @ aV)
            rho = Pe.sum(-1, keepdim=True) + (n_s + 16) * U * Pw.sum(-1, keepdim=True)
            e_pre = (num + O.abs() * rho) / (1 - rho)
            e_o = e_pre + _rel(3) * (O.abs() + e_pre)
            ref[t, g * rep:(g + 1) * rep] = O
            bnd[t, g * rep:(g + 1) * rep] = ulp(O.abs() + e_o, dtype) + e_o
    return ref, bnd


def gating_reference(logits, K, normalize):
    """``(P, bound, order)``: float64 softmax of ``logits [T, E]``, a bound on the kernel's fp32 probabilities and the
    stable descending order of P (ties to the lowest index).

    The kernel forms ``v = __expf(x - max)`` (the subtraction rounds, ``__expf`` errs by ``4U`` plus ``2U |x - max|``
    through its argument), sums the E values in fp32 and multiplies by ``1 / sum`` (two roundings): ``3U |x - max| +
    (E + 8) U`` as a relative error of each probability, plus the ``2**-126`` below which ``__expf`` flushes."""
    x = logits.double()
    P = torch.softmax(x, -1)
    y = (x - x.max(-1, keepdim=True).values).abs()
    y = torch.where(torch.isfinite(y), y, 0.0)  # a -inf logit: p = 0 exactly
    bound = P * torch.expm1(3 * U * y + (logits.shape[1] + 8) * U) + 2.0**-126
    order = torch.sort(P, dim=-1, descending=True, stable=True).indices
    return P, bound, order


def check_gating(ids, w, counts, logits, K, normalize, what="gating"):
    """The exact selection oracle for top-k gating.  For each row and rank r, the chosen expert ``i = ids[r]``:

    * is in range and not chosen at an earlier rank;
    * beats every expert e not chosen by rank r within the bounds: ``P[e] - b[e] <= P[i] + b[i]``;
    * on an exact float64 tie ``P[e] == P[i]`` (equal logits: the kernel computes the same fp32 value), is the lower index.

    Weights lie within the bound of ``P[i]`` (renormalized over the chosen K when ``normalize``: K fp32 adds and a
    division on top), and ``counts`` is exactly the histogram of ``ids``."""
    P, b, _ = gating_reference(logits, K, normalize)
    T, E = P.shape
    ids = ids.long().cpu()
    P, b = P.cpu(), b.cpu()
    assert bool(((ids >= 0) & (ids < E)).all()), f"{what}: id out of range"
    taken = torch.zeros(T, E, dtype=torch.bool)
    rows = torch.arange(T)
    for r in range(K):
        i = ids[:, r]
        assert not bool(taken[rows, i].any()), f"{what}: an expert chosen twice (rank {r})"
        pi, bi = P[rows, i], b[rows, i]
        free = ~taken
        free[rows, i] = False
        beaten = free & ((P - b) > (pi + bi)[:, None])
        tie = free & (P == pi[:, None]) & (torch.arange(E)[None, :] < i[:, None])
        bad = beaten | tie
        if bool(bad.any()):
            t = int(bad.any(-1).nonzero()[0])
            raise AssertionError(f"{what}: row {t} rank {r} chose {int(i[t])} (p={float(pi[t])!r}) over "
                                 f"{bad[t].nonzero().flatten().tolist()[:8]}")
        taken[rows, i] = True
    Wsel = P.gather(1, ids)
    Bsel = b.gather(1, ids)
    if normalize:
        S = Wsel.sum(-1, keepdim=True)
        rel = (Bsel.sum(-1, keepdim=True) / S) + Bsel / Wsel.clamp_min(1e-300)
        ref = Wsel / S
        bound = ref * (torch.expm1(rel + (K + 2) * U)) + 2.0**-126
    else:
        ref, bound = Wsel, Bsel + U * Wsel
    assert_within(w.cpu().double(), ref, bound, f"{what}: weights")
    want = torch.bincount(ids.reshape(-1), minlength=E).to(torch.int32)
    assert torch.equal(counts.cpu(), want), f"{what}: counts"


def wq_codes(mode, N, K, gen, spread=True):
    """Random weight codes ``[N, K]`` of a weight-only format and their float64 values: int8 in [-127, 127], int4 in
    [-8, 7], every e4m3 code but NaN, every e3m2 code."""
    if mode == "int8":
        c = torch.randint(-127, 128, (N, K), generator=gen)
        return c, c.double()
    if mode == "int4":
        c = torch.randint(-8, 8, (N, K), generator=gen)
        return c, c.double()
    fmt = "e4m3" if mode == "fp8" else "e3m2"
    top = 256 if mode == "fp8" else 64
    c = torch.randint(0, top, (N, K), generator=gen)
    if mode == "fp8":
        c = torch.where((c & 0x7F) == 0x7F, c - 1, c)  # no NaN codes
    return c, torch.from_numpy(fp_decode(c.numpy(), fmt))


def wq_pack(codes, mode):
    """Byte layout the kernels read: int8 one byte per code, int4 two's-complement nibbles (low first), e4m3 one byte,
    e3m2 a little-endian 6-bit stream (8 codes in 6 bytes); rows of ``K`` codes."""
    N, K = codes.shape
    c = codes.numpy().astype(np.int64)
    if mode in ("int8", "fp8"):
        return torch.from_numpy((c & 0xFF).astype(np.uint8).view(np.int8).copy())
    if mode == "int4":
        n = c & 0xF
        return torch.from_numpy((n[:, 0::2] | (n[:, 1::2] << 4)).astype(np.uint8).view(np.int8).copy())
    return torch.from_numpy(pack_bits(c.reshape(N, K), 6).view(np.int8).copy())


def wq_bounds(x, wdq, bias, dtype, tile, k_steps, w_round=0.0):
    """``(ref, bound)`` float64 ``[M, N]`` of ``x @ wdq^T + bias`` (``wdq`` the exact float64 dequantized weight) for the
    weight-only GEMMs.  Products of the stored activations and the integer / minifloat codes are exact in fp32.

    * ``tile`` products are summed in fp32 (the tensor core may truncate) before the group scale touches the sum: the
      mma.sync GEMV accumulates each 64 (int8, fp8) or 128 (int4) element chunk into its own tile, ``2 tile U`` of
      ``|x| |W|``;
    * ``k_steps`` more fp32 roundings of the running sum: one ``fmaf(tile, scale, acc)`` per chunk, the 8-warp reduction
      and the bias add for the GEMV, or the wgmma accumulation for the tensor-core GEMM;
    * ``w_round``: the tensor-core GEMM rounds ``code * scale`` to fp32 and then to bf16 before the MMA (``2**-8 + U``
      of every ``|W|``); the GEMV scales in fp32 instead and passes 0;
    * the output's rounding to ``dtype``: one :func:`ulp`."""
    ref = x.double() @ wdq.t()
    if bias is not None:
        ref = ref + bias.double()[None, :]
    mag = x.double().abs() @ wdq.abs().t()
    e = w_round * mag + (2 * tile + k_steps) * U * (1 + w_round) * mag
    if bias is not None:
        e = e + U * (ref.abs() + e)
    return ref, ulp(ref.abs() + e, dtype) + e
