"""CPU tier: the float64 attention reference and the per-element bounds of ``tests/numerics.py`` that the GPU tests hold
the wgmma training attention to.

* The fp32 emulation of the kernels' algorithm (:func:`attention_emulation`) lies inside :func:`attention_bounds` for
  every output, on every data family: the bounds' derivation covers the algorithm's own roundings.
* The bounds have teeth: the emulation of a neighbouring operation -- the window off by one, a document boundary moved
  by a row, the causal diagonal shifted by one, the scale times 1.02, one 64-key block dropped from one 128-row tile --
  falls outside the bounds of the true operation in at least one element.
"""
import math

import pytest
import torch

from tests.numerics import (ATTN_FAMILIES, assert_within, attention_bounds, attention_data, attention_documents,
                            attention_emulation, attention_reference, attention_visible)

# (name, head dim, hq, hkv, document lengths (None: one sequence of S rows), S, causal, window)
CASES = [
    ("dense-causal-d128-gqa3", 128, 6, 2, None, 384, True, None),
    ("dense-full-d64-gqa4", 64, 8, 2, None, 256, False, None),
    ("window65-d64-gqa3", 64, 6, 2, None, 448, True, 65),
    ("window128-d128-gqa4", 128, 4, 1, None, 320, True, 128),
    ("packed-causal-d128-gqa4", 128, 4, 1, [5, 63, 0, 129, 200, 1], None, True, None),
    ("packed-full-d64-gqa4", 64, 8, 2, [77, 0, 128, 65], None, False, None),
    ("packed-window63-d64-gqa3", 64, 6, 2, [1, 64, 130, 200], None, True, 63),
]
OUTS = ("o", "lse", "dq", "dk", "dv")


def _setup(case, family, seed=0):
    name, d, hq, hkv, lens, S, causal, window = case
    cu = None if lens is None else [0] + [sum(lens[:i + 1]) for i in range(len(lens))]
    T = S if lens is None else cu[-1]
    g = torch.Generator().manual_seed(seed + sum(map(ord, name + family)))
    q, k, v, do = attention_data(family, T, hq, hkv, d, g)
    return q, k, v, do, cu, causal, window


def _full_mask(T, cu, causal, window, diag=0):
    """bool ``[T, T]``: the visibility rule inside each document, with the causal diagonal moved by ``diag`` keys."""
    m = torch.zeros(T, T, dtype=torch.bool)
    for s, e in attention_documents(T, cu):
        L = e - s
        if causal:
            i = torch.arange(L)
            diff = i[:, None] - i[None, :] + diag
            vis = diff >= 0
            if window is not None:
                vis = vis & (diff - diag < window)
        else:
            vis = attention_visible(L, False)
        m[s:e, s:e] = vis
    return m


def _drop_block(T, cu, causal, window):
    """The rule with one 64-key block removed from one 128-row tile of the longest document: rows [128, 256) (or
    [0, 128)) lose the first 64-key block any of them sees."""
    m = _full_mask(T, cu, causal, window)
    s, e = max(attention_documents(T, cu), key=lambda se: se[1] - se[0])
    r0 = 128 if e - s > 128 else 0
    rows = slice(s + r0, min(s + r0 + 128, e))
    seen = m[rows, s:e].any(0).nonzero().flatten()
    b0 = s + int(seen[0]) // 64 * 64
    m[rows, b0:b0 + 64] = False
    return m


def _neighbours(case, T, cu):
    """(label, emulation keyword arguments) of the operations next to ``case``."""
    name, d, hq, hkv, lens, S, causal, window = case
    c = 1.0 / math.sqrt(d)
    out = [("scale x1.02", dict(cu_seqlens=cu, causal=causal, window=window, scale=1.02 * c)),
           ("one 64-key block dropped", dict(cu_seqlens=cu, mask=_drop_block(T, cu, causal, window)))]
    if window is not None:
        out.append(("window + 1", dict(cu_seqlens=cu, causal=True, window=window + 1)))
        if window > 1:
            out.append(("window - 1", dict(cu_seqlens=cu, causal=True, window=window - 1)))
    if causal:
        out.append(("diagonal + 1", dict(cu_seqlens=cu, mask=_full_mask(T, cu, True, window, diag=1))))
        out.append(("diagonal - 1", dict(cu_seqlens=cu, mask=_full_mask(T, cu, True, window, diag=-1))))
    if cu is not None:
        inner = [i for i in range(1, len(cu) - 1) if cu[i - 1] < cu[i] < cu[i + 1]]
        for i, step in ((inner[0], 1), (inner[-1], -1)):
            moved = list(cu)
            moved[i] += step
            out.append((f"boundary {cu[i]} {step:+d}", dict(cu_seqlens=moved, causal=causal, window=window)))
    return out


@pytest.mark.parametrize("family", ATTN_FAMILIES)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_emulation_inside_bounds(case, family):
    q, k, v, do, cu, causal, window = _setup(case, family)
    ref, bnd = attention_bounds(q, k, v, do, cu, causal, window)
    emu = attention_emulation(q, k, v, do, cu, causal, window)
    for n in OUTS:
        assert torch.isfinite(bnd[n]).all(), n
        assert_within(emu[n], ref[n], bnd[n], f"{case[0]} {family}: {n}")


@pytest.mark.parametrize("family", ["diffuse", "peaked"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_bounds_reject_neighbouring_operations(case, family):
    q, k, v, do, cu, causal, window = _setup(case, family)
    T = q.shape[0]
    ref, bnd = attention_bounds(q, k, v, do, cu, causal, window)
    for label, kw in _neighbours(case, T, cu):
        emu = attention_emulation(q, k, v, do, **kw)
        rejected = [n for n in OUTS if not bool(((emu[n].double() - ref[n]).abs() <= bnd[n]).all())]
        assert rejected, f"{case[0]} {family}: the bounds accept the emulation of '{label}'"


def test_reference_matches_autograd():
    """The explicit backward formulas equal autograd through a float64 softmax, GQA and documents included."""
    case = CASES[-1]
    q, k, v, do, cu, causal, window = _setup(case, "diffuse")
    ref = attention_reference(q, k, v, do, cu, causal, window)
    T, hq, d = q.shape
    rep = hq // k.shape[1]
    x = [t.double().requires_grad_(True) for t in (q, k, v)]
    o = torch.zeros(T, hq, d, dtype=torch.float64)
    lse = torch.zeros(hq, T, dtype=torch.float64)
    for s, e in attention_documents(T, cu):
        vis = attention_visible(e - s, causal, window)
        kk, vv = (t[s:e].repeat_interleave(rep, 1) for t in x[1:])
        sc = torch.einsum("qhd,khd->hqk", x[0][s:e], kk) / math.sqrt(d)
        sc = sc.masked_fill(~vis, -math.inf)
        o = o.index_put((torch.arange(s, e), ), torch.einsum("hqk,khd->qhd", torch.softmax(sc, -1), vv))
        lse = lse.index_put((torch.arange(hq)[:, None], torch.arange(s, e)[None, :]), torch.logsumexp(sc, -1))
    o.backward(do.double())
    for n, want in (("o", o), ("lse", lse), ("dq", x[0].grad), ("dk", x[1].grad), ("dv", x[2].grad)):
        torch.testing.assert_close(ref[n], want.detach(), rtol=1e-12, atol=1e-12, msg=n)


def test_kv_heads_subset():
    """Only the listed kv groups are computed; the others have reference 0 and bound inf, and the computed ones equal
    the full computation."""
    case = CASES[0]
    q, k, v, do, cu, causal, window = _setup(case, "peaked")
    full = attention_reference(q, k, v, do, cu, causal, window)
    ref, bnd = attention_bounds(q, k, v, do, cu, causal, window, kv_heads=[1])
    hq, hkv = q.shape[1], k.shape[1]
    rep = hq // hkv
    assert torch.equal(ref["o"][:, rep:], full["o"][:, rep:]) and torch.equal(ref["dk"][:, 1], full["dk"][:, 1])
    assert bool((ref["o"][:, :rep] == 0).all()) and bool(torch.isinf(bnd["dv"][:, 0]).all())
