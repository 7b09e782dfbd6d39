"""GPU tier: the wgmma training attention (``csrc/cuda/attn_sm90.cu``) checked per element, through
``attention_sm100.fwd / bwd / fwd_varlen / bwd_varlen``.

* exact selection oracle -- every query scores one visible key (its target) ``16 d`` above any other, so every other
  ``ex2`` is exactly 0 and the target's P is exactly 1: O is bit-equal to the target's V row, the LSE is the target's
  scaled score, and on grid data dS is exactly 0 and dV is the exact sum of the dO rows that select each key;
* rows that see one key (window 1, and row 0 of a causal sequence) are exact the same way;
* bounded -- random data of four families against float64 with :func:`tests.numerics.attention_bounds`, at the
  modes, edge lengths and windows where kernels go wrong and at the Llama / Mistral training shapes, where the kernel's
  error is also held to twice the error of the algorithm's own fp32 emulation;
* masks hold bit for bit: future keys and rows past the end change nothing they must not;
* layouts: separate q / k / v with their own row strides, outputs inside NaN guard bands, a strided ``d_o``;
* every refusal of the four entry points raises and writes nothing.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from deepspeed_b200.ops.kernels import attention_sm100 as A
from deepspeed_b200.ops.native import NativeOpError
from tests.numerics import (ATTN_FAMILIES, U, assert_attention_bounded, assert_bits_equal, attention_bounds,
                            attention_data, attention_documents, attention_emulation, exact_grid)

pytestmark = pytest.mark.gpu

NAN = float("nan")
BF16 = torch.bfloat16
# document lengths on both sides of the 64-key and 128-row tile edges, with empty documents between them
EDGE_LENS = [1, 0, 63, 64, 65, 0, 127, 128, 129, 0]
RAGGED = [5, 1, 63, 64, 65, 0, 127, 128, 129, 200, 1000, 0]


def _gen(*seed):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(seed).encode()))


def _cu_list(lens):
    return [0] + np.cumsum(lens).tolist()


def _packed_lengths(seed, rows=2, row_len=4096, lo=16, hi=4096):
    """Document lengths drawn from [lo, hi] and cut to fill ``rows`` rows of ``row_len`` tokens."""
    rng = np.random.default_rng(seed)
    lens = []
    for _ in range(rows):
        left = row_len
        while left:
            n = min(int(rng.integers(lo, hi + 1)), left)
            lens.append(n)
            left -= n
    return lens


def _cols(buf, hq, hkv, d):
    return buf[:, :hq * d], buf[:, hq * d:(hq + hkv) * d], buf[:, (hq + hkv) * d:]


def _run(q, k, v, do=None, cu=None, B=1, causal=True, window=None, scale=None):
    """q [T, hq, d], k / v [T, hkv, d] as columns of one packed buffer through the dense (``cu`` None: B sequences of
    T / B rows) or varlen entry points, and the backward for ``do``.  Returns ``o [T, hq, d]``, ``lse [hq, T]`` and
    ``dq``, ``dk``, ``dv`` written into a NaN-filled packed buffer."""
    T, hq, d = q.shape
    hkv = k.shape[1]
    buf = torch.cat([q.reshape(T, -1), k.reshape(T, -1), v.reshape(T, -1)], 1)
    q2, k2, v2 = _cols(buf, hq, hkv, d)
    kw = dict(causal=causal, window=window, scale=scale, head_dim=d)
    if cu is None:
        S = T // B
        o, lse = A.fwd(q2, k2, v2, B, S, hq, hkv, **kw)
        lse_t = lse.permute(1, 0, 2).reshape(hq, T)
    else:
        cu_t = torch.tensor(cu, dtype=torch.int32, device="cuda")
        ms = max(1, max(e - s for s, e in zip(cu[:-1], cu[1:])))
        o, lse = A.fwd_varlen(q2, k2, v2, cu_t, ms, hq, hkv, **kw)
        lse_t = lse
    out = {"o": o.unflatten(1, (hq, d)), "lse": lse_t}
    if do is not None:
        g = torch.full_like(buf, NAN)
        dq, dk, dv = _cols(g, hq, hkv, d)
        d_o = do.reshape(T, -1)
        if cu is None:
            A.bwd(d_o, q2, k2, v2, o, lse, B, S, hq, hkv, dq=dq, dk=dk, dv=dv, **kw)
        else:
            A.bwd_varlen(d_o, q2, k2, v2, o, lse, cu_t, ms, hq, hkv, dq=dq, dk=dk, dv=dv, **kw)
        out.update(dq=dq.unflatten(1, (hq, d)), dk=dk.unflatten(1, (hkv, d)), dv=dv.unflatten(1, (hkv, d)))
    return out


def _seq_cu(T, B):
    """The dense batch's sequences as documents for the reference."""
    return None if B == 1 else [i * (T // B) for i in range(B + 1)]


# ---- (a) exact selection oracle --------------------------------------------------------------------------------------------
def _hadamard(n):
    h = torch.ones(1, 1)
    while h.shape[0] < n:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)], 0)
    return h


def _selection(lens, hq, hkv, d, causal, window, seed):
    """Codes, queries and targets of the selection oracle.  Key at position p of its document carries
    ``[H[p // n], H[p % n]]`` (``n = d / 2``); query (i, h) is ``32 code(t)`` for a target t drawn among its visible keys,
    a different draw for every head.  Returns ``(q, k, targets [T, hq])``."""
    n = d // 2
    H = _hadamard(n).cuda()
    T = sum(lens)
    pos = torch.cat([torch.arange(L) for L in lens]).cuda()
    codes = torch.cat([H[pos // n], H[pos % n]], 1)  # [T, d]
    k = codes[:, None, :].expand(T, hkv, d).bfloat16()
    rng = np.random.default_rng(seed)
    tgt = np.zeros((T, hq), dtype=np.int64)
    for s, e in attention_documents(T, _cu_list(lens)):
        for i in range(e - s):
            lo = max(0, i - window + 1) if window is not None else 0
            hi = i if causal else e - s - 1
            tgt[s + i] = s + rng.integers(lo, hi + 1, size=hq)
    tgt = torch.from_numpy(tgt).cuda()
    q = (32 * codes[tgt]).bfloat16()  # [T, hq, d]
    return q, k, tgt


SELECT = [  # (name, head dim, hq, hkv, lens, B (dense) or None (packed), causal, window)
    ("dense-causal", 128, 6, 2, [512, 512], 2, True, None),
    ("dense-causal", 64, 6, 2, [512, 512], 2, True, None),
    ("dense-full", 128, 4, 1, [384], 1, False, None),
    ("dense-full", 64, 8, 2, [256, 256], 2, False, None),
    ("dense-window65", 128, 6, 2, [512, 512], 2, True, 65),
    ("dense-window1000", 64, 6, 2, [1024], 1, True, 1000),
    ("packed-causal", 128, 6, 2, RAGGED, None, True, None),
    ("packed-causal", 64, 8, 2, RAGGED, None, True, None),
    ("packed-full", 128, 4, 2, RAGGED, None, False, None),
    ("packed-full", 64, 6, 2, RAGGED, None, False, None),
    ("packed-window63", 128, 6, 2, RAGGED, None, True, 63),
    ("packed-window128", 64, 6, 2, RAGGED, None, True, 128),
    ("llama3.2-3b-packed", 128, 24, 8, _packed_lengths(0), None, True, None),
    ("llama3.2-1b-packed", 64, 32, 8, _packed_lengths(1, hi=1024), None, True, None),
]


@pytest.mark.parametrize("case", SELECT, ids=[f"{c[0]}-d{c[1]}-{c[2]}x{c[3]}" for c in SELECT])
def test_selection_oracle_is_exact(case):
    name, d, hq, hkv, lens, B, causal, window = case
    T = sum(lens)
    rep = hq // hkv
    q, k, tgt = _selection(lens, hq, hkv, d, causal, window, zlib.crc32(name.encode()) + d)
    g = _gen("select", name, d)
    v = exact_grid(T, hkv * d, g, emin=-2, emax=2)[0].view(T, hkv, d)  # distinct per kv head
    do = exact_grid(T, hq * d, g, emin=-2, emax=2)[0].view(T, hq, d)
    out = _run(q, k, v, do, cu=None if B else _cu_list(lens), B=B or 1, causal=causal, window=window)
    kv_of = torch.arange(hq, device="cuda") // rep
    assert_bits_equal(out["o"], v[tgt, kv_of[None, :]], f"{name} O")
    want_lse = torch.full((hq, T), 32.0 * d / math.sqrt(d), dtype=torch.float64, device="cuda")
    err = (out["lse"].double() - want_lse).abs()
    assert float(err.max()) <= math.expm1(6 * math.log1p(U)) * float(want_lse.max()), (name, float(err.max()))
    dv = torch.zeros(T, hkv, d, dtype=torch.float64, device="cuda")
    for h in range(hq):
        dv[:, h // rep].index_add_(0, tgt[:, h], do[:, h].double())
    assert_bits_equal(out["dv"], dv.to(BF16), f"{name} dV")
    for n in ("dq", "dk"):
        assert bool((out[n] == 0).all()), f"{name} {n}: {int((out[n] != 0).sum())} nonzero elements"


# ---- (b) rows with one visible key -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("lens,B", [([256, 256], 2), (RAGGED, None)], ids=["dense", "packed"])
def test_window_one_is_exact(d, lens, B):
    """Window 1: every row sees only its own key, so O = V, dQ = dK = 0 and dV is the sum of dO over the group."""
    hq, hkv = 6, 2
    T = sum(lens)
    g = _gen("w1", d, B)
    q, k, _, _ = attention_data("peaked", T, hq, hkv, d, g)
    v = exact_grid(T, hkv * d, g, emin=-2, emax=2)[0].view(T, hkv, d)
    do = exact_grid(T, hq * d, g, emin=-2, emax=2)[0].view(T, hq, d)
    out = _run(q, k, v, do, cu=None if B else _cu_list(lens), B=B or 1, causal=True, window=1)
    assert_bits_equal(out["o"], v.repeat_interleave(hq // hkv, 1), "O")
    assert_bits_equal(out["dv"], do.double().unflatten(1, (hkv, hq // hkv)).sum(2).to(BF16), "dV")
    for n in ("dq", "dk"):
        assert bool((out[n] == 0).all()), n


@pytest.mark.parametrize("d", [64, 128])
def test_first_row_of_every_causal_document_is_exact(d):
    hq, hkv = 8, 2
    lens = RAGGED
    T = sum(lens)
    g = _gen("row0", d)
    q, k, _, _ = attention_data("diffuse", T, hq, hkv, d, g)
    v = exact_grid(T, hkv * d, g, emin=-2, emax=2)[0].view(T, hkv, d)
    do = exact_grid(T, hq * d, g, emin=-2, emax=2)[0].view(T, hq, d)
    out = _run(q, k, v, do, cu=_cu_list(lens), causal=True)
    first = torch.tensor([s for s, _ in attention_documents(T, _cu_list(lens))], device="cuda")
    assert_bits_equal(out["o"][first], v[first].repeat_interleave(hq // hkv, 1), "O")
    assert bool((out["dq"][first] == 0).all())


# ---- (c) per-element bounds ------------------------------------------------------------------------------------------------
MODES = {  # name: (lens, B (dense) or None (packed), causal, window, hq, hkv)
    "dense-causal": ([512, 512], 2, True, None, 6, 2),
    "dense-full": ([384], 1, False, None, 8, 2),
    "packed-causal": (RAGGED, None, True, None, 6, 2),
    "packed-full": (RAGGED, None, False, None, 8, 2),
    "window-dense": ([512, 512], 2, True, 65, 6, 2),
    "window-packed": (RAGGED, None, True, 127, 8, 2),
}


def _bounded(family, lens, B, causal, window, hq, hkv, d, scale=None, kv_heads=None, seed=0):
    T = sum(lens)
    q, k, v, do = attention_data(family, T, hq, hkv, d, _gen(family, tuple(lens), B, window, hq, hkv, d, seed))
    cu = _seq_cu(T, B) if B else _cu_list(lens)
    out = _run(q, k, v, do, cu=None if B else cu, B=B or 1, causal=causal, window=window, scale=scale)
    worst = assert_attention_bounded(out, q, k, v, do, cu, causal, window, scale, kv_heads)
    print(f"\n[err/bound] {family} d={d} lens={len(lens)} B={B} causal={causal} window={window} scale={scale}: "
          f"{ {n: round(x, 3) for n, x in worst.items()} }")
    return q, k, v, do, cu, out, worst


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("family", ATTN_FAMILIES)
def test_bounded_on_random_data(family, mode, d):
    lens, B, causal, window, hq, hkv = MODES[mode]
    _bounded(family, lens, B, causal, window, hq, hkv, d)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("window", [1, 63, 64, 65, 127, 128, 129, 256, 5000])
def test_bounded_at_edge_windows(window, d):
    _bounded("peaked", [256, 256], 2, True, window, 6, 2, d)
    _bounded("peaked", EDGE_LENS + [200], None, True, window, 6, 2, d)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
def test_bounded_at_edge_document_lengths(causal, d):
    lens = EDGE_LENS + ([4096] if d == 128 else [1024])
    _bounded("peaked", lens, None, causal, None, 4, 1, d)


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("S", [77, 200, 1000])
@pytest.mark.parametrize("causal", [True, False])
def test_bounded_ragged_dense_forward(S, causal, d):
    """B = 1 with S not a multiple of 128: the forward masks the ragged last block (the backward needs S % 128 = 0)."""
    hq, hkv = 6, 2
    q, k, v, _ = attention_data("diffuse", S, hq, hkv, d, _gen("ragged", S, causal, d))
    out = _run(q, k, v, None, B=1, causal=causal)
    assert_attention_bounded(out, q, k, v, None, None, causal)


@pytest.mark.parametrize("d", [64, 128])
def test_bounded_with_a_non_default_scale(d):
    for scale in (0.05, 0.3):
        _bounded("diffuse", [256, 256], 2, True, None, 4, 2, d, scale=scale)
        _bounded("peaked", RAGGED, None, True, 100, 4, 2, d, scale=scale)


# ---- (c) + (d) training shapes: bounds, and the kernel's error against the emulation's --------------------------------------
TRAINING = {  # name: (head dim, hq, hkv, lens, B (dense) or None (packed), window)
    "llama3.2-3b-dense": (128, 24, 8, [4096, 4096], 2, None),
    "llama3.2-3b-packed": (128, 24, 8, _packed_lengths(0), None, None),
    "llama3.2-1b-packed": (64, 32, 8, _packed_lengths(1), None, None),
    "mistral-7b-window4096": (128, 32, 8, [4096], 1, 4096),
    "mistral-7b-window1024": (128, 32, 8, [4096], 1, 1024),
    "gqa64x8": (128, 64, 8, [512, 512], 2, None),
}
KV_CHECKED = [0, 7]  # the float64 reference runs on the first and last GQA groups


def _error_ratio(out, emu, ref, cu, T, heads_of):
    """max over (sequence, head) of kernel / emulation for the RMS and the max error against float64."""
    rms, mx = 0.0, 0.0
    for s, e in attention_documents(T, cu):
        for h in heads_of:
            ek = (out[s:e, h].double() - ref[s:e, h]).abs()
            ee = (emu[s:e, h].double() - ref[s:e, h]).abs()
            if float(ee.max()) == 0.0:
                assert float(ek.max()) == 0.0
                continue
            rms = max(rms, float(ek.pow(2).mean().sqrt() / ee.pow(2).mean().sqrt()))
            mx = max(mx, float(ek.max() / ee.max()))
    return rms, mx


@pytest.mark.parametrize("shape", list(TRAINING))
def test_training_shape_bounded_and_no_worse_than_the_algorithm(shape):
    d, hq, hkv, lens, B, window = TRAINING[shape]
    rep = hq // hkv
    q, k, v, do, cu, out, worst = _bounded("diffuse", lens, B, True, window, hq, hkv, d, kv_heads=KV_CHECKED)
    T = q.shape[0]
    ref, _ = attention_bounds(q, k, v, do, cu, True, window, None, KV_CHECKED)
    emu = attention_emulation(q, k, v, do, cu, True, window)
    qh = [h for g in KV_CHECKED for h in range(g * rep, (g + 1) * rep)]
    ratios = {}
    for n, heads in (("o", qh), ("dq", qh), ("dk", KV_CHECKED), ("dv", KV_CHECKED)):
        ratios[n] = _error_ratio(out[n], emu[n], ref[n], cu, T, heads)
    ratios["lse"] = _error_ratio(out["lse"].t(), emu["lse"].t(), ref["lse"].t(), cu, T, qh)
    print(f"\n{shape}: err/bound {worst}; kernel/emulation (rms, max) {ratios}")
    for n, (rms, mx) in ratios.items():
        assert rms <= 2.0 and mx <= 2.0, (shape, n, rms, mx)


# ---- (e) masks hold exactly -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("window", [None, 100])
def test_future_keys_change_nothing_before_them(d, window):
    """K / V rows >= r of every sequence get large finite values: rows < r of O, LSE and dQ do not change by a bit."""
    B, S, hq, hkv = 2, 512, 6, 2
    T = B * S
    q, k, v, do = attention_data("diffuse", T, hq, hkv, d, _gen("future", d, window))
    base = _run(q, k, v, do, B=B, causal=True, window=window)
    for r in (63, 64, 65, 127, 128, 129, 191, 256):
        k2, v2 = k.clone(), v.clone()
        for b in range(B):
            k2[b * S + r:(b + 1) * S] = 12.0
            v2[b * S + r:(b + 1) * S] = 3000.0
        got = _run(q, k2, v2, do, B=B, causal=True, window=window)
        keep = (torch.arange(T, device="cuda") % S) < r
        for n in ("o", "dq"):
            assert_bits_equal(got[n][keep], base[n][keep], f"r={r} {n}")
        assert_bits_equal(got["lse"][:, keep], base["lse"][:, keep], f"r={r} lse")
        assert not torch.equal(got["o"][~keep], base["o"][~keep])


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
def test_rows_past_the_end_change_nothing(d, causal):
    """The varlen forms over T rows (T not a multiple of 64) and the dense forward at B = 1 read and write no row past T:
    the operands are views of buffers with more rows, and what those rows hold changes no result."""
    hq, hkv = 4, 2
    lens = [5, 64, 0, 130]
    T = sum(lens)  # 199
    q, k, v, do = attention_data("diffuse", T, hq, hkv, d, _gen("past", d, causal))
    cols = (hq + 2 * hkv) * d
    results = []
    for fill in (0.0, 3000.0, NAN):
        buf = torch.full((T + 77, cols), fill, dtype=BF16, device="cuda")
        buf[:T] = torch.cat([q.reshape(T, -1), k.reshape(T, -1), v.reshape(T, -1)], 1)
        dob = torch.full((T + 77, hq * d), fill, dtype=BF16, device="cuda")
        dob[:T] = do.reshape(T, -1)
        q2, k2, v2 = _cols(buf[:T], hq, hkv, d)
        cu = torch.tensor(_cu_list(lens), dtype=torch.int32, device="cuda")
        o = torch.full((T + 77, hq * d), NAN, dtype=BF16, device="cuda")
        _, lse = A.fwd_varlen(q2, k2, v2, cu, max(lens), hq, hkv, causal=causal, out=o[:T], head_dim=d)
        g = torch.full((T + 77, cols), NAN, dtype=BF16, device="cuda")
        dq, dk, dv = _cols(g[:T], hq, hkv, d)
        A.bwd_varlen(dob[:T], q2, k2, v2, o[:T], lse, cu, max(lens), hq, hkv, causal=causal, dq=dq, dk=dk, dv=dv,
                     head_dim=d)
        od = torch.full((T + 77, hq * d), NAN, dtype=BF16, device="cuda")
        _, lse_d = A.fwd(q2, k2, v2, 1, T, hq, hkv, causal=causal, out=od[:T], head_dim=d)
        assert bool(o[T:].isnan().all()) and bool(g[T:].isnan().all()) and bool(od[T:].isnan().all())
        assert bool(torch.isfinite(o[:T].float()).all()) and bool(torch.isfinite(g[:T].float()).all())
        results.append((o[:T], lse, g[:T], od[:T], lse_d))
    for other in results[1:]:
        for a, b in zip(results[0], other):
            assert_bits_equal(a, b, "rows past T")


# ---- (f) layouts -------------------------------------------------------------------------------------------------------------
def _guarded(rows, cols, r0=3, c0=8, extra=16):
    """A NaN buffer with guard rows and columns around a ``[rows, cols]`` view (row stride ``cols + c0 + extra``)."""
    buf = torch.full((rows + 2 * r0, cols + c0 + extra), NAN, dtype=BF16, device="cuda")
    return buf, buf[r0:r0 + rows, c0:c0 + cols]


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("packed", [False, True])
def test_layouts_are_bit_identical(d, packed):
    """Separate q / k / v tensors with different row strides, O / dQ / dK / dV inside NaN guard bands and a strided
    ``d_o`` give the bits of the packed-buffer run; the guards stay NaN; relaunches are bit-identical."""
    hq, hkv = 6, 2
    lens = [512, 512] if not packed else RAGGED
    T = sum(lens)
    q, k, v, do = attention_data("peaked", T, hq, hkv, d, _gen("layout", d, packed))
    cu = _cu_list(lens)
    B = None if packed else 2
    base = _run(q, k, v, do, cu=cu if packed else None, B=B or 1)
    again = _run(q, k, v, do, cu=cu if packed else None, B=B or 1)
    for n in base:
        assert_bits_equal(again[n], base[n], f"relaunch {n}")
    ops = []
    for x, extra in ((q, 8), (k, 24), (v, 64)):
        buf, view = _guarded(T, x.shape[1] * d, extra=extra)
        view.copy_(x.reshape(T, -1))
        ops.append(view)
    ob, o = _guarded(T, hq * d, extra=40)
    dob, d_o = _guarded(T, hq * d, extra=8)
    d_o.copy_(do.reshape(T, -1))
    grads = [_guarded(T, c * d, extra=e) for c, e in ((hq, 16), (hkv, 32), (hkv, 48))]
    kw = dict(causal=True, head_dim=d)
    if packed:
        cu_t = torch.tensor(cu, dtype=torch.int32, device="cuda")
        _, lse = A.fwd_varlen(*ops, cu_t, max(lens), hq, hkv, out=o, **kw)
        A.bwd_varlen(d_o, *ops, o, lse, cu_t, max(lens), hq, hkv, dq=grads[0][1], dk=grads[1][1], dv=grads[2][1], **kw)
    else:
        _, lse_b = A.fwd(*ops, 2, T // 2, hq, hkv, out=o, **kw)
        A.bwd(d_o, *ops, o, lse_b, 2, T // 2, hq, hkv, dq=grads[0][1], dk=grads[1][1], dv=grads[2][1], **kw)
        lse = lse_b.permute(1, 0, 2).reshape(hq, T)
    assert_bits_equal(o, base["o"].reshape(T, -1), "O")
    assert_bits_equal(lse, base["lse"], "LSE")
    for (buf, view), n in zip(grads, ("dq", "dk", "dv")):
        assert_bits_equal(view, base[n].reshape(T, -1), n)
    for buf, view in [(ob, o)] + grads:
        inside = torch.zeros_like(buf, dtype=torch.bool)
        inside[3:3 + T, 8:8 + view.shape[1]] = True
        assert bool(buf[~inside].isnan().all()), "a guard was written"
        assert not bool(view.isnan().any()), "an output element was left unwritten"


# ---- (g) refusals --------------------------------------------------------------------------------------------------------------
def _refusal(kind, T, hq, hkv, d, B=1, causal=True, window=None, head_dim=None, n_docs=1, shift=None, ld_extra=None):
    """``(outputs, launch)`` for one entry point: NaN-filled outputs and a call that writes them.  ``shift = (name, n)``
    moves that operand's pointer by n elements, ``ld_extra = (name, n)`` adds n elements to its row stride."""
    hd = head_dim or d
    g = _gen("refuse", T, hq, hkv, d)

    def operand(name, cols, fill=None):
        off = shift[1] if shift and shift[0] == name else 0
        ld = cols + (ld_extra[1] if ld_extra and ld_extra[0] == name else 0)
        store = torch.full((T * ld + off + 64, ), NAN, dtype=BF16, device="cuda")
        x = store[off:off + T * ld].view(T, ld)[:, :cols]
        if fill == "randn":
            x.copy_(torch.randn(T, cols, device="cuda", generator=g) * 0.5)
        elif fill is not None:
            x.fill_(fill)
        return x

    q, k, v = operand("q", hq * d, "randn"), operand("k", hkv * d, "randn"), operand("v", hkv * d, "randn")
    cu = torch.tensor([0] * n_docs + [T], dtype=torch.int32, device="cuda")
    kw = dict(causal=causal, window=window, head_dim=hd)
    if kind.startswith("fwd"):
        o = operand("o", hq * hd)
        if kind == "fwd":
            return [o], lambda: A.fwd(q, k, v, B, T // B, hq, hkv, out=o, **kw)
        return [o], lambda: A.fwd_varlen(q, k, v, cu, T, hq, hkv, out=o, **kw)
    o, d_o = operand("o", hq * d, 0.0), operand("do", hq * d, 1.0)
    lse = torch.zeros(B, hq, T // B, dtype=torch.float32, device="cuda")
    dq, dk, dv = operand("dq", hq * hd), operand("dk", hkv * hd), operand("dv", hkv * hd)
    if kind == "bwd":
        return [dq, dk, dv], lambda: A.bwd(d_o, q, k, v, o, lse, B, T // B, hq, hkv, dq=dq, dk=dk, dv=dv, **kw)
    return [dq, dk, dv], lambda: A.bwd_varlen(d_o, q, k, v, o, lse.view(hq, T), cu, T, hq, hkv, dq=dq, dk=dk, dv=dv,
                                              **kw)


ALL = ("fwd", "fwd_varlen", "bwd", "bwd_varlen")
BWD = ("bwd", "bwd_varlen")
REFUSALS = [  # (label, entry points, keyword arguments of _refusal)
    ("head-dim-96", ALL, dict(head_dim=96)),
    ("hq-3-hkv-2", ALL, dict(hq=3, hkv=2)),
    ("q-row-stride", ALL, dict(ld_extra=("q", 4))),
    ("v-row-stride", ALL, dict(ld_extra=("v", 4))),
    ("o-row-stride", ALL, dict(ld_extra=("o", 4))),
    ("do-row-stride", BWD, dict(ld_extra=("do", 4))),
    ("dq-row-stride", BWD, dict(ld_extra=("dq", 4))),
    ("dk-row-stride", BWD, dict(ld_extra=("dk", 4))),
    ("dv-row-stride", BWD, dict(ld_extra=("dv", 4))),
    ("misaligned-q", ALL, dict(shift=("q", 4))),
    ("misaligned-k", ALL, dict(shift=("k", 4))),
    ("misaligned-o", ALL, dict(shift=("o", 4))),
    ("misaligned-do", BWD, dict(shift=("do", 4))),
    ("misaligned-dq", BWD, dict(shift=("dq", 4))),
    ("misaligned-dk", BWD, dict(shift=("dk", 2))),
    ("misaligned-dv", BWD, dict(shift=("dv", 1))),
    ("batch-2-S-100", ("fwd", "bwd"), dict(B=2, T=200)),
    ("window-without-causal", ALL, dict(causal=False, window=64)),
    ("n-docs-65536", ("fwd_varlen", "bwd_varlen"), dict(n_docs=65536)),
]


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("label,kinds,kw", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals_raise_and_write_nothing(label, kinds, kw, d, monkeypatch):
    # the Python wrapper rejects a window without causal itself: let the entry point see it
    monkeypatch.setattr(A, "_window", lambda window, causal: 0 if window is None else int(window))
    kw = dict(kw)
    hq, hkv, T = kw.pop("hq", 4), kw.pop("hkv", 2), kw.pop("T", 256)
    for kind in kinds:
        outs, launch = _refusal(kind, T, hq, hkv, d, **kw)
        with pytest.raises(NativeOpError):
            launch()
        torch.cuda.synchronize()
        for x in outs:
            assert bool(x.isnan().all()), f"{kind}: an output was written"


@pytest.mark.parametrize("kind", ALL)
def test_refusal_setup_runs_when_nothing_is_wrong(kind):
    """The refusal test's operands launch and write every output when no condition is broken."""
    outs, launch = _refusal(kind, 256, 4, 2, 128)
    launch()
    torch.cuda.synchronize()
    for x in outs:
        assert not bool(x.isnan().any())
