"""The ragged-inference CUDA per element: the three paged-attention kernels and their split-KV merge against a float64
reference with a bound built from the kernels' arithmetic (``tests/numerics.py``), KV append / embedding / row gather
bit for bit, top-k gating against an exact selection oracle, MoE routing exactly, and the weight-only quantized GEMV,
wgmma GEMM and its grouped MoE form against float64 with per-element bounds.  Every output is written into a buffer with
sentinel guard bands."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import numerics as R
from deepspeed_b200.ops import native as N
from deepspeed_b200.ops.kernels import moe_ops as M
from deepspeed_b200.ops.kernels import ragged_ops as RO

pytestmark = pytest.mark.gpu

GUARD = 256


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


class Guarded:
    """A ``shape`` tensor inside a sentinel-filled buffer with ``GUARD`` elements on each side."""

    def __init__(self, shape, dtype, sentinel=-1234.5):
        n = math.prod(shape)
        self.buf = torch.full((n + 2 * GUARD, ), sentinel, dtype=dtype, device="cuda")
        self.ref = self.buf.clone()
        self.t = self.buf[GUARD:GUARD + n].view(shape)

    def guards_intact(self):
        torch.cuda.synchronize()
        return torch.equal(self.buf[:GUARD], self.ref[:GUARD]) and torch.equal(self.buf[-GUARD:], self.ref[-GUARD:])

    def untouched(self):
        torch.cuda.synchronize()
        return torch.equal(self.buf, self.ref)


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ---------------------------------------------------------------------------------------------------------------------
# paged attention
# ---------------------------------------------------------------------------------------------------------------------
def paged_problem(ctx, hq, hkv, d, block_size, dtype, g, **kw):
    return R.paged_problem(ctx, hq, hkv, d, block_size, dtype, g, **kw)


def run_decode(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, block_size, scale, nsplit):
    """``dsb_paged_decode`` with an explicit split count into a guarded output and guarded workspaces."""
    T = qkv.shape[0]
    out = Guarded((T, hq * d), qkv.dtype)
    ws_acc = Guarded((T * hq * nsplit * d, ), torch.float32)
    ws_ml = Guarded((T * hq * nsplit * 2, ), torch.float32)
    rc = N.cuda().dsb_paged_decode(P(qkv), P(cache), P(out.t), P(ws_acc.t), P(ws_ml.t), P(seq_of), P(pos_of), P(bt), T,
                                   hq, hkv, d, qkv.shape[1], block_size, bt.shape[1], ctypes.c_float(scale), nsplit,
                                   N.dt(qkv), N.stream())
    assert rc == 0, rc
    assert out.guards_intact() and ws_acc.guards_intact() and ws_ml.guards_intact()
    return out.t


def run_generic(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, block_size, scale):
    T = qkv.shape[0]
    out = Guarded((T, hq * d), qkv.dtype)
    rc = N.cuda().dsb_paged_attention(P(qkv), P(cache), P(out.t), P(seq_of), P(pos_of), P(bt), T, hq, hkv, d,
                                      qkv.shape[1], block_size, bt.shape[1], ctypes.c_float(scale), N.dt(qkv), N.stream())
    assert rc == 0, rc
    assert out.guards_intact()
    return out.t


def check_paged(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, block_size, scale, nsplit, mma, what):
    T = qkv.shape[0]
    q = qkv.view(T, hq + 2 * hkv, d)[:, :hq]
    ref, bnd = R.paged_attention_bounds(q, cache, seq_of.cpu(), pos_of.cpu(), bt.cpu(), block_size, scale, qkv.dtype,
                                        nsplit=nsplit, mma=mma)
    R.assert_within(out.view(T, hq, d), ref, bnd, what)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d,rep", [(64, 1), (64, 8), (128, 1), (128, 2), (128, 4), (128, 8), (256, 1), (256, 2),
                                   (256, 4), (256, 8)])
def test_paged_decode_kernels_bounded(dtype, d, rep):
    """The tensor-core kernel (d 64 / 128) and the CUDA-core kernel (d 256), reached by shape, at contexts that end on
    and around 16-key and cache-block edges, with split counts from 1 to 32 (many splits of the short sequences are
    empty)."""
    hkv, bs = 2, 64
    hq = hkv * rep
    path = RO.paged_attention_path(dtype, hq, hkv, d, (hq + 2 * hkv) * d)
    assert path == ("mma" if d in (64, 128) else "cuda_core")
    ctx = [1, 15, 16, 17, bs - 1, bs, bs + 1, 333, 1000]
    g = gen(d * 10 + rep)
    qkv, cache, seq_of, pos_of, bt = paged_problem(ctx, hq, hkv, d, bs, dtype, g, max_blocks=32)
    scale = 1.0 / math.sqrt(d)
    for nsplit in (1, 2, 3, 7, 32):
        out = run_decode(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, scale, nsplit)
        check_paged(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, scale, nsplit, path == "mma",
                    f"{path} d={d} rep={rep} nsplit={nsplit}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_paged_decode_mma_d128_long_peaked_context(dtype):
    """The tensor-core kernel at d = 128 on the long, peaked contexts of the host tier's mutation tests (the same data,
    generated on the host): there an emulated kernel that rounds ``q * scale`` to bf16 before QK^T leaves the bound."""
    hq, hkv, d, bs = 8, 2, 128, 128
    prob = R.paged_problem([1500, 700], hq, hkv, d, bs, dtype, torch.Generator().manual_seed(3))
    qkv, cache, seq_of, pos_of, bt = (t.cuda() for t in prob)
    for nsplit in (1, 4):
        out = run_decode(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 1.0 / math.sqrt(d), nsplit)
        check_paged(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 1.0 / math.sqrt(d), nsplit, True,
                    f"mma d=128 long nsplit={nsplit}")


@pytest.mark.parametrize("block_size", [16, 64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_paged_attention_routes_and_chunks(block_size, dtype):
    """``ragged_ops.paged_attention`` end to end: prefill-chunk tokens and decode tokens of the same sequences in one
    batch, each with its own causal limit, q read at the packed-QKV stride, at every block size."""
    hq, hkv, d = 8, 2, 128
    ctx, chunk = [40, 300, 129, 17], [24, 1, 5, 17]
    qkv, cache, seq_of, pos_of, bt = paged_problem(ctx, hq, hkv, d, block_size, dtype, gen(block_size), chunk=chunk)
    out = RO.paged_attention(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, block_size)
    nsplit = RO.decode_splits(qkv.shape[0], hkv, bt.shape[1] * block_size)
    check_paged(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, block_size, 1.0 / math.sqrt(d), nsplit, True,
                f"paged_attention bs={block_size}")


@pytest.mark.parametrize("dtype,d,rep,v1", [(torch.float32, 80, 7, False), (torch.float32, 96, 7, False),
                                            (torch.float32, 128, 2, False), (torch.bfloat16, 96, 7, False),
                                            (torch.bfloat16, 128, 4, True), (torch.float16, 64, 2, True)])
def test_paged_attention_generic_kernel_bounded(monkeypatch, dtype, d, rep, v1):
    """The one-CTA-per-head kernel: fp32, head dims 80 / 96, a head ratio of 7, and any shape under ``DSB200_PAGED_V1=1``."""
    if v1:
        monkeypatch.setenv("DSB200_PAGED_V1", "1")
    hkv, bs = 2, 16
    hq = hkv * rep
    assert RO.paged_attention_path(dtype, hq, hkv, d, (hq + 2 * hkv) * d) == "generic"
    qkv, cache, seq_of, pos_of, bt = paged_problem([1, 15, 16, 17, 200], hq, hkv, d, bs, dtype, gen(d + rep),
                                                   chunk=[1, 3, 1, 17, 2])
    out = RO.paged_attention(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs)
    check_paged(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 1.0 / math.sqrt(d), 1, False, f"generic d={d}")
    out2 = run_generic(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 0.3)
    check_paged(out2, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 0.3, 1, False, f"generic d={d} scale 0.3")


def test_paged_decode_llama32_3b_shape_and_graph_replay():
    """Llama-3.2-3B decode (24 query heads, 8 kv heads, d 128, 64 sequences x 2048 context).  ``paged_attention``
    routes the head ratio 3 to the generic kernel; the tensor-core decode kernel, which takes any ratio up to 8, is
    checked at the same shape through ``dsb_paged_decode``.  A CUDA-graph replay of the decode gives the same bits."""
    hq, hkv, d, bs = 24, 8, 128, 64
    qkv, cache, seq_of, pos_of, bt = paged_problem([2048] * 64, hq, hkv, d, bs, torch.bfloat16, gen(3))
    assert RO.paged_attention_path(qkv.dtype, hq, hkv, d, qkv.shape[1]) == "generic"
    out = RO.paged_attention(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs)
    nsplit = RO.decode_splits(64, hkv, bt.shape[1] * bs)
    mma = run_decode(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 1.0 / math.sqrt(d), nsplit)
    rows = torch.arange(0, 64, 9)  # a sample of the sequences: the float64 reference is ~1 s per sequence
    q = qkv.view(64, hq + 2 * hkv, d)[rows, :hq]
    for got, split, is_mma in ((out, 1, False), (mma, nsplit, True)):
        ref, bnd = R.paged_attention_bounds(q, cache, seq_of[rows].cpu(), pos_of[rows].cpu(), bt.cpu(), bs,
                                            1.0 / math.sqrt(d), torch.bfloat16, nsplit=split, mma=is_mma)
        R.assert_within(got.view(64, hq, d)[rows], ref, bnd, f"Llama-3.2-3B decode mma={is_mma}")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        RO.paged_attention(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs)  # warm the workspace outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gout = RO.paged_attention(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs)
    gout.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    R.assert_bits_equal(gout, out, "graph replay")


# ---------------------------------------------------------------------------------------------------------------------
# KV append, embedding, row gather
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("rot_dim", [0, 64, 128])
def test_kv_rotary_append_bit_exact(dtype, rot_dim):
    """Rotated q / k and every cache slot bit for bit against the fp32 / fma emulation (the host path), at positions past
    the first block; slots nobody wrote keep their sentinel."""
    hq, hkv, d, bs, S = 6, 2, 128, 16, 3
    g = gen(rot_dim)
    max_pos = 100
    ang = torch.rand(max_pos, max(rot_dim // 2, 1), generator=g, device="cuda") * 100
    cos, sin = torch.cos(ang).contiguous(), torch.sin(ang).contiguous()
    seq_of = torch.tensor([0, 0, 1, 2, 2, 2], dtype=torch.int32, device="cuda")
    pos_of = torch.tensor([15, 16, 0, 33, 34, 63], dtype=torch.int32, device="cuda")
    bt = torch.tensor([[5, 1, 9, 0], [2, 3, 4, 6], [7, 8, 10, 11]], dtype=torch.int32, device="cuda")
    qkv = (torch.randn(6, (hq + 2 * hkv) * d, generator=g, device="cuda") * 3).to(dtype)
    sent = {torch.float32: -1234.5, torch.bfloat16: -1234.0, torch.float16: -1234.0}[dtype]
    cache = Guarded((12, bs, 2, hkv, d), dtype, sentinel=sent)
    got = qkv.clone()
    RO.kv_rotary_append(got, cache.t, cos, sin, seq_of, pos_of, bt, hq, hkv, d, rot_dim, bs)
    assert cache.guards_intact()
    want_qkv = qkv.cpu().clone()
    want_cache = torch.full((12, bs, 2, hkv, d), sent, dtype=dtype)
    RO.kv_rotary_append(want_qkv, want_cache, cos.cpu(), sin.cpu(), seq_of.cpu(), pos_of.cpu(), bt.cpu(), hq, hkv, d, rot_dim,
                        bs)
    R.assert_bits_equal(got.cpu(), want_qkv, "rotated qkv")
    R.assert_bits_equal(cache.t.cpu(), want_cache, "paged cache")
    # the emulation the host path stands for, computed independently in numpy
    if rot_dim:
        half = rot_dim // 2
        v = qkv.cpu().float().view(6, hq + 2 * hkv, d)[:, :hq + hkv].numpy()
        c = cos.cpu().numpy()[pos_of.cpu().long().numpy()][:, None, :]
        s = sin.cpu().numpy()[pos_of.cpu().long().numpy()][:, None, :]
        a, b = v[..., :half], v[..., half:rot_dim]
        lo = R.fmaf(a, c, -(b * s))
        hi = R.fmaf(b, c, a * s)
        want = torch.from_numpy(np.concatenate([lo, hi], -1)).to(dtype)
        R.assert_bits_equal(got.cpu().view(6, hq + 2 * hkv, d)[:, :hq + hkv, :rot_dim], want, "rotation emulation")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_ragged_embed_and_row_gather_bit_exact(dtype):
    g = gen(11)
    H = 96
    wte = (torch.randn(100, H, generator=g, device="cuda")).to(dtype)
    wpe = (torch.randn(50, H, generator=g, device="cuda")).to(dtype)
    ids = torch.randint(0, 100, (17, ), generator=g, device="cuda", dtype=torch.int32)
    pos = torch.randint(0, 40, (17, ), generator=g, device="cuda", dtype=torch.int32)
    for pe in (None, wpe):
        out = Guarded((17, H), dtype)
        rc = N.cuda().dsb_ragged_embed(P(ids), P(pos if pe is not None else None), P(wte), P(pe), P(out.t), 17, H, 2,
                                       N.dt(wte), N.stream())
        assert rc == 0 and out.guards_intact()
        want = wte.cpu()[ids.cpu().long()].float()
        if pe is not None:
            want = want + wpe.cpu()[pos.cpu().long() + 2].float()  # one fp32 add of two stored values, rounded once
        R.assert_bits_equal(out.t.cpu(), want.to(dtype), f"ragged_embed wpe={pe is not None}")
        R.assert_bits_equal(out.t.cpu(), RO.ragged_embed(ids.cpu(), wte.cpu(), pos.cpu(), None if pe is None else wpe.cpu(),
                                                         2), "ragged_embed host path")
    idx = torch.tensor([3, 0, 16, 3], dtype=torch.int32, device="cuda")
    h = (torch.randn(17, H, generator=g, device="cuda")).to(dtype)
    out = Guarded((4, H), dtype)
    rc = N.cuda().dsb_row_gather(P(h), P(idx), P(out.t), 4, H, N.dt(h), N.stream())
    assert rc == 0 and out.guards_intact()
    R.assert_bits_equal(out.t, h[idx.long()], "row_gather")


# ---------------------------------------------------------------------------------------------------------------------
# MoE gating and routing
# ---------------------------------------------------------------------------------------------------------------------
def gating_logits(T, E, dtype, g, ties=True):
    x = torch.randn(T, E, generator=g, device="cuda") * 2
    if ties:
        x[::3, E // 2] = x[::3, 0]  # exact ties: equal logits, equal probabilities
        x[1::3, -1] = x[1::3, 1]
        x[2::7] = 0.5  # a whole row tied
    return x.to(dtype)


def run_gating(logits, K, normalize):
    T, E = logits.shape
    ids = Guarded((T, K), torch.int32, sentinel=-7)
    w = Guarded((T, K), torch.float32)
    counts = Guarded((E, ), torch.int32, sentinel=0)
    probs = Guarded((T, E), torch.float32)
    rc = N.cuda().dsb_top_k_gating(P(logits), P(ids.t), P(w.t), P(counts.t), P(probs.t), T, E, K, int(normalize),
                                   N.dt(logits), N.stream())
    assert rc == 0, rc
    for b in (ids, w, counts, probs):
        assert b.guards_intact()
    return ids.t, w.t, counts.t, probs.t


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("E", [8, 60, 64, 128, 256])
@pytest.mark.parametrize("K", [1, 2, 4, 8])
def test_top_k_gating_selection_oracle(dtype, E, K):
    if K > E:
        pytest.skip("K > E is refused")
    logits = gating_logits(300, E, dtype, gen(E * 10 + K))
    for normalize in (True, False):
        ids, w, counts, probs = run_gating(logits, K, normalize)
        R.check_gating(ids, w, counts, logits, K, normalize, f"gating E={E} K={K} norm={normalize}")
        Pr, b, _ = R.gating_reference(logits, K, normalize)
        R.assert_within(probs, Pr, b, "gating probabilities")
        hids, hw, hcounts = M.top_k_gating(logits.cpu(), K, normalize)
        R.check_gating(hids, hw, hcounts, logits.cpu(), K, normalize, "host gating")
        dids, dw, dcounts = M.top_k_gating(logits, K, normalize)
        assert torch.equal(dids, ids) and torch.equal(dcounts, counts)


def test_top_k_gating_nonfinite_rows_stay_in_range():
    """A NaN or +inf logit, or a row without a finite logit, routes to experts 0..K-1 with NaN weights; ids and counts
    stay in range and the finite rows are unaffected."""
    E, K = 60, 4
    logits = gating_logits(12, E, torch.float32, gen(5), ties=False)
    logits[1, 7] = float("nan")
    logits[3, 59] = float("inf")
    logits[5] = -float("inf")
    logits[7] = float("nan")
    logits[9, :30] = -float("inf")  # finite: half the experts are impossible
    bad = torch.tensor([1, 3, 5, 7])
    for normalize in (True, False):
        ids, w, counts, _ = run_gating(logits, K, normalize)
        assert torch.equal(ids[bad].cpu(), torch.arange(K, dtype=torch.int32).expand(4, K))
        assert bool(torch.isnan(w[bad]).all())
        ok = torch.tensor([i for i in range(12) if i not in bad.tolist()])
        R.check_gating(ids[ok], w[ok], torch.bincount(ids[ok].reshape(-1).long().cpu(), minlength=E).to(torch.int32),
                       logits[ok], K, normalize, "finite rows")
        assert torch.equal(counts.cpu(), torch.bincount(ids.reshape(-1).long().cpu(), minlength=E).to(torch.int32))
        hids, hw, hcounts = M.top_k_gating(logits.cpu(), K, normalize)
        assert torch.equal(hids, ids.cpu()) and torch.equal(hcounts, counts.cpu())
        assert torch.equal(torch.isnan(hw), torch.isnan(w.cpu()))


@pytest.mark.parametrize("E,K", [(257, 2), (64, 9), (4, 5)])
def test_top_k_gating_refused_arguments_write_nothing(E, K):
    logits = torch.randn(5, E, device="cuda")
    ids = Guarded((5, K), torch.int32, sentinel=-7)
    w = Guarded((5, K), torch.float32)
    counts = Guarded((E, ), torch.int32, sentinel=3)
    rc = N.cuda().dsb_top_k_gating(P(logits), P(ids.t), P(w.t), P(counts.t), None, 5, E, K, 1, N.dt(logits), N.stream())
    assert rc == -2
    assert ids.untouched() and w.untouched() and counts.untouched()
    with pytest.raises(Exception):
        M.top_k_gating(logits, K)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("capacity", [0, 3])
def test_route_scatter_gather_exact(dtype, capacity):
    """Positions, offsets and counts exactly in token-major order; scatter copies bit for bit (dropped assignments get
    slot -1 under a capacity); the weighted gather and its backward within float64 bounds.  Experts 0, 5 and 11 are
    empty."""
    E, K, T, H = 12, 2, 37, 64
    g = gen(capacity + 1)
    live = torch.tensor([1, 2, 3, 4, 6, 7, 8, 9, 10], device="cuda")
    ids = live[torch.randint(0, 9, (T, K), generator=g, device="cuda")].to(torch.int32)
    positions, counts, offsets = M.route(ids, E)
    hp, hc, ho = M.route(ids.cpu(), E)
    assert torch.equal(positions.cpu(), hp) and torch.equal(counts.cpu(), hc) and torch.equal(offsets.cpu(), ho)
    flat = ids.reshape(-1).cpu().tolist()
    seen = [0] * E
    want_pos = []
    for e in flat:
        want_pos.append(seen[e])
        seen[e] += 1
    assert positions.cpu().tolist() == want_pos
    assert offsets.cpu().tolist() == [0] + list(np.cumsum(seen))
    x = torch.randn(T, H, generator=g, device="cuda").to(dtype)
    rows = E * capacity if capacity else T * K
    out, slots = M.scatter(x, ids, positions, offsets, K, capacity, rows)
    hout, hslots = M.scatter(x.cpu(), ids.cpu(), hp, ho, K, capacity, rows)
    assert torch.equal(slots.cpu(), hslots)
    R.assert_bits_equal(out.cpu(), hout, "scatter")
    if capacity:
        assert bool((slots.cpu() == -1).any())
    w = torch.rand(T, K, generator=g, device="cuda")
    eo = torch.randn(rows, H, generator=g, device="cuda").to(dtype).requires_grad_(True)
    wt = w.clone().requires_grad_(True)
    y = M.gather(eo, wt, slots, T, K)
    s = slots.long().cpu().view(T, K)
    ok = (s >= 0).double()
    rowsv = eo.detach().cpu().double()[s.clamp(min=0)] * ok[..., None]
    ref = (rowsv * w.cpu().double()[..., None]).sum(1)
    mag = (rowsv.abs() * w.cpu().double()[..., None]).sum(1)
    R.assert_within(y.detach().cpu(), ref, R.ulp(ref.abs() + 2 * K * R.U * mag, dtype) + 2 * K * R.U * mag, "gather")
    dy = torch.randn(T, H, generator=g, device="cuda").to(dtype)
    y.backward(dy)
    dyd = dy.cpu().double()
    d_eo = torch.zeros(rows, H, dtype=torch.float64)
    dw = torch.zeros(T, K, dtype=torch.float64)
    for t in range(T):
        for k in range(K):
            if s[t, k] >= 0:
                d_eo[s[t, k]] = dyd[t] * float(w[t, k])
                dw[t, k] = (dyd[t] * eo.detach().cpu().double()[s[t, k]]).sum()
    R.assert_within(eo.grad.cpu(), d_eo, R.ulp(d_eo.abs(), dtype) + R.U * d_eo.abs(), "gather backward: expert rows")
    dmag = torch.zeros(T, K, dtype=torch.float64)
    for t in range(T):
        for k in range(K):
            if s[t, k] >= 0:
                dmag[t, k] = (dyd[t].abs() * eo.detach().cpu().double()[s[t, k]].abs()).sum()
    R.assert_within(wt.grad.cpu(), dw, (H + 8) * R.U * dmag, "gather backward: weights")


# ---------------------------------------------------------------------------------------------------------------------
# weight-only quantized GEMMs
# ---------------------------------------------------------------------------------------------------------------------
MODES = ["int8", "int4", "fp8", "fp6"]


def quantized(mode, N_, K_, gs, g, dtype=torch.bfloat16, experts=None):
    """A hand-built ``QuantizedWeight``: random codes of ``mode`` and per-group scales that vary by 2^+-3 from group to
    group (a scale applied to the neighbouring group cannot pass), and the exact float64 dequantized weight."""
    from deepspeed_b200.inference.quantization.layers import QuantizedWeight
    cpu = torch.Generator().manual_seed(int(g.initial_seed()))
    codes, vals = R.wq_codes(mode, N_, K_, cpu)
    scales = torch.ldexp(torch.rand(N_ * K_ // gs, generator=cpu) + 0.5, torch.randint(-9, -3, (N_ * K_ // gs, ),
                                                                                        generator=cpu)).float()
    wdq = (vals.view(N_, K_ // gs, gs) * scales.double().view(N_, K_ // gs, 1)).view(N_, K_)
    q = R.wq_pack(codes, mode).cuda()
    return QuantizedWeight(q, scales.cuda(), (N_, K_), mode, gs, dtype), wdq.cuda()


@pytest.mark.parametrize("mode", ["int8", "int4", "fp8"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("gs", [64, 128, 256])
def test_wq_gemv_bounded(mode, dtype, gs):
    """The mma.sync GEMV at M = 1..32 (both row tiles), with and without bias, N not a multiple of the 16 / 32 feature
    tile."""
    from deepspeed_b200.inference.quantization.layers import _wq_gemv
    if mode == "int4" and gs == 64:
        pytest.skip("int4 chunks are 128 weights: group 64 is not eligible")
    g = gen(gs + len(mode))
    N_, K_ = 200, 512
    qw, wdq = quantized(mode, N_, K_, gs, g, dtype)
    tile = 128 if mode == "int4" else 64
    for M_ in (1, 7, 16, 17, 32):
        x = torch.randn(M_, K_, generator=g, device="cuda").to(dtype)
        for bias in (None, torch.randn(N_, generator=g, device="cuda").to(dtype)):
            y = _wq_gemv(x, qw, bias)
            assert y is not None and y.dtype == dtype
            ref, bnd = R.wq_bounds(x, wdq, bias, dtype, tile, K_ // tile // 8 + 12)
            R.assert_within(y, ref, bnd, f"wq_gemv {mode} M={M_} bias={bias is not None}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M_", [33, 64, 65, 127, 128, 129, 256, 512])
def test_wq_tc_gemm_bounded(mode, M_):
    """The wgmma GEMM at row counts around its 128-token tile, N not a multiple of the 128-feature tile."""
    from deepspeed_b200.inference.quantization.layers import wq_tc_linear
    g = gen(M_ + len(mode))
    N_, K_, gs = 200, 768, 128 if M_ % 2 else 256
    qw, wdq = quantized(mode, N_, K_, gs, g)
    x = torch.randn(M_, K_, generator=g, device="cuda").bfloat16()
    bias = torch.randn(N_, generator=g, device="cuda").bfloat16() if M_ % 2 else None
    y = wq_tc_linear(x, qw, bias, max_rows=512)
    assert y is not None
    ref, bnd = R.wq_bounds(x, wdq, bias, torch.bfloat16, 16, 2 * K_, w_round=2.0**-8 + R.U)
    R.assert_within(y, ref, bnd, f"wq_tc {mode} M={M_}")


@pytest.mark.parametrize("M_", [1, 128])
@pytest.mark.parametrize("NK", [(5120, 3072), (3072, 3072), (16384, 3072), (3072, 8192)])
def test_wq_llama32_3b_projections(M_, NK):
    """The Llama-3.2-3B decode projections (fused QKV, O, fused gate/up, down) through ``maybe_quantized_linear``: the
    GEMV at one row, the wgmma GEMM at 128, int4 weights in groups of 128; every 16th output column is checked."""
    from deepspeed_b200.inference.quantization.layers import maybe_quantized_linear
    N_, K_ = NK
    g = gen(N_ + K_ + M_)
    qw, wdq = quantized("int4", N_, K_, 128, g)
    x = torch.randn(M_, K_, generator=g, device="cuda").bfloat16()
    y = maybe_quantized_linear(x, qw)
    cols = torch.arange(0, N_, 16, device="cuda")
    tc = M_ > 32
    ref, bnd = R.wq_bounds(x, wdq[cols], None, torch.bfloat16, 16 if tc else 128, 2 * K_ if tc else K_ // 128 // 8 + 12,
                           w_round=(2.0**-8 + R.U) if tc else 0.0)
    R.assert_within(y[:, cols], ref, bnd, f"Llama-3.2-3B [{M_} x {N_} x {K_}]")


@pytest.mark.parametrize("mode", ["int8", "int4"])
def test_wq_int4_and_int8_code_order_pinned(mode):
    """One-hot activations read single weights: codes that differ at every position of a packed word come back in place,
    exactly (power-of-two scales), through the GEMV and the wgmma GEMM."""
    from deepspeed_b200.inference.quantization.layers import QuantizedWeight, _wq_gemv, wq_tc_linear
    N_, K_ = 24, 128
    n, k = torch.meshgrid(torch.arange(N_), torch.arange(K_), indexing="ij")
    codes = ((k + 3 * n) % 16) - 8 if mode == "int4" else ((k * 7 + n * 13) % 255) - 127
    scales = torch.full((N_, ), 0.25)
    qw = QuantizedWeight(R.wq_pack(codes, mode).cuda(), scales.cuda(), (N_, K_), mode, 128, torch.bfloat16)
    want = (codes.double() * 0.25).t()  # out[k, n] for x = identity
    eye = torch.eye(K_, device="cuda", dtype=torch.bfloat16)
    y = wq_tc_linear(eye, qw, None, max_rows=512)
    R.assert_bits_equal(y.cpu(), want.to(torch.bfloat16), "wgmma GEMM code order")
    for r0 in range(0, K_, 32):
        y = _wq_gemv(eye[r0:r0 + 32], qw, None)
        R.assert_bits_equal(y.cpu(), want[r0:r0 + 32].to(torch.bfloat16), f"GEMV code order rows {r0}..")


def test_wq_eligibility_boundaries_return_none():
    from deepspeed_b200.inference.quantization.layers import _wq_gemv, wq_tc_linear
    g = gen(1)
    qw, _ = quantized("int8", 64, 192, 64, g)
    assert wq_tc_linear(torch.randn(600, 192, device="cuda").bfloat16(), qw) is None  # over the row limit
    assert _wq_gemv(torch.randn(33, 192, device="cuda").bfloat16(), qw, None) is None
    qw2, _ = quantized("int8", 64, 96 * 2, 96, g)  # group 96: not a multiple of 64
    assert wq_tc_linear(torch.randn(64, 192, device="cuda").bfloat16(), qw2) is None
    assert _wq_gemv(torch.randn(4, 192, device="cuda").bfloat16(), qw2, None) is None
    qw3, _ = quantized("int8", 64, 160, 32, g)  # K % 64 != 0
    assert wq_tc_linear(torch.randn(64, 160, device="cuda").bfloat16(), qw3) is None
    assert _wq_gemv(torch.randn(4, 160, device="cuda").bfloat16(), qw3, None) is None


@pytest.mark.parametrize("mode", MODES)
def test_mixed_moe_gemm_grouped_bounded(mode):
    """The grouped form in one launch: the first, a middle and the last expert empty, ragged tails, rows outside the
    experts' ranges untouched."""
    from deepspeed_b200.inference.v2.kernels.cutlass_ops.moe_gemm.mixed_moe_gemm import MixedMoEGEMM
    E, N_, K_, gs = 6, 136, 256, 128
    rows = [0, 70, 129, 0, 5, 0]
    g = gen(len(mode) + 40)
    qws, wdqs = zip(*[quantized(mode, N_, K_, gs, gen(100 + e)) for e in range(E)])
    bias = torch.randn(E, N_, generator=g, device="cuda").bfloat16()
    Mt = sum(rows)
    x = torch.randn(Mt, K_, generator=g, device="cuda").bfloat16()
    out = Guarded((Mt, N_), torch.bfloat16)
    cum = torch.tensor(np.cumsum(rows), dtype=torch.int32, device="cuda")
    MixedMoEGEMM(torch.bfloat16, num_bits=8)(out.t, x, list(qws), None, cum, bias)
    assert out.guards_intact()
    s = 0
    for e, r in enumerate(rows):
        if r:
            ref, bnd = R.wq_bounds(x[s:s + r], wdqs[e], bias[e], torch.bfloat16, 16, 2 * K_, w_round=2.0**-8 + R.U)
            R.assert_within(out.t[s:s + r], ref, bnd, f"grouped {mode} expert {e}")
        s += r
