"""Host tier of the ragged-inference checks (``tests/gpu/test_inference_exact_gpu.py``): the host paths held to the
same references, the references themselves against ``math.fsum``, and mutation tests -- each plausible kernel bug,
emulated on the host, is refused by the check the GPU tests apply."""
import math

import numpy as np
import pytest
import torch

from tests import numerics as R
from deepspeed_b200.ops.kernels import moe_ops as M
from deepspeed_b200.ops.kernels import ragged_ops as RO


# ---------------------------------------------------------------------------------------------------------------------
# paged attention
# ---------------------------------------------------------------------------------------------------------------------
def paged_problem(ctx, hq, hkv, d, block_size, dtype, seed, peak=20.0, chunk=None):
    """The GPU tests' problem (permuted, non-contiguous block tables, peaked logits) on the host."""
    return R.paged_problem(ctx, hq, hkv, d, block_size, dtype, torch.Generator().manual_seed(seed), peak=peak, chunk=chunk)


def emulate_decode(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, scale, nsplit, mma, q_round=False, drop_split=None,
                   double_split=None, rows=None):
    """Split-KV decode in torch fp32, the way the kernels split and merge: per split a max, ``p = exp(x - m)``, ``l``
    and ``acc = p V`` (p rounded to the storage type first for the tensor-core kernel), merged with ``exp(m_s - max)``.

    Mutations: ``q_round`` rounds ``q * scale`` to the storage type before QK^T; ``drop_split`` / ``double_split``
    leave one split out of the merge or count it twice; ``rows(seq, n) -> (blocks, slots)`` replaces the cache
    addressing of the keys."""
    T = qkv.shape[0]
    dt = qkv.dtype
    c = torch.tensor(scale, dtype=torch.float32)
    rep = hq // hkv
    out = torch.zeros(T, hq, d, dtype=torch.float32)
    q = qkv.view(T, hq + 2 * hkv, d)[:, :hq].float()
    for t in range(T):
        n = int(pos_of[t]) + 1
        seq = int(seq_of[t])
        if rows is None:
            j = torch.arange(n)
            blk, slot = bt[seq].long()[j // bs], j % bs
        else:
            blk, slot = rows(seq, n)
        kv = cache[blk, slot].float()  # [n, 2, hkv, d]
        per = -(-n // nsplit)
        if mma:
            per = (per + 15) // 16 * 16
        for h in range(hq):
            g = h // rep
            K, V = kv[:, 0, g], kv[:, 1, g]
            if q_round:
                x = (q[t, h] * c).to(dt).float() @ K.t()
            else:
                x = (q[t, h] @ K.t()) * c
            parts = []
            for s in range(nsplit):
                k0, k1 = s * per, min(n, (s + 1) * per)
                if k0 >= k1:
                    continue
                m = x[k0:k1].max()
                p = torch.exp(x[k0:k1] - m)
                pv = p.to(dt).float() if mma else p
                parts.append((s, m, p.sum(), pv @ V[k0:k1]))
            parts = [pt for pt in parts if pt[0] != drop_split] + [pt for pt in parts if pt[0] == double_split]
            gm = max(pt[1] for pt in parts)
            l = sum(pt[2] * torch.exp(pt[1] - gm) for pt in parts)
            o = sum(pt[3] * torch.exp(pt[1] - gm) for pt in parts)
            out[t, h] = o / l
    return out.to(dt)


def bounded(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, scale, nsplit, mma):
    T = qkv.shape[0]
    q = qkv.view(T, hq + 2 * hkv, d)[:, :hq]
    ref, bnd = R.paged_attention_bounds(q, cache, seq_of, pos_of, bt, bs, scale, qkv.dtype, nsplit=nsplit, mma=mma)
    R.assert_within(out.view(T, hq, d), ref, bnd, "paged attention")


def refused(fn):
    with pytest.raises(AssertionError, match="outside the bound"):
        fn()


def test_paged_reference_against_fsum():
    """The float64 reference: scores and the softmax-weighted sum against exactly rounded ``math.fsum`` sums."""
    hq, hkv, d, bs = 2, 1, 16, 4
    qkv, cache, seq_of, pos_of, bt = paged_problem([7], hq, hkv, d, bs, torch.float32, 0)
    ref, _ = R.paged_attention_bounds(qkv.view(1, 4, d)[:, :hq], cache, seq_of, pos_of, bt, bs, 0.25, torch.float32)
    k, v = R.paged_rows(cache, bt, 0, 7, bs)
    q = qkv.view(1, 4, d)[0, :hq].double()
    for h in range(hq):
        x = [math.fsum(float(q[h, i]) * float(k[j, 0, i]) for i in range(d)) * 0.25 for j in range(7)]
        mx = max(x)
        e = [math.exp(xi - mx) for xi in x]
        L = math.fsum(e)
        for i in range(d):
            o = math.fsum(e[j] * float(v[j, 0, i]) for j in range(7)) / L
            assert abs(o - float(ref[0, h, i])) <= 1e-14 * (1 + abs(o))
    # the paged addressing: the rows come from the table's blocks in order
    j = 5
    assert torch.equal(k[j], cache[bt[0, j // bs], j % bs, 0])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_paged_attention_host_path_within_bound(dtype):
    hq, hkv, d, bs = 4, 2, 64, 16
    qkv, cache, seq_of, pos_of, bt = paged_problem([1, 17, 40, 100], hq, hkv, d, bs, dtype, 1, chunk=[1, 3, 1, 5])
    out = RO.paged_attention(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs)
    bounded(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 1 / math.sqrt(d), 1, False)


@pytest.mark.parametrize("mma,nsplit", [(True, 1), (True, 4), (False, 3)])
def test_split_kv_emulation_within_bound(mma, nsplit):
    """A correct fp32 implementation of the kernels' split-and-merge, P rounding included, passes the bound."""
    hq, hkv, d, bs = 4, 1, 128, 64
    qkv, cache, seq_of, pos_of, bt = paged_problem([15, 17, 300], hq, hkv, d, bs, torch.bfloat16, 2)
    out = emulate_decode(qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 1 / math.sqrt(d), nsplit, mma)
    bounded(out, qkv, cache, seq_of, pos_of, bt, hq, hkv, d, bs, 1 / math.sqrt(d), nsplit, mma)


LONG = dict(ctx=[1500, 700], hq=8, hkv=2, d=128, bs=128)


def long_problem(dtype=torch.bfloat16, seed=3):
    L = LONG
    return paged_problem(L["ctx"], L["hq"], L["hkv"], L["d"], L["bs"], dtype, seed)


@pytest.mark.parametrize("peak", [20.0, 0.2])
def test_mutation_sixteen_keys_from_wrong_slots(peak):
    """16 keys (one MMA key block) read from the slots 16 positions on: the slip a block-table or slot index bug inside a
    key block makes.  Refused with peaked and with near-uniform attention."""
    L = LONG
    qkv, cache, seq_of, pos_of, bt = paged_problem(L["ctx"], L["hq"], L["hkv"], L["d"], L["bs"], torch.bfloat16, 3, peak=peak)

    def rows(seq, n):
        j = torch.arange(n)
        j = torch.where((j >= 640) & (j < 656), j + 16, j)
        return bt[seq].long()[j // L["bs"]], j % L["bs"]

    out = emulate_decode(qkv, cache, seq_of, pos_of, bt, L["hq"], L["hkv"], L["d"], L["bs"], 1 / math.sqrt(L["d"]), 4, True,
                         rows=rows)
    refused(lambda: bounded(out, qkv, cache, seq_of, pos_of, bt, L["hq"], L["hkv"], L["d"], L["bs"], 1 / math.sqrt(L["d"]),
                            4, True))


@pytest.mark.parametrize("how", ["drop", "double"])
def test_mutation_split_dropped_or_counted_twice(how):
    L = LONG
    qkv, cache, seq_of, pos_of, bt = long_problem()
    kw = {"drop_split" if how == "drop" else "double_split": 2}
    out = emulate_decode(qkv, cache, seq_of, pos_of, bt, L["hq"], L["hkv"], L["d"], L["bs"], 1 / math.sqrt(L["d"]), 4, True,
                         **kw)
    refused(lambda: bounded(out, qkv, cache, seq_of, pos_of, bt, L["hq"], L["hkv"], L["d"], L["bs"], 1 / math.sqrt(L["d"]),
                            4, True))


def test_mutation_scaled_query_rounded_to_bf16():
    """``q * scale`` rounded back to bf16 before QK^T at d = 128, where the scale is not a power of two (the tensor-core
    kernel did this before the scale moved to the fp32 scores)."""
    L = LONG
    qkv, cache, seq_of, pos_of, bt = long_problem()
    args = (qkv, cache, seq_of, pos_of, bt, L["hq"], L["hkv"], L["d"], L["bs"], 1 / math.sqrt(L["d"]), 4, True)
    bounded(emulate_decode(*args), *args)
    refused(lambda: bounded(emulate_decode(*args, q_round=True), *args))


def test_mutation_block_table_off_by_one():
    """The last cache block of a sequence looked up one table entry early."""
    L = LONG
    qkv, cache, seq_of, pos_of, bt = long_problem()

    def rows(seq, n):
        j = torch.arange(n)
        e = j // L["bs"]
        e = torch.where(e == (n - 1) // L["bs"], e - 1, e)
        return bt[seq].long()[e], j % L["bs"]

    out = emulate_decode(qkv, cache, seq_of, pos_of, bt, L["hq"], L["hkv"], L["d"], L["bs"], 1 / math.sqrt(L["d"]), 1, True,
                         rows=rows)
    refused(lambda: bounded(out, qkv, cache, seq_of, pos_of, bt, L["hq"], L["hkv"], L["d"], L["bs"], 1 / math.sqrt(L["d"]),
                            1, True))


def test_path_helper_follows_the_routing(monkeypatch):
    monkeypatch.delenv("DSB200_PAGED_V1", raising=False)
    monkeypatch.delenv("DSB200_PAGED_DECODE_MMA", raising=False)
    bf = torch.bfloat16
    assert RO.paged_attention_path(bf, 32, 8, 128, 48 * 128) == "mma"
    assert RO.paged_attention_path(bf, 24, 8, 128, 40 * 128) == "generic"  # ratio 3: the Llama-3.2-3B heads
    assert RO.paged_attention_path(torch.float16, 8, 1, 64, 10 * 64) == "mma"
    assert RO.paged_attention_path(bf, 8, 8, 256, 24 * 256) == "cuda_core"
    assert RO.paged_attention_path(torch.float32, 8, 2, 128, 12 * 128) == "generic"
    assert RO.paged_attention_path(bf, 14, 2, 128, 18 * 128) == "generic"  # ratio 7
    assert RO.paged_attention_path(bf, 4, 2, 96, 8 * 96) == "generic"
    monkeypatch.setenv("DSB200_PAGED_DECODE_MMA", "0")
    assert RO.paged_attention_path(bf, 32, 8, 128, 48 * 128) == "cuda_core"
    monkeypatch.setenv("DSB200_PAGED_V1", "1")
    assert RO.paged_attention_path(bf, 32, 8, 128, 48 * 128) == "generic"
    monkeypatch.delenv("DSB200_PAGED_V1")
    monkeypatch.delenv("DSB200_PAGED_DECODE_MMA")
    assert RO.decode_splits(64, 8, 2048) == 1
    assert RO.decode_splits(1, 1, 8192) == 32
    assert RO.decode_splits(1, 1, 600) == 2


# ---------------------------------------------------------------------------------------------------------------------
# KV append, embedding, row gather
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("rot_dim", [0, 32, 64])
def test_kv_rotary_append_host_path_bit_exact(dtype, rot_dim):
    """The host path's rotation is the kernels' ``fmaf(a, c, -(b * s))`` / ``fmaf(b, c, a * s)`` bit for bit; cache slots
    outside the written ones keep their sentinel."""
    hq, hkv, d, bs = 4, 2, 64, 16
    g = torch.Generator().manual_seed(rot_dim)
    ang = torch.rand(80, max(rot_dim // 2, 1), generator=g) * 100
    cos, sin = torch.cos(ang), torch.sin(ang)
    seq_of = torch.tensor([0, 0, 1, 1], dtype=torch.int32)
    pos_of = torch.tensor([15, 16, 40, 63], dtype=torch.int32)
    bt = torch.tensor([[3, 0, 1, 2], [4, 5, 6, 7]], dtype=torch.int32)
    qkv = (torch.randn(4, (hq + 2 * hkv) * d, generator=g) * 3).to(dtype)
    cache = torch.full((8, bs, 2, hkv, d), -1234.0, dtype=dtype)
    got = qkv.clone()
    RO.kv_rotary_append(got, cache, cos, sin, seq_of, pos_of, bt, hq, hkv, d, rot_dim, bs)
    v = qkv.float().view(4, hq + 2 * hkv, d).numpy()
    want = v.copy()
    if rot_dim:
        half = rot_dim // 2
        c = cos.numpy()[pos_of.long().numpy()][:, None, :]
        s = sin.numpy()[pos_of.long().numpy()][:, None, :]
        a, b = v[:, :hq + hkv, :half], v[:, :hq + hkv, half:rot_dim]
        want[:, :hq + hkv, :half] = R.fmaf(a, c, -(b * s))
        want[:, :hq + hkv, half:rot_dim] = R.fmaf(b, c, a * s)
    want = torch.from_numpy(want).to(dtype)
    R.assert_bits_equal(got.view(4, hq + 2 * hkv, d), want, "rotated qkv")
    written = torch.zeros(8, bs, dtype=torch.bool)
    for t in range(4):
        blk, slot = int(bt[seq_of[t], pos_of[t] // bs]), int(pos_of[t] % bs)
        written[blk, slot] = True
        R.assert_bits_equal(cache[blk, slot], want[t, hq:].view(2, hkv, d), f"cache slot of token {t}")
    assert bool((cache[~written] == -1234.0).all())
    if rot_dim and dtype == torch.float32:
        # the unfused form rounds differently somewhere: the bit-exact check tells the two apart
        unfused = torch.from_numpy(a * c - b * s)
        assert not torch.equal(unfused, want[:, :hq + hkv, :half])


def test_ragged_embed_and_row_gather_host_exact():
    wte, wpe = torch.randn(50, 32).bfloat16(), torch.randn(20, 32).bfloat16()
    ids, pos = torch.tensor([3, 49, 0, 3], dtype=torch.int32), torch.tensor([0, 5, 17, 2], dtype=torch.int32)
    got = RO.ragged_embed(ids, wte, pos, wpe, 2)
    want = (wte.float()[ids.long()] + wpe.float()[pos.long() + 2]).bfloat16()
    R.assert_bits_equal(got, want, "ragged_embed")
    R.assert_bits_equal(RO.row_gather(got, torch.tensor([3, 0], dtype=torch.int32)), got[[3, 0]], "row_gather")


# ---------------------------------------------------------------------------------------------------------------------
# MoE gating and routing
# ---------------------------------------------------------------------------------------------------------------------
def logits_with_ties(T, E, seed):
    x = torch.randn(T, E, generator=torch.Generator().manual_seed(seed)) * 2
    x[::3, E // 2] = x[::3, 0]
    x[1::3, -1] = x[1::3, 1]
    x[2::7] = 0.5
    return x


@pytest.mark.parametrize("E", [8, 60, 256])
@pytest.mark.parametrize("K", [1, 2, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_top_k_gating_host_path_meets_the_oracle(E, K, dtype):
    if K > E:
        pytest.skip("K > E is refused")
    logits = logits_with_ties(60, E, E + K).to(dtype)
    for normalize in (True, False):
        ids, w, counts = M.top_k_gating(logits, K, normalize)
        R.check_gating(ids, w, counts, logits, K, normalize, "host gating")


def test_gating_reference_against_fsum():
    x = torch.randn(3, 9, dtype=torch.float64)
    P, _, order = R.gating_reference(x, 2, True)
    for t in range(3):
        e = [math.exp(float(v)) for v in x[t]]
        s = math.fsum(e)
        for j in range(9):
            assert abs(P[t, j].item() - e[j] / s) <= 1e-15
    assert torch.equal(order, torch.sort(P, dim=-1, descending=True, stable=True).indices)


def test_mutation_gating_tie_break_reversed():
    """Ties going to the highest index instead of the lowest are refused."""
    logits = logits_with_ties(30, 16, 1)
    P = torch.softmax(logits.double(), -1)
    rev = torch.sort(P.flip(-1), dim=-1, descending=True, stable=True).indices
    ids = (15 - rev[:, :2]).to(torch.int32)
    w = P.gather(1, ids.long()).float()
    counts = torch.bincount(ids.reshape(-1).long(), minlength=16).to(torch.int32)
    with pytest.raises(AssertionError, match="chose"):
        R.check_gating(ids, w, counts, logits, 2, False)


def test_mutation_gating_wrong_counts_and_weights():
    logits = logits_with_ties(30, 16, 2)
    ids, w, counts = M.top_k_gating(logits, 2, False)
    bad = counts.clone()
    bad[3] += 1
    with pytest.raises(AssertionError, match="counts"):
        R.check_gating(ids, w, bad, logits, 2, False)
    with pytest.raises(AssertionError, match="weights"):
        R.check_gating(ids, w * (1 + 2.0**-12), counts, logits, 2, False)


def kernel_argmax(v, E, K):
    """The warp arg-max of ``top_k_gating_kernel`` as written before the non-finite guard: 32 lanes each keep the best
    of their ``v[lane + 32 j]`` (strictly greater, starting from -1), a butterfly over the lanes, ties to the lower
    index; the winner is removed by setting it to -1."""
    v = list(v) + [-math.inf] * (256 - len(v))
    ids = []
    for _ in range(K):
        best, bi = [-1.0] * 32, [0x7FFFFFFF] * 32
        for lane in range(32):
            for j in range(8):
                e = lane + 32 * j
                if e < E and v[e] > best[lane]:
                    best[lane], bi[lane] = v[e], e
        o = 16
        while o:
            nb, ni = best[:], bi[:]
            for lane in range(32):
                ob, oi = best[lane ^ o], bi[lane ^ o]
                if ob > best[lane] or (ob == best[lane] and oi < bi[lane]):
                    nb[lane], ni[lane] = ob, oi
            best, bi = nb, ni
            o >>= 1
        ids.append(bi[0])
        if bi[0] != 0x7FFFFFFF:
            v[bi[0]] = -1.0
    return ids


def test_nonfinite_row_breaks_the_warp_argmax_and_the_guard_catches_it():
    """A row with no finite logit makes every ``exp(x - max)`` NaN, and so does a row of NaNs; when fewer than K values
    are left that the arg-max can compare, it returns 0x7fffffff (an out-of-range expert id and counts index).  The
    kernel's guard (the sum of exps is NaN) fires on every such row -- and on any row with a NaN or +inf logit, whose
    weights are NaN anyway -- and the host path gives those rows the same ids and NaN weights."""
    E, K = 40, 3
    rows = {"nan": [0.0] * E, "inf": [0.0] * E, "all_-inf": [-math.inf] * E, "finite": [0.0] * E, "some_-inf": [0.0] * E,
            "mostly_nan": [math.nan] * E}
    rows["nan"][5] = math.nan
    rows["inf"][7] = math.inf
    rows["mostly_nan"][9] = 1.0
    for j in range(10):
        rows["some_-inf"][j] = -math.inf
    rows["finite"][3] = 1.0
    logits = torch.tensor(list(rows.values()), dtype=torch.float32)
    for r, (name, x) in enumerate(rows.items()):
        x = np.asarray(x, np.float32)
        with np.errstate(invalid="ignore"):
            mx = np.float32(-np.inf)
            for xi in x:
                mx = np.fmax(mx, xi)  # fmaxf drops a NaN operand
            v = np.exp(x - mx)
        guard = bool(np.isnan(v.sum()))
        ids = kernel_argmax([float(t) for t in v], E, K)
        assert guard == (name in ("nan", "inf", "all_-inf", "mostly_nan")), name
        assert (0x7FFFFFFF in ids) == (name in ("all_-inf", "mostly_nan")), (name, ids)
    ids, w, counts = M.top_k_gating(logits, K, True)
    bad = torch.tensor([0, 1, 2, 5])
    assert ids[bad].tolist() == [[0, 1, 2]] * 4
    assert bool(torch.isnan(w[bad]).all()) and not bool(torch.isnan(w[3:5]).any())
    assert ids[3].tolist()[0] == 3 and min(ids[4].tolist()) >= 10
    assert int(counts.sum()) == 6 * K


@pytest.mark.parametrize("capacity", [0, 2])
def test_route_scatter_gather_host_exact(capacity):
    E, K, T, H = 6, 2, 11, 8
    g = torch.Generator().manual_seed(capacity)
    ids = torch.tensor([1, 2, 4, 1, 2, 3, 4, 1, 3, 2, 1, 4, 2, 3, 4, 1, 2, 3, 1, 4, 2, 3], dtype=torch.int32).view(T, K)
    positions, counts, offsets = M.route(ids, E)
    seen = [0] * E
    want = []
    for e in ids.reshape(-1).tolist():
        want.append(seen[e])
        seen[e] += 1
    assert positions.tolist() == want and counts.tolist() == seen
    assert offsets.tolist() == [0] + list(np.cumsum(seen))
    x = torch.randn(T, H, generator=g).bfloat16()
    rows = E * capacity if capacity else T * K
    out, slots = M.scatter(x, ids, positions, offsets, K, capacity, rows)
    for a in range(T * K):
        s = int(slots[a])
        if capacity and want[a] >= capacity:
            assert s == -1
        else:
            assert s == (int(ids.view(-1)[a]) * capacity + want[a] if capacity else int(offsets[ids.view(-1)[a]]) + want[a])
            R.assert_bits_equal(out[s], x[a // K], "scatter row")
    eo = torch.randn(rows, H, generator=g).bfloat16()
    w = torch.rand(T, K, generator=g)
    y = M.gather(eo, w, slots, T, K)
    s = slots.long().view(T, K)
    ref = torch.zeros(T, H, dtype=torch.float64)
    for t in range(T):
        for k in range(K):
            if s[t, k] >= 0:
                ref[t] += float(w[t, k]) * eo[s[t, k]].double()
    R.assert_within(y, ref, R.ulp(ref.abs() + 1e-6, torch.bfloat16) + 1e-6, "gather")


# ---------------------------------------------------------------------------------------------------------------------
# weight-only quantized GEMMs: the bound refuses the plausible bugs
# ---------------------------------------------------------------------------------------------------------------------
def wq_problem(mode, N, K, gs, seed):
    g = torch.Generator().manual_seed(seed)
    codes, vals = R.wq_codes(mode, N, K, g)
    scales = torch.ldexp(torch.rand(N * K // gs, generator=g) + 0.5, torch.randint(-9, -3, (N * K // gs, ), generator=g))
    x = torch.randn(8, K, generator=g).bfloat16()
    return codes, vals, scales.float(), x


def emulate_gemv(x, vals, scales, gs, tile, bias=None, scale_shift=0):
    """The GEMV's order in fp32: each ``tile`` of products summed, times its group's scale (group ``g + scale_shift``,
    wrapping), accumulated; one bias add; rounded to bf16."""
    N, K = vals.shape
    xs = x.float()
    s = scales.view(N, K // gs)
    acc = torch.zeros(x.shape[0], N)
    for k0 in range(0, K, tile):
        gi = (k0 // gs + scale_shift) % (K // gs)
        acc = acc + (xs[:, k0:k0 + tile] @ vals[:, k0:k0 + tile].float().t()) * s[:, gi][None, :]
    if bias is not None:
        acc = acc + bias.float()
    return acc.bfloat16()


@pytest.mark.parametrize("mode", ["int8", "int4", "fp8", "fp6"])
def test_wq_codes_and_packing_roundtrip(mode):
    codes, vals = R.wq_codes(mode, 4, 64, torch.Generator().manual_seed(0))
    packed = R.wq_pack(codes, mode).numpy().view(np.uint8).astype(np.int64)
    if mode in ("int8", "fp8"):
        back = packed
    elif mode == "int4":
        back = np.stack([packed & 0xF, packed >> 4], -1).reshape(4, 64)
    else:
        bits = ((packed[:, :, None] >> np.arange(8)) & 1).reshape(4, -1)
        back = (bits[:, :64 * 6].reshape(4, 64, 6) << np.arange(6)).sum(-1)
    mask = {"int8": 0xFF, "int4": 0xF, "fp8": 0xFF, "fp6": 0x3F}[mode]
    assert np.array_equal(back, codes.numpy() & mask)
    assert torch.isfinite(vals).all()


@pytest.mark.parametrize("mode,gs", [("int8", 64), ("int4", 128), ("fp8", 256)])
def test_wq_gemv_emulation_within_bound_and_mutations_refused(mode, gs):
    N, K = 24, 512
    codes, vals, scales, x = wq_problem(mode, N, K, gs, 5)
    tile = 128 if mode == "int4" else 64
    wdq = (vals.view(N, K // gs, gs) * scales.double().view(N, K // gs, 1)).view(N, K)
    bias = torch.randn(N).bfloat16()
    ref, bnd = R.wq_bounds(x, wdq, bias, torch.bfloat16, tile, K // tile // 8 + 12)
    R.assert_within(emulate_gemv(x, vals, scales, gs, tile, bias), ref, bnd, "GEMV emulation")
    # a group's scale applied to the neighbouring group
    refused(lambda: R.assert_within(emulate_gemv(x, vals, scales, gs, tile, bias, scale_shift=1), ref, bnd, "shifted"))
    if mode == "int4":
        # the two nibbles of every byte swapped
        swapped = vals.view(N, K // 2, 2).flip(-1).reshape(N, K)
        refused(lambda: R.assert_within(emulate_gemv(x, swapped, scales, gs, tile, bias), ref, bnd, "nibbles"))
    # the weight rounded to bf16 the way the wgmma GEMM does is outside the GEMV's bound, inside the GEMM's
    wb = wdq.bfloat16().double()
    got = (x.double() @ wb.t() + bias.double()).bfloat16()
    ref2, bnd2 = R.wq_bounds(x, wdq, bias, torch.bfloat16, 16, 2 * K, w_round=2.0**-8 + R.U)
    R.assert_within(got, ref2, bnd2, "bf16 weights under the wgmma bound")
