"""GPU tier: QK-norm attention (Qwen3) on the fused ``transformer.cu`` kernels.

* ``qk_norm_rope_kernel`` / ``qk_norm_rope_bwd_kernel`` against float64 references with per-element bounds (head dim 64
  and 128, the Llama / Qwen3 head counts, 1 to 8192 tokens, positions null / explicit / per document, weights with zeros
  and negatives), guard bands around a strided buffer, V bit-untouched, dw bit-reproducible, and a mutation test showing
  that the bounds reject plausible bugs;
* every attention path with ``qk_norm`` (native dense, varlen and windowed; SDPA dense and per document) equals the
  unfused composition (the standalone kernels around the same attention call) bit for bit;
* activation-checkpointed layers with ``qk_norm`` equal no recompute bit for bit;
* a 2-layer ZeRO-3 Llama with ``qk_norm`` learns a bigram stream in bf16 and with ``fp8=True``, moving the norm weights;
  a tiny ``MixtralConfig(qk_norm=True)`` trains.
"""
import math

import pytest
import torch

from deepspeed_b200.ops import native as N
from deepspeed_b200.ops.kernels import transformer_ops as T
from tests.common import run_distributed
from tests.numerics import U, assert_bits_equal, assert_within, ulp

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
EPS = 1e-6


# ---------------------------------------------------------------------------------------------------------------------
# float64 references and bounds
# ---------------------------------------------------------------------------------------------------------------------
def _rot(x, c, s, sign):
    """Rotate-half of float64 ``x [T, H, d]`` by ``c / s [T, 1, d/2]`` (``sign`` -1: the transpose), and the magnitude
    ``|x c| + |partner s|`` of each output's two products."""
    h = x.shape[-1] // 2
    a, b = x[..., :h], x[..., h:]
    mag = torch.cat([(a * c).abs() + (b * s).abs(), (b * c).abs() + (a * s).abs()], -1)
    return torch.cat([a * c - b * s * sign, b * c + a * s * sign], -1), mag


def _cs(table, positions, tokens, seq_len):
    pos = positions.long() if positions is not None else torch.arange(tokens, device=table.cos.device) % seq_len
    return table.cos[pos].double()[:, None], table.sin[pos].double()[:, None]


def _weights(w_q, w_k, hq, hkv):
    return torch.cat([w_q.double().expand(hq, -1), w_k.double().expand(hkv, -1)])


def _rel(d):
    """fp32 relative error of the kernels' rstd and of the products around it, in U: the sum of squares (at most d
    terms), the eps add, rsqrtf (2 ulp) and two products; doubled."""
    return 2 * (d + 8)


def fwd_reference(x, w, c, s, eps, mutation=None):
    """``x [T, H, d]`` pre-norm heads (float64), ``w [H, d]``.  Returns ``(y, bound)``, the bound without the final
    rounding to the output's dtype."""
    d = x.shape[-1]
    rstd = 1.0 / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    if mutation == "eps_outside_rsqrt":
        rstd = 1.0 / torch.sqrt(x.pow(2).mean(-1, keepdim=True)) + eps
    n = x * rstd * w
    y, mag = _rot(n, c, s, 1.0)
    if mutation == "rope_before_norm":
        y = _rot(x * rstd, c, s, 1.0)[0] * w
    return y, mag * (_rel(d) + 4) * U


def bwd_reference(dy, x, w, c, s, eps, mutation=None):
    """Gradient of the forward for the output gradient ``dy [T, H, d]`` (float64).  Returns ``(dx, dx_bound, terms,
    terms_abs)``: the bound without the final rounding, and the terms ``rope^-1(dy) * xhat [T, H, d]`` summed into dw
    with magnitudes that cover their own error."""
    d = x.shape[-1]
    rstd = 1.0 / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    r, rmag = _rot(dy, c, s, 1.0 if mutation == "rotation_sign_bwd" else -1.0)
    xhat = x * rstd
    g = w * r
    m2 = (g * xhat).mean(-1, keepdim=True)
    dx = rstd * (g - xhat * m2)
    gmag = (w.abs() * rmag * xhat.abs()).mean(-1, keepdim=True)
    mag = rstd * (w.abs() * rmag + xhat.abs() * gmag)
    return dx, mag * (2 * _rel(d) + 16) * U, r * xhat, rmag * xhat.abs()


def dw_bound(terms_abs, ref, depth, dtype):
    """A sum of ``terms`` per column, ``depth`` additions deep, each term off by ``_rel`` U, rounded to ``dtype``."""
    d = terms_abs.shape[-1]
    return ulp(ref, dtype) + terms_abs * (depth + _rel(d) + 8) * U


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
def _data(Tn, hq, hkv, d, dtype, gen, pad=40):
    """A strided ``[Tn, (hq + 2 hkv) d]`` view into a guarded buffer (a row before, a row after, ``pad`` columns past
    each row, all NaN), heads scaled by 2**U(-12, 3) so mean(x^2) runs from far below eps to far above it (2**U(-6, 2)
    in fp16, whose range the gradient would leave)."""
    width = (hq + 2 * hkv) * d
    heads = hq + 2 * hkv
    lo, hi = (-6, 2) if dtype == torch.float16 else (-12, 3)
    x = torch.randn(Tn, heads, d, generator=gen, device="cuda")
    x = x * torch.exp2(torch.randint(lo, hi + 1, (Tn, heads, 1), generator=gen, device="cuda").float())
    store = torch.full((Tn + 2, width + pad), float("nan"), device="cuda", dtype=dtype)
    view = store[1:Tn + 1, :width]
    view.copy_(x.reshape(Tn, width))
    return store, view


def _norm_weights(d, gen, dtype):
    w = torch.randn(2, d, generator=gen, device="cuda") * 1.5
    w[0, ::7] = 0
    w[1, 3::11] = 0
    return w[0].to(dtype), w[1].to(dtype)


def _positions(kind, Tn, gen):
    if kind == "null":
        return None, max(Tn // 3, 1)
    if kind == "explicit":
        return torch.randint(0, 4096, (Tn, ), generator=gen, device="cuda", dtype=torch.int32), Tn
    cuts = torch.sort(torch.randint(0, Tn + 1, (5, ), generator=gen, device="cuda")).values
    cu = torch.cat([torch.zeros(1, device="cuda", dtype=torch.long), cuts, torch.full((1, ), Tn, device="cuda")])
    from deepspeed_b200.ops.attention import document_positions
    return document_positions(cu.to(torch.int32), Tn), Tn


def _check_kernels(Tn, hq, hkv, d, dtype, pos_kind, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    store, qkv = _data(Tn, hq, hkv, d, dtype, gen)
    w_q, w_k = _norm_weights(d, gen, dtype)
    positions, seq_len = _positions(pos_kind, Tn, gen)
    table = T.RotaryTable(d, 8192, 1e6, "cuda")
    qk = (hq + hkv) * d
    before = store.clone()
    x = qkv[:, :qk].double().view(Tn, hq + hkv, d)
    w = _weights(w_q, w_k, hq, hkv)
    c, s = _cs(table, positions, Tn, seq_len)

    raw = T.qk_norm_rope_inplace(qkv, hq, hkv, d, table, w_q, w_k, EPS, positions, seq_len)
    assert_bits_equal(raw, before[1:Tn + 1, :qk], "raw")
    y, b = fwd_reference(x, w, c, s, EPS)
    assert_within(qkv[:, :qk].view(Tn, hq + hkv, d), y, ulp(y, dtype) + b, "forward")
    after = store.clone()
    after[1:Tn + 1, :qk] = before[1:Tn + 1, :qk]
    assert_bits_equal(after, before, "guard bands and V")

    dstore, dqkv = _data(Tn, hq, hkv, d, dtype, gen)
    dbefore = dstore.clone()
    dy = dqkv[:, :qk].double().view(Tn, hq + hkv, d)
    dw_q, dw_k = T.qk_norm_rope_bwd_inplace(dqkv, raw, hq, hkv, d, table, w_q, w_k, EPS, positions, seq_len)
    dx, db, terms, terms_abs = bwd_reference(dy, x, w, c, s, EPS)
    assert_within(dqkv[:, :qk].view(Tn, hq + hkv, d), dx, ulp(dx, dtype) + db, "backward dQ|dK")
    dafter = dstore.clone()
    dafter[1:Tn + 1, :qk] = dbefore[1:Tn + 1, :qk]
    assert_bits_equal(dafter, dbefore, "backward guard bands and dV")
    grid = N.cuda().dsb_qk_norm_rope_bwd_grid(N.c_i64(Tn), hq + hkv, d, N.dt(dtype))
    lanes = d // (4 if dtype == torch.float32 else 8)  # per head; a CTA of 256 threads covers 256 / lanes heads a pass
    depth = math.ceil(Tn * (hq + hkv) / (grid * 256 // lanes)) + 16 + grid
    for name, got, sl in (("dw_q", dw_q, slice(0, hq)), ("dw_k", dw_k, slice(hq, hq + hkv))):
        ref = terms[:, sl].sum((0, 1))
        assert_within(got, ref, dw_bound(terms_abs[:, sl].sum((0, 1)), ref, depth, dtype), name)

    # bit-reproducible from run to run
    dqkv2 = dqkv.clone()
    dqkv2[:, :qk] = dbefore[1:Tn + 1, :qk]
    dw2 = T.qk_norm_rope_bwd_inplace(dqkv2, raw, hq, hkv, d, table, w_q, w_k, EPS, positions, seq_len)
    assert_bits_equal(dqkv2, dqkv, "dqkv rerun")
    assert_bits_equal(dw2[0], dw_q, "dw_q rerun")
    assert_bits_equal(dw2[1], dw_k, "dw_k rerun")


HEADS = [(4, 2), (16, 8), (24, 8), (32, 8)]


@pytest.mark.parametrize("pos_kind", ["null", "explicit", "documents"])
@pytest.mark.parametrize("Tn", [1, 37, 8192])
@pytest.mark.parametrize("hq,hkv", HEADS)
@pytest.mark.parametrize("d", [64, 128])
def test_kernels_bf16(d, hq, hkv, Tn, pos_kind):
    _check_kernels(Tn, hq, hkv, d, BF16, pos_kind, seed=d * 1000 + hq * 10 + Tn)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("Tn", [37, 1000])
def test_kernels_fp16_fp32(dtype, d, Tn):
    _check_kernels(Tn, 16, 8, d, dtype, "explicit", seed=d + Tn)


def test_other_head_dims_run_the_composition():
    """Head dim 96 and a partial rotary table have no kernel: the fp32 composition runs, with the same semantics."""
    gen = torch.Generator(device="cuda").manual_seed(0)
    for d, rot in ((96, 96), (128, 64)):
        store, qkv = _data(37, 4, 2, d, BF16, gen)
        w_q, w_k = _norm_weights(d, gen, BF16)
        table = T.RotaryTable(rot, 256, 1e4, "cuda")
        x = qkv[:, :6 * d].double().view(37, 6, d)
        raw = T.qk_norm_rope_inplace(qkv, 4, 2, d, table, w_q, w_k, EPS, None, 37)
        assert_bits_equal(raw, x.reshape(37, -1).to(BF16), "raw")
        rstd = 1.0 / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + EPS)
        n = x * rstd * _weights(w_q, w_k, 4, 2)
        c, s = _cs(table, None, 37, 37)
        y, _ = _rot(n[..., :rot], c, s, 1.0)
        y = torch.cat([y, n[..., rot:]], -1)
        assert_within(qkv[:, :6 * d].view(37, 6, d), y, 2 * ulp(y, BF16) + 1e-4 * y.abs(), f"d={d} rot={rot}")


MUTATIONS = ["rope_before_norm", "w_q_on_k_heads", "eps_outside_rsqrt", "rotation_sign_bwd"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_bounds_reject_mutations(mutation):
    """The bounds have teeth: for each plausible kernel bug, the real kernel's output falls outside the bound of a
    reference that carries that bug."""
    Tn, hq, hkv, d = 37, 4, 2, 128
    gen = torch.Generator(device="cuda").manual_seed(11)
    _, qkv = _data(Tn, hq, hkv, d, BF16, gen)
    w_q, w_k = _norm_weights(d, gen, BF16)
    positions, seq_len = _positions("explicit", Tn, gen)
    table = T.RotaryTable(d, 8192, 1e6, "cuda")
    qk = (hq + hkv) * d
    x = qkv[:, :qk].double().view(Tn, hq + hkv, d)
    w = _weights(w_q, w_k, hq, hkv)
    c, s = _cs(table, positions, Tn, seq_len)
    raw = T.qk_norm_rope_inplace(qkv, hq, hkv, d, table, w_q, w_k, EPS, positions, seq_len)
    got = qkv[:, :qk].view(Tn, hq + hkv, d)
    y, b = fwd_reference(x, w, c, s, EPS)
    assert_within(got, y, ulp(y, BF16) + b, "unmutated forward")
    _, dqkv = _data(Tn, hq, hkv, d, BF16, gen)
    dy = dqkv[:, :qk].double().view(Tn, hq + hkv, d)
    T.qk_norm_rope_bwd_inplace(dqkv, raw, hq, hkv, d, table, w_q, w_k, EPS, positions, seq_len)
    dgot = dqkv[:, :qk].view(Tn, hq + hkv, d)
    dx, db, _, _ = bwd_reference(dy, x, w, c, s, EPS)
    assert_within(dgot, dx, ulp(dx, BF16) + db, "unmutated backward")
    with pytest.raises(AssertionError):
        if mutation == "rotation_sign_bwd":
            dx, db, _, _ = bwd_reference(dy, x, w, c, s, EPS, mutation)
            assert_within(dgot, dx, ulp(dx, BF16) + db, mutation)
        else:
            wm = _weights(w_q, w_q, hq, hkv) if mutation == "w_q_on_k_heads" else w
            y, b = fwd_reference(x, wm, c, s, EPS, mutation)
            assert_within(got, y, ulp(y, BF16) + b, mutation)


# ---------------------------------------------------------------------------------------------------------------------
# attention paths
# ---------------------------------------------------------------------------------------------------------------------
PATHS = {
    "native-dense": dict(backend="native"),
    "native-varlen": dict(backend="native", cu=[0, 100, 256, 300, 301, 512]),
    "native-window": dict(backend="native", sliding_window=64),
    "native-varlen-window": dict(backend="native", cu=[0, 200, 512], sliding_window=48),
    "sdpa-dense": dict(backend="math"),
    "sdpa-documents": dict(backend="math", cu=[0, 100, 256, 300, 301, 512]),
}


@pytest.mark.parametrize("d,hq,hkv", [(128, 4, 2), (64, 8, 2)])
@pytest.mark.parametrize("path", sorted(PATHS))
def test_attention_path_equals_unfused_composition(path, d, hq, hkv):
    """The fused node against the standalone kernels around the same attention call without ``qk_norm`` / ``rope``:
    forward output, the rotated buffer, dqkv and both weight gradients bit for bit.  SDPA runs its math backend, whose
    backward is deterministic."""
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from deepspeed_b200.ops.attention import causal_attention, document_positions
    kw = dict(PATHS[path])
    cu = kw.pop("cu", None)
    B, S = 2, 256
    Tn = B * S
    gen = torch.Generator(device="cuda").manual_seed(5)
    base = (torch.randn(Tn, (hq + 2 * hkv) * d, generator=gen, device="cuda") * 2).to(BF16)
    w_q, w_k = (w.float().requires_grad_(True) for w in _norm_weights(d, gen, BF16))
    dout = torch.randn(Tn, hq * d, generator=gen, device="cuda").to(BF16)
    table = T.RotaryTable(d, 1024, 1e6, "cuda")
    cu_t = torch.tensor(cu, dtype=torch.int32) if cu is not None else None
    positions = document_positions(cu_t.cuda(), Tn) if cu is not None else None
    seq_len = Tn if cu is not None else S
    with sdpa_kernel([SDPBackend.MATH]):
        qkv = base.clone().requires_grad_(True)
        buf = qkv.view(Tn, -1) * 1  # the projection output is a non-leaf the node rotates in place
        out = causal_attention(buf, B, S, hq, hkv, d, table, None, cu_seqlens=cu_t, qk_norm=(w_q, w_k, EPS), **kw)
        out.backward(dout)

        ref_buf = base.clone()
        raw = T.qk_norm_rope_inplace(ref_buf, hq, hkv, d, table, w_q.detach(), w_k.detach(), EPS, positions, seq_len)
        ref_in = ref_buf.clone().requires_grad_(True)
        ref_out = causal_attention(ref_in * 1, B, S, hq, hkv, d, None, None, cu_seqlens=cu_t, **kw)
        ref_out.backward(dout)
    dref = ref_in.grad.clone()
    dw = T.qk_norm_rope_bwd_inplace(dref, raw, hq, hkv, d, table, w_q.detach(), w_k.detach(), EPS, positions, seq_len)
    assert_bits_equal(buf.detach(), ref_buf, "rotated buffer")
    assert_bits_equal(out.detach(), ref_out.detach(), "output")
    assert_bits_equal(qkv.grad, dref, "dqkv")
    assert_bits_equal(w_q.grad, dw[0], "dw_q")
    assert_bits_equal(w_k.grad, dw[1], "dw_k")


# ---------------------------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------------------------
def _model(**kw):
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    kw = {**dict(hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2, vocab_size=1024,
                 num_hidden_layers=2, max_position_embeddings=512, qk_norm=True), **kw}
    cfg = llama_config("tiny", **kw)
    with torch.device("cuda"):
        m = LlamaForCausalLM(cfg).to(BF16)
    with torch.no_grad():
        for layer in m.model.layers:
            layer.self_attn.q_norm.weight.uniform_(0.5, 1.5)
            layer.self_attn.k_norm.weight.uniform_(0.5, 1.5)
    return m


INPUTS = {"dense": {}, "packed": {"cu": [0, 100, 256, 300, 301, 512]}, "window": {"sliding_window": 64}}


@pytest.mark.parametrize("inputs", sorted(INPUTS))
def test_recompute_equals_no_recompute(inputs):
    kw = dict(INPUTS[inputs])
    cu = kw.pop("cu", None)
    cu = torch.tensor(cu, dtype=torch.int32) if cu is not None else None
    ids = torch.randint(0, 1024, (2, 256), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    res = []
    for layers in (0, 2):
        m = _model(checkpoint_layers=layers, attention_backend="native", **kw)
        m.train()
        loss = m(ids, labels=ids, cu_seqlens=cu)
        loss.backward()
        res.append((loss.detach(), {n: p.grad for n, p in m.named_parameters()}))
    (l0, g0), (l1, g1) = res
    assert_bits_equal(l1, l0, "loss")
    assert g0["model.layers.0.self_attn.q_norm.weight"].abs().sum() > 0
    for n in g0:
        assert_bits_equal(g1[n], g0[n], n)


def _bigram_batches(steps, vocab=256, B=2, S=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    probs = torch.softmax(torch.randn(vocab, vocab, generator=g) * 3, -1)
    out = []
    for _ in range(steps):
        ids = torch.empty(B, S, dtype=torch.long)
        ids[:, 0] = torch.randint(0, vocab, (B, ), generator=g)
        for t in range(1, S):
            ids[:, t] = torch.multinomial(probs[ids[:, t - 1]], 1, generator=g).squeeze(1)
        out.append(ids)
    return out


def _zero3_bigram():
    import deepspeed_b200 as ds
    from deepspeed_b200.utils.tensor_fragment import safe_get_full_fp32_param
    batches = _bigram_batches(100)
    for fp8 in (False, True):
        model = _model(vocab_size=256, fp8=fp8, checkpoint_layers=1)
        engine, _, _, _ = ds.initialize(model=model, config={
            "train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
            "optimizer": {"type": "AdamW", "params": {"lr": 2e-3}}, "zero_optimization": {"stage": 3}})
        norms = [p for n, p in engine.module.named_parameters() if n.endswith(("q_norm.weight", "k_norm.weight"))]
        assert len(norms) == 4
        w0 = [safe_get_full_fp32_param(p).detach().clone() for p in norms]
        losses = []
        for ids in batches:
            ids = ids.cuda()
            loss = engine(ids, labels=ids)
            engine.backward(loss)
            engine.step()
            losses.append(float(loss))
        final = sum(losses[-10:]) / 10
        print(f"[qk_norm zero3 fp8={fp8}] first {losses[0]:.4f} final {final:.4f}")
        assert all(math.isfinite(v) for v in losses), losses
        assert final < math.log(256) - 1.0, (fp8, final)
        for a, p in zip(w0, norms):
            moved = (safe_get_full_fp32_param(p) - a).abs().max()
            assert moved > 1e-3, (fp8, float(moved))
        del engine


def test_zero3_bigram_learns_with_qk_norm():
    run_distributed(_zero3_bigram, 1, (), timeout=600)


def test_mixtral_qk_norm_trains_one_step():
    from deepspeed_b200.models.mixtral import MixtralForCausalLM, mixtral_config
    torch.manual_seed(0)
    cfg = mixtral_config("tiny-moe", hidden_size=256, intermediate_size=384, num_attention_heads=4, num_key_value_heads=2,
                         vocab_size=1024, num_hidden_layers=2, num_local_experts=4, max_position_embeddings=512,
                         drop_tokens=False, qk_norm=True)
    model = MixtralForCausalLM(cfg).cuda().to(BF16)
    assert cfg.head_dim == 64
    norms = [p for n, p in model.named_parameters() if n.endswith(("q_norm.weight", "k_norm.weight"))]
    assert len(norms) == 4
    before = [p.detach().clone() for p in norms]
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2)
    ids = torch.randint(0, cfg.vocab_size, (2, 256), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    launches = N.launch_count
    loss = model(ids, labels=ids)
    loss.backward()
    assert math.isfinite(float(loss.detach())) and N.launch_count > launches
    for p in norms:
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()) and p.grad.abs().sum() > 0
    opt.step()
    assert all(not torch.equal(a, p.detach()) for a, p in zip(before, norms))
    with torch.no_grad():
        assert math.isfinite(float(model(ids, labels=ids)))
