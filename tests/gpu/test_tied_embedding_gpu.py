"""H100: the native embedding backward and tied-embedding Llama training under ZeRO-3.

* ``transformer_ops.embedding_bwd_`` against float64 with a per-element bound (fp32 summation over each id's rows plus
  half an ulp of the output), over token counts, widths, vocabularies, id distributions (uniform, one hot id, one id
  everywhere) and bf16 / fp32 gradient views;
* rows whose id does not occur keep a sentinel bit for bit; two runs are bit-identical;
* operands the kernel refuses (a width that is not a multiple of 8, a misaligned buffer) run the torch path with the same
  semantics;
* ``llama3.2-1b`` cut to 2 layers (its real vocabulary and width), ZeRO-3 with every unit sharded: the step fused into
  backward tracks the unfused engine, and the model learns a bigram stream; the same on 2 GPUs where there are two.
"""
import math

import pytest
import torch

from tests.common import run_distributed

pytestmark = pytest.mark.gpu

U = 2.0**-24
HALF_ULP = {torch.bfloat16: 2.0**-8, torch.float32: 2.0**-24}


def _ids(kind, T, Vs, g):
    if kind == "uniform":
        return torch.randint(0, Vs, (T, ), generator=g, device="cuda")
    if kind == "hot":  # half the tokens on one id (padding / BOS), the rest uniform
        ids = torch.randint(0, Vs, (T, ), generator=g, device="cuda")
        ids[torch.rand(T, generator=g, device="cuda") < 0.5] = Vs // 2
        return ids
    return torch.full((T, ), Vs - 1, dtype=torch.long, device="cuda")


def _check(T, H, Vs, kind, out_dtype, dy_dtype=torch.bfloat16, seed=0):
    from deepspeed_b200.ops.kernels.transformer_ops import embedding_bwd_
    g = torch.Generator("cuda").manual_seed(seed)
    ids = _ids(kind, T, Vs, g)
    dy = torch.randn(T, H, generator=g, device="cuda").to(dy_dtype)
    sentinel = -3.25
    out = torch.full((Vs, H), sentinel, dtype=out_dtype, device="cuda")
    uniq = torch.unique(ids)
    out[uniq] = torch.randn(uniq.numel(), H, generator=g, device="cuda").to(out_dtype)  # prior contribution on touched rows
    prior = out[uniq].double()
    embedding_bwd_(dy, ids, out)
    # float64 reference on the touched rows only
    inv = torch.searchsorted(uniq, ids)
    want = prior.clone().index_add_(0, inv, dy.double())
    mag = prior.abs().index_add_(0, inv, dy.double().abs())
    n = torch.zeros(uniq.numel(), dtype=torch.float64, device="cuda").index_add_(
        0, inv, torch.ones(T, dtype=torch.float64, device="cuda"))
    got = out[uniq].double()
    bound = (n[:, None] + 2) * U * mag + HALF_ULP[out_dtype] * want.abs()
    err = (got - want).abs()
    assert bool((err <= bound).all()), (T, H, Vs, kind, out_dtype, float((err - bound).max()))
    out[uniq] = sentinel
    assert bool((out == sentinel).all()), "rows of ids that do not occur were written"


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("kind", ["uniform", "hot", "all_equal"])
@pytest.mark.parametrize("Vs", [97, 128256])
@pytest.mark.parametrize("H", [64, 2048, 3072, 4096])
@pytest.mark.parametrize("T", [1, 7, 4096, 8192])
def test_embedding_bwd_matches_float64(T, H, Vs, kind, out_dtype):
    _check(T, H, Vs, kind, out_dtype)


@pytest.mark.parametrize("dy_dtype", [torch.float16, torch.float32])
def test_embedding_bwd_other_gradient_dtypes(dy_dtype):
    _check(4096, 2048, 1000, "hot", torch.float32, dy_dtype)


def test_embedding_bwd_is_bit_reproducible():
    from deepspeed_b200.ops.kernels.transformer_ops import embedding_bwd_
    g = torch.Generator("cuda").manual_seed(1)
    for kind in ("uniform", "hot", "all_equal"):
        ids = _ids(kind, 8192, 128256, g)
        dy = torch.randn(8192, 2048, generator=g, device="cuda").bfloat16()
        a = torch.zeros(128256, 2048, dtype=torch.bfloat16, device="cuda")
        b = torch.zeros_like(a)
        embedding_bwd_(dy, ids, a)
        embedding_bwd_(dy, ids, b)
        assert torch.equal(a, b), kind


def test_refused_operands_fall_back_with_the_same_semantics():
    from deepspeed_b200.ops import native as N
    from deepspeed_b200.ops.kernels import transformer_ops as T
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, 50, (300, ), generator=g).cuda()
    calls = []
    orig = T._embedding_bwd_torch
    T._embedding_bwd_torch = lambda *a: calls.append(1) or orig(*a)
    try:
        for H, offset in ((36, 0), (64, 1)):  # width not a multiple of 8; an out view 2 bytes off a 16-byte boundary
            dy = torch.randn(300, H, generator=g).bfloat16().cuda()
            buf = torch.zeros(50 * H + 8, dtype=torch.bfloat16, device="cuda")
            out = buf[offset:offset + 50 * H].view(50, H)
            T.embedding_bwd_(dy, ids, out)
            want = torch.zeros(50, H, dtype=torch.float64, device="cuda").index_add_(0, ids, dy.double())
            assert torch.allclose(out.double(), want, atol=1e-6, rtol=2.0**-8)
        assert len(calls) == 2
        dy = torch.randn(300, 64, generator=g).bfloat16().cuda()
        assert N.cuda().dsb_embedding_bwd(T._p(dy), T._p(ids), T._p(ids), T._p(dy), T._p(buf[1:]), N.c_i64(300), 64,
                                          N.dt(dy), N.dt(buf), N.stream()) == -2
    finally:
        T._embedding_bwd_torch = orig


# ---------------------------------------------------------------------------------------------------------------------
# llama3.2-1b, 2 layers, ZeRO-3
# ---------------------------------------------------------------------------------------------------------------------
def _bigram_batches(steps, vocab=256, Bsz=2, S=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    probs = torch.softmax(torch.randn(vocab, vocab, generator=g) * 3, -1)
    out = []
    for _ in range(steps):
        ids = torch.empty(Bsz, S, dtype=torch.long)
        ids[:, 0] = torch.randint(0, vocab, (Bsz, ), generator=g)
        for t in range(1, S):
            ids[:, t] = torch.multinomial(probs[ids[:, t - 1]], 1, generator=g).squeeze(1)
        out.append(ids)
    return out


def _run(fused, batches):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("llama3.2-1b", num_hidden_layers=2, max_position_embeddings=8192)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    conf = {"train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
            "optimizer": {"type": "AdamW", "params": {"lr": 2e-3}},
            "zero_optimization": {"stage": 3, "stage3_param_persistence_threshold": 0,
                                  "b200_fused_optimizer_in_backward": fused}}
    eng, _, _, _ = ds.initialize(model=model, config=conf)
    assert eng.optimizer.fused_in_backward == fused
    r, w = ds.comm.get_rank(), ds.comm.get_world_size()
    losses = []
    for ids in batches:
        ids = ids.cuda()[r::w] if w > 1 else ids.cuda()
        loss = eng(ids, labels=ids)
        eng.backward(loss)
        eng.step()
        mean = loss.detach().float().clone()
        ds.comm.all_reduce(mean)
        losses.append(float(mean) / w)
    del eng
    torch.cuda.empty_cache()
    return losses


def _fused_vs_unfused_and_learning():
    batches = _bigram_batches(100, Bsz=2 * torch.distributed.get_world_size())
    fused = _run(True, batches)
    unfused = _run(False, batches)
    gap = max(abs(a - b) for a, b in zip(fused[:20], unfused[:20]))
    final = sum(fused[-10:]) / 10
    if torch.distributed.get_rank() == 0:
        print(f"[tied llama3.2-1b x2 layers] first {fused[0]:.4f} final {final:.4f} fused-unfused max gap (20 steps) "
              f"{gap:.2e}")
    assert abs(fused[0] - math.log(128256)) < 1.0, fused[0]  # not pinned at ln V: the head reads the real weight
    assert gap < 0.05, gap
    assert final < math.log(256), final  # the model learned which 256 tokens occur and their successors


def test_tied_llama32_1b_zero3_one_gpu():
    run_distributed(_fused_vs_unfused_and_learning, 1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_tied_llama32_1b_zero3_two_gpus():
    run_distributed(_fused_vs_unfused_and_learning, 2)
