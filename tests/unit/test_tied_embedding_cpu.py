"""CPU tier: Llama models whose LM head is tied to the input embedding, trained under ZeRO.

* the embedding node's torch path against float64 autograd: repeated ids, one id everywhere, ids 0 and V - 1, stored
  into a fresh gradient view (rows of absent ids zero) and accumulated onto one that already holds a contribution;
* with no engine, a tied ``LlamaForCausalLM`` matches an fp32 composition of ``nn.Embedding`` and a tied linear head;
* ZeRO stages 1, 2 and 3 on 2 ranks with every unit sharded, the step fused into backward and not, with gradient
  accumulation and with activation checkpointing: losses and fp32 master weights match one process of torch AdamW (the
  step-0 loss is the model's, not ln V), and the embedding unit is reduced exactly once per backward;
* once the unit order is traced, the head's fetch of the embedding unit is a prefetch hit;
* a tied HF ``LlamaForCausalLM`` (an ``nn.Linear`` head that reads the weight in backward) trains at stage 3 on 2 ranks;
* a stage-3 checkpoint of the tied model resumes to the uninterrupted run's next loss;
* ``convert_hf_state_dict`` fills the ``lm_head.weight`` that tied HF checkpoints omit.
"""
import copy
import math
import os
import weakref

import pytest
import torch
import torch.nn.functional as F

from tests.common import run_distributed

V = 2000
TINY = dict(vocab_size=V, hidden_size=64, intermediate_size=96, num_attention_heads=4, num_key_value_heads=2,
            tie_word_embeddings=True)


def _cfg(**kw):
    from deepspeed_b200.models.llama import llama_config
    return llama_config("tiny", **{**TINY, **kw})


# ---------------------------------------------------------------------------------------------------------------------
# the embedding node
# ---------------------------------------------------------------------------------------------------------------------
class _Owner:
    """Fake ZeRO owner of one weight: its gradient view, fresh until written, and the readiness marks."""

    def __init__(self, w, view, fresh):
        self.view, self.fresh, self.marks = view, fresh, 0
        w._ds_zero = weakref.ref(self)

    def grad_view_for(self, w):
        return self.view

    def grad_is_fresh(self, w):
        return self.fresh

    def mark_grad_ready(self, w):
        self.fresh = False
        self.marks += 1


IDS = {
    "repeated": lambda g: torch.tensor([[5, 3, 5, 5], [7, 3, 0, 5]]),
    "all_equal": lambda g: torch.full((3, 9), 11),
    "ends": lambda g: torch.tensor([[0, 96, 0, 96, 50]]),
    "random": lambda g: torch.randint(0, 97, (4, 33), generator=g),
}


@pytest.mark.parametrize("ids_kind", sorted(IDS))
@pytest.mark.parametrize("mode", ["no_owner", "fresh_view", "accumulate_view"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_embedding_node_torch_path_matches_float64(ids_kind, mode, dtype):
    from deepspeed_b200.ops.linear import embedding
    g = torch.Generator().manual_seed(0)
    Vs, H = 97, 16
    ids = IDS[ids_kind](g)
    w = torch.nn.Parameter(torch.randn(Vs, H, generator=g).to(dtype))
    dy = torch.randn(*ids.shape, H, generator=g).to(dtype)
    w64 = w.detach().double().requires_grad_()
    F.embedding(ids, w64).backward(dy.double())
    want = w64.grad
    owner = None
    if mode != "no_owner":
        prior = torch.randn(Vs, H, generator=g).to(dtype)
        view = torch.full((Vs, H), float("nan"), dtype=dtype) if mode == "fresh_view" else prior.clone()
        owner = _Owner(w, view, fresh=mode == "fresh_view")
        if mode == "accumulate_view":
            want = want + prior.double()
    y = embedding(ids, w)
    assert torch.equal(y, F.embedding(ids, w.detach()))
    y.backward(dy)
    got = w.grad if owner is None else owner.view
    if owner is not None:
        assert w.grad is None and owner.marks == 1
    seen = torch.zeros(Vs, dtype=torch.bool)
    seen[ids.reshape(-1)] = True
    if mode == "accumulate_view":  # rows of ids that do not occur: untouched, bit for bit
        assert torch.equal(got[~seen], prior[~seen])
    else:
        assert torch.equal(got[~seen].float(), torch.zeros_like(got[~seen].float()))
    # fp32 sums of at most 36 rows, then one rounding to the gradient's dtype
    n = ids.numel()
    bound = n * 2.0**-24 * (dy.double().abs().sum() + (prior.double().abs().max() if owner and mode != "fresh_view" else 0))
    half_ulp = 2.0**-8 if dtype == torch.bfloat16 else 2.0**-24
    err = (got.double() - want).abs()
    assert bool((err <= bound + half_ulp * want.abs() + 1e-30).all()), float(err.max())


# ---------------------------------------------------------------------------------------------------------------------
# the model without an engine
# ---------------------------------------------------------------------------------------------------------------------
def test_tied_llama_matches_fp32_composition():
    from deepspeed_b200.models.llama import LlamaForCausalLM, TiedEmbedding
    torch.manual_seed(0)
    cfg = _cfg()
    m = LlamaForCausalLM(cfg)
    assert isinstance(m.model.embed_tokens, TiedEmbedding) and m.lm_head.weight is m.model.embed_tokens.weight
    assert "lm_head.weight" in m.state_dict() and "model.embed_tokens.weight" in m.state_dict()
    ref = copy.deepcopy(m)
    ref.model.embed_tokens.__class__ = torch.nn.Embedding  # plain lookup, autograd's embedding backward
    ids = torch.randint(0, V, (2, 24))
    loss = m(ids, labels=ids)
    loss.backward()
    logits = F.linear(ref.model(ids), ref.lm_head.weight)
    rl = F.cross_entropy(logits[:, :-1].reshape(-1, V), ids[:, 1:].reshape(-1))
    rl.backward()
    torch.testing.assert_close(loss, rl, atol=1e-5, rtol=1e-5)
    for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        torch.testing.assert_close(p.grad, q.grad, atol=1e-5, rtol=1e-4, msg=n)


def test_untied_llama_keeps_plain_embedding_and_head():
    from deepspeed_b200.models.llama import LlamaForCausalLM
    m = LlamaForCausalLM(_cfg(tie_word_embeddings=False))
    assert type(m.model.embed_tokens) is torch.nn.Embedding and not m.lm_head.defer_ready


# ---------------------------------------------------------------------------------------------------------------------
# ZeRO on 2 ranks against one process of torch AdamW
# ---------------------------------------------------------------------------------------------------------------------
def _engine(model, stage, fused, gas=1):
    import deepspeed_b200 as ds
    conf = {"train_micro_batch_size_per_gpu": 2, "gradient_accumulation_steps": gas,
            "optimizer": {"type": "AdamW", "params": {"lr": 1e-3, "weight_decay": 0.1}},
            "zero_optimization": {"stage": stage, "stage3_param_persistence_threshold": 0,
                                  "b200_fused_optimizer_in_backward": fused}}
    eng, _, _, _ = ds.initialize(model=model, config=conf)
    return eng


def _train_tied(stage, fused, gas, ckpt, steps=3):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM
    from deepspeed_b200.utils import safe_get_full_fp32_param
    torch.manual_seed(0)
    cfg = _cfg(checkpoint_layers=ckpt)
    m = LlamaForCausalLM(cfg)
    ref = LlamaForCausalLM(cfg)
    ref.load_state_dict(m.state_dict())
    eng = _engine(m, stage, fused, gas)
    zo = eng.optimizer
    emb = zo.unit_of_param[id(m.model.embed_tokens.weight)]
    assert [n for n, _ in emb.u.borrowers] == ["lm_head"]
    assert zo.fused_in_backward == (fused and gas == 1)
    reduced = []
    orig = zo._reduce_unit

    def counting(rt):
        reduced.append(rt.u.index)
        return orig(rt)

    zo._reduce_unit = counting
    r, w = ds.comm.get_rank(), ds.comm.get_world_size()
    ropt = torch.optim.AdamW(ref.parameters(), lr=1e-3, weight_decay=0.1)
    g = torch.Generator().manual_seed(1)
    for step in range(steps):
        for _ in range(gas):
            ids = torch.randint(0, V, (2 * w, 32), generator=g)
            reduced.clear()
            loss = eng(ids[r * 2:(r + 1) * 2], labels=ids[r * 2:(r + 1) * 2])
            eng.backward(loss)
            assert reduced.count(emb.u.index) == 1, reduced
            eng.step()
            rl = sum(ref(ids[k * 2:(k + 1) * 2], labels=ids[k * 2:(k + 1) * 2]) for k in range(w)) / (w * gas)
            rl.backward()
            mean = loss.detach().clone()
            ds.comm.all_reduce(mean)
            assert abs(float(mean) / w - float(rl) * gas) < 1e-4, (step, float(mean) / w, float(rl) * gas)
            if step == 0:
                assert abs(float(mean) / w - math.log(V)) > 1e-3  # all-zero logits would give ln V
        ropt.step()
        ropt.zero_grad()
    worst = max((safe_get_full_fp32_param(p).cpu() - q).abs().max().item()
                for p, q in zip(m.parameters(), ref.parameters()))
    assert worst < 5e-5, worst


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("stage", [1, 2, 3])
def test_tied_llama_zero_matches_torch(stage, fused):
    run_distributed(_train_tied, 2, (stage, fused, 1, 0))


@pytest.mark.parametrize("stage", [2, 3])
def test_tied_llama_zero_grad_accumulation(stage):
    run_distributed(_train_tied, 2, (stage, True, 2, 0))


@pytest.mark.parametrize("fused", [True, False])
def test_tied_llama_zero3_checkpointed_layer(fused):
    run_distributed(_train_tied, 2, (3, fused, 1, 1))


def _prefetch_hit():
    os.environ["DSB200_ZERO_PROFILE"] = "1"
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM
    torch.manual_seed(0)
    m = LlamaForCausalLM(_cfg(num_hidden_layers=3))
    eng = _engine(m, 3, True)
    zo = eng.optimizer
    emb = zo.unit_of_param[id(m.model.embed_tokens.weight)]
    borrows = []
    orig = zo.fetch_unit

    def watch(rt, forward=True, prefetch=True, borrow=False):
        c = zo.param_profiler.event_counters
        hit, miss = c["fetch_hit"][0], c["fetch_miss"][0]
        orig(rt, forward, prefetch, borrow)
        if borrow:
            borrows.append((rt.u.index, c["fetch_hit"][0] - hit, c["fetch_miss"][0] - miss))

    zo.fetch_unit = watch
    r = ds.comm.get_rank()
    g = torch.Generator().manual_seed(1)
    for _ in range(3):
        ids = torch.randint(0, V, (4, 32), generator=g)
        loss = eng(ids[r * 2:(r + 1) * 2], labels=ids[r * 2:(r + 1) * 2])
        eng.backward(loss)
        eng.step()
    # one borrow per forward (the head's backward reads no weight); the first, untraced one gathers on demand
    assert borrows == [(emb.u.index, 0, 1), (emb.u.index, 1, 0), (emb.u.index, 1, 0)], borrows
    assert zo._trace[-1] == emb.u.index and zo._borrow_pos == {len(zo._trace) - 1}
    assert zo._trace[:-1] == sorted(set(zo._trace[:-1]))


def test_head_fetch_is_a_prefetch_hit_once_traced():
    run_distributed(_prefetch_hit, 2)


def _untied_trace():
    from deepspeed_b200.models.llama import LlamaForCausalLM
    torch.manual_seed(0)
    m = LlamaForCausalLM(_cfg(tie_word_embeddings=False))
    eng = _engine(m, 3, True)
    zo = eng.optimizer
    assert all(not u.borrowers for u in zo.units)
    ids = torch.randint(0, V, (2, 32))
    for _ in range(2):
        eng.backward(eng(ids, labels=ids))
        eng.step()
    assert zo._trace == [u.index for u in zo.units] and not zo._borrow_pos


def test_untied_llama_has_no_borrowers_and_the_same_trace():
    run_distributed(_untied_trace, 2)


# ---------------------------------------------------------------------------------------------------------------------
# a tied HF model: its nn.Linear head reads the weight in backward
# ---------------------------------------------------------------------------------------------------------------------
def _hf_model():
    from transformers import LlamaConfig as HFConfig, LlamaForCausalLM as HF
    torch.manual_seed(0)
    return HF(HFConfig(vocab_size=V, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=4,
                       num_key_value_heads=2, max_position_embeddings=64, tie_word_embeddings=True,
                       attn_implementation="eager")).float()


def _hf_tied_stage3():
    import deepspeed_b200 as ds
    from deepspeed_b200.utils import safe_get_full_fp32_param
    m = _hf_model()
    ref = copy.deepcopy(m)
    assert m.lm_head.weight is m.model.embed_tokens.weight
    eng = _engine(m, 3, True)
    emb = eng.optimizer.unit_of_param[id(m.model.embed_tokens.weight)]
    assert [n for n, _ in emb.u.borrowers] == ["lm_head"]
    r, w = ds.comm.get_rank(), ds.comm.get_world_size()
    ropt = torch.optim.AdamW(ref.parameters(), lr=1e-3, weight_decay=0.1)
    g = torch.Generator().manual_seed(1)
    for step in range(3):
        ids = torch.randint(0, V, (2 * w, 16), generator=g)
        loss = eng(input_ids=ids[r * 2:(r + 1) * 2], labels=ids[r * 2:(r + 1) * 2]).loss
        eng.backward(loss)
        eng.step()
        rl = sum(ref(input_ids=ids[k * 2:(k + 1) * 2], labels=ids[k * 2:(k + 1) * 2]).loss for k in range(w)) / w
        rl.backward()
        ropt.step()
        ropt.zero_grad()
        mean = loss.detach().clone()
        ds.comm.all_reduce(mean)
        assert abs(float(mean) / w - float(rl)) < 1e-4, (step, float(mean) / w, float(rl))
    worst = max((safe_get_full_fp32_param(p).cpu() - q).abs().max().item()
                for p, q in zip(m.parameters(), ref.parameters()))
    assert worst < 5e-5, worst


def test_hf_tied_llama_zero3_matches_torch():
    run_distributed(_hf_tied_stage3, 2)


# ---------------------------------------------------------------------------------------------------------------------
# checkpoint and HF interop
# ---------------------------------------------------------------------------------------------------------------------
def _ckpt_run(d, resume):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM
    torch.manual_seed(123 if resume else 0)  # the resumed run gets everything from the checkpoint
    eng = _engine(LlamaForCausalLM(_cfg()), 3, True)
    r = ds.comm.get_rank()
    g = torch.Generator().manual_seed(1)
    batches = [torch.randint(0, V, (4, 32), generator=g) for _ in range(4)]

    def step(ids):
        loss = eng(ids[r * 2:(r + 1) * 2], labels=ids[r * 2:(r + 1) * 2])
        eng.backward(loss)
        eng.step()
        return float(loss)

    if resume:
        path, _ = eng.load_checkpoint(d)
        assert path is not None and eng.global_steps == 3
        got = step(batches[3])
        want = torch.load(os.path.join(d, f"next_loss_{r}.pt"))
        assert got == want, (got, want)
        return
    for ids in batches[:3]:
        step(ids)
    eng.save_checkpoint(d, tag="t3")
    torch.save(step(batches[3]), os.path.join(d, f"next_loss_{r}.pt"))


def test_tied_llama_zero3_checkpoint_round_trip(tmp_path):
    run_distributed(_ckpt_run, 2, (str(tmp_path), False))
    run_distributed(_ckpt_run, 2, (str(tmp_path), True))


def test_convert_hf_state_dict_fills_tied_head():
    from deepspeed_b200.models.llama import LlamaConfig, LlamaForCausalLM
    hf = _hf_model().eval()
    sd = {k: v for k, v in hf.state_dict().items() if k != "lm_head.weight"}
    cfg = LlamaConfig(vocab_size=V, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, max_position_embeddings=64, rope_theta=hf.config.rope_parameters["rope_theta"]
                      if hasattr(hf.config, "rope_parameters") else hf.config.rope_theta, tie_word_embeddings=True,
                      rms_norm_eps=hf.config.rms_norm_eps)
    m = LlamaForCausalLM(cfg).float().eval()
    m.load_state_dict(LlamaForCausalLM.convert_hf_state_dict(sd, cfg))
    assert m.lm_head.weight is m.model.embed_tokens.weight
    ids = torch.randint(0, V, (2, 20), generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        torch.testing.assert_close(m(ids), hf(ids).logits, atol=2e-5, rtol=1e-4)
