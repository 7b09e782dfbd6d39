"""GPU tier: engine + flagship model end to end on one H100."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_native_library_is_loaded():
    from deepspeed_b200.ops import native
    lib = native.cuda()
    assert lib is not None
    maps = open("/proc/self/maps").read()
    assert "libdsb200_cuda.so" in maps


def test_llama_bf16_matches_hf_on_gpu():
    from transformers import LlamaConfig as HFC, LlamaForCausalLM as HFL
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=1024, num_hidden_layers=2)
    hf = HFL(HFC(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                 num_hidden_layers=cfg.num_hidden_layers, num_attention_heads=cfg.num_attention_heads,
                 num_key_value_heads=cfg.num_key_value_heads, max_position_embeddings=cfg.max_position_embeddings,
                 rms_norm_eps=cfg.rms_norm_eps, tie_word_embeddings=False)).cuda()
    m = LlamaForCausalLM(cfg).cuda()
    m.load_state_dict(LlamaForCausalLM.convert_hf_state_dict(hf.state_dict(), cfg))
    ids = torch.randint(0, cfg.vocab_size, (2, 128), device="cuda")
    ref = hf(input_ids=ids, labels=ids).loss  # fp32 reference
    mb = m.to(torch.bfloat16)
    loss = mb(ids, labels=ids)
    assert abs(loss.item() - ref.item()) < 5e-2, (loss.item(), ref.item())
    loss.backward()
    ref.backward()
    g = mb.model.layers[1].mlp.down_proj.weight.grad.float()
    gr = hf.model.layers[1].mlp.down_proj.weight.grad
    cos = torch.nn.functional.cosine_similarity(g.flatten(), gr.flatten(), dim=0)
    assert cos > 0.99, cos


@pytest.mark.parametrize("stage", [0, 2, 3])
def test_engine_trains_tiny_llama(stage):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    from deepspeed_b200.ops import native
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=1024, num_hidden_layers=2, checkpoint_layers=1)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    eng, _, _, _ = ds.initialize(model=model, config={
        "train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
        "optimizer": {"type": "AdamW", "params": {"lr": 2e-3}},
        "zero_optimization": {"stage": stage}, "gradient_clipping": 1.0 if stage == 2 else 0.0})
    ids = torch.randint(0, cfg.vocab_size, (2, 128), device="cuda")
    before = native.launch_count
    losses = []
    for _ in range(8):
        loss = eng(ids, labels=ids)
        eng.backward(loss)
        eng.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0] - 0.5, losses
    assert native.launch_count - before > 50
    if stage == 2:
        assert eng.get_global_grad_norm() is not None and eng.get_global_grad_norm() > 0


def test_checkpoint_roundtrip_gpu(tmp_path):
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    cfg = llama_config("tiny")
    conf = {"train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
            "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}}, "zero_optimization": {"stage": 3}}
    torch.manual_seed(0)
    with torch.device("cuda"):
        m1 = LlamaForCausalLM(cfg).to(torch.bfloat16)
    e1, _, _, _ = ds.initialize(model=m1, config=conf)
    ids = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda")
    for _ in range(2):
        loss = e1(ids, labels=ids)
        e1.backward(loss)
        e1.step()
    e1.save_checkpoint(str(tmp_path), tag="t1", client_state={"foo": 7})
    with torch.device("cuda"):
        m2 = LlamaForCausalLM(cfg).to(torch.bfloat16)
    e2, _, _, _ = ds.initialize(model=m2, config=conf)
    path, client = e2.load_checkpoint(str(tmp_path))
    assert path is not None and client["foo"] == 7 and e2.global_steps == 2
    l1 = e1(ids, labels=ids)
    l2 = e2(ids, labels=ids)
    assert abs(l1.item() - l2.item()) < 1e-3
    e1.backward(l1); e1.step()
    e2.backward(l2); e2.step()
    l1b, l2b = e1(ids, labels=ids).item(), e2(ids, labels=ids).item()
    assert abs(l1b - l2b) < 2e-3


@pytest.mark.parametrize("tier,clip", [("cpu", 1.0), ("cpu", 0.0), ("nvme", 1.0)])
def test_offload_tiers_match_device_optimizer(tier, clip, tmp_path):
    """ZeRO-3 with the optimizer state on the host (pinned memory, AVX Adam) or on NVMe-backed swap files streams through
    the same math as the on-device fused Adam (config #4 of BASELINE.json at toy size)."""
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    from deepspeed_b200.utils import safe_get_full_fp32_param
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=1024, num_hidden_layers=2)
    ids = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    results = {}
    for mode in ("device", tier):
        torch.manual_seed(0)
        with torch.device("cuda"):
            model = LlamaForCausalLM(cfg).to(torch.bfloat16)
        zo = {"stage": 3, "stage3_param_persistence_threshold": 0}
        conf = {"train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True}, "gradient_clipping": clip,
                "optimizer": {"type": "AdamW", "params": {"lr": 1e-3, "weight_decay": 0.1}}, "zero_optimization": zo}
        if mode == "cpu":
            zo["offload_optimizer"] = {"device": "cpu", "pin_memory": True}
        elif mode == "nvme":
            zo["offload_optimizer"] = {"device": "nvme", "nvme_path": str(tmp_path), "b200_swap_window": 100_000,
                                       "pipeline_read": True, "pipeline_write": True}
            conf["aio"] = {"block_size": 1 << 20, "queue_depth": 8}
        eng, *_ = ds.initialize(model=model, config=conf)
        if mode == "cpu":  # without clipping the CPU Adam of each unit runs on a worker thread while backward continues
            assert eng.optimizer.host_step_in_backward == (clip == 0.0)
        losses = []
        for _ in range(4):
            loss = eng(ids, labels=ids)
            eng.backward(loss)
            eng.step()
            losses.append(loss.item())
        results[mode] = (losses, [safe_get_full_fp32_param(p).float().cpu() for p in model.parameters()])
        eng.destroy()
    la, lb = results["device"][0], results[tier][0]
    assert all(abs(a - b) < 2e-2 for a, b in zip(la, lb)), (la, lb)
    worst = max((a - b).abs().max().item() for a, b in zip(results["device"][1], results[tier][1]))
    assert worst < 5e-3, worst


def test_mixtral_moe_and_phi3_zero2_train():
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    from deepspeed_b200.models.mixtral import MixtralConfig, MixtralForCausalLM
    torch.manual_seed(0)
    mcfg = MixtralConfig(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4,
                         num_key_value_heads=2, num_local_experts=4, num_experts_per_tok=2, max_position_embeddings=256)
    with torch.device("cuda"):
        moe = MixtralForCausalLM(mcfg).to(torch.bfloat16)
    eng, *_ = ds.initialize(model=moe, config={"train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
                                               "optimizer": {"type": "AdamW", "params": {"lr": 2e-3}},
                                               "zero_optimization": {"stage": 2}})
    ids = torch.randint(0, 512, (2, 64), device="cuda")
    first = last = None
    for _ in range(8):
        out = eng(ids, labels=ids)
        loss = out[0] if isinstance(out, tuple) else out
        eng.backward(loss)
        eng.step()
        first = first if first is not None else loss.item()
        last = loss.item()
    assert last < first - 0.3, (first, last)
    eng.destroy()
    # Phi-3-mini shaped (MHA, fused qkv/gate_up) under ZeRO-2 with gradient accumulation
    cfg = llama_config("phi3-mini", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=4,
                       vocab_size=1024, num_hidden_layers=2)
    with torch.device("cuda"):
        phi = LlamaForCausalLM(cfg).to(torch.bfloat16)
    eng, *_ = ds.initialize(model=phi, config={"train_micro_batch_size_per_gpu": 2, "gradient_accumulation_steps": 2,
                                               "bf16": {"enabled": True}, "gradient_clipping": 1.0,
                                               "optimizer": {"type": "AdamW", "params": {"lr": 2e-3}},
                                               "zero_optimization": {"stage": 2}})
    ids = torch.randint(0, 1024, (2, 64), device="cuda")
    losses = []
    for _ in range(12):
        loss = eng(ids, labels=ids)
        eng.backward(loss)
        eng.step()
        losses.append(loss.item())
    assert eng.global_steps == 6 and losses[-1] < losses[0] - 0.3, losses


def test_hybrid_engine_generate_between_training_steps_gpu():
    """RLHF loop on the device: bf16 ZeRO training steps interleaved with generation from the CURRENT weights through the
    ragged fused-kernel engine (paged KV, CUDA-graphed decode); greedy tokens must match the model's own no-cache decode."""
    import deepspeed_b200 as ds
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    from deepspeed_b200.runtime.hybrid_engine import DeepSpeedHybridEngine
    torch.manual_seed(0)
    cfg = llama_config("tiny", hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2,
                       vocab_size=512, num_hidden_layers=2, max_position_embeddings=256)
    with torch.device("cuda"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16)
    eng, *_ = ds.initialize(model=model, config={
        "train_micro_batch_size_per_gpu": 2, "bf16": {"enabled": True},
        "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}}, "zero_optimization": {"stage": 2},
        "hybrid_engine": {"enabled": True, "max_out_tokens": 64, "release_inference_cache": True}})
    assert isinstance(eng, DeepSpeedHybridEngine)
    prompt = torch.randint(0, cfg.vocab_size, (2, 9), device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    g = torch.Generator(device="cuda").manual_seed(1)
    agree = []
    for round_ in range(2):
        out = eng.generate(prompt, max_new_tokens=6)
        ref = model.generate_greedy(prompt, max_new_tokens=6)
        agree.append((out[:, :prompt.shape[1] + 6] == ref).float().mean().item())
        for _ in range(2):
            ids = torch.randint(0, cfg.vocab_size, (2, 64), device="cuda", generator=g)
            loss = eng(ids, labels=ids)
            eng.backward(loss[0] if isinstance(loss, tuple) else loss)
            eng.step()
    # bf16 kernels vs the training-path kernels: near ties may flip a token, the bulk must agree
    assert min(agree) > 0.8, agree
    assert eng._packed_at_step == 2 and eng.get_latency_report()["generate_s"] > 0


def test_exact_size_pinned_arena_and_offload_step():
    """ops/pinned.py: big offload arenas are page-locked at their exact size (torch's pinned allocator rounds to a power of
    two), report ``is_pinned`` and copy asynchronously; a ZeRO-3 + CPU-offload step runs on top of them."""
    import deepspeed_b200 as ds
    from deepspeed_b200.ops import pinned
    n = (300 << 20) // 4 + 12345  # just over the native-allocation threshold, deliberately not a power of two
    before = pinned.live_bytes()
    t = pinned.pinned_empty(n, torch.float32)
    assert t.is_pinned() and t.numel() == n and pinned.live_bytes() - before == n * 4
    src = torch.randn(n, device="cuda")
    t.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    torch.testing.assert_close(t, src.cpu())
    back = t.to("cuda", non_blocking=True)
    torch.cuda.synchronize()
    torch.testing.assert_close(back, src)
    del t, back
    import gc
    gc.collect()
    assert pinned.live_bytes() == before
    pinned_threshold = pinned.THRESHOLD_BYTES
    pinned.THRESHOLD_BYTES = 1 << 16  # force the engine's (small) arenas through the native allocator too
    try:
        torch.manual_seed(0)
        model = torch.nn.Sequential(torch.nn.Linear(512, 1024), torch.nn.GELU(), torch.nn.Linear(1024, 512)).cuda().bfloat16()
        conf = {"train_micro_batch_size_per_gpu": 4, "bf16": {"enabled": True},
                "optimizer": {"type": "AdamW", "params": {"lr": 1e-3}},
                "zero_optimization": {"stage": 3, "offload_optimizer": {"device": "cpu", "pin_memory": True}}}
        eng, *_ = ds.initialize(model=model, config=conf)
        assert eng.optimizer.master.is_pinned() and pinned.live_bytes() > before
        x = torch.randn(4, 512, device="cuda").bfloat16()
        l0 = None
        for _ in range(5):
            loss = eng(x).float().pow(2).mean()
            eng.backward(loss)
            eng.step()
            l0 = l0 if l0 is not None else loss.item()
        assert loss.item() < l0
        eng.destroy()
    finally:
        pinned.THRESHOLD_BYTES = pinned_threshold
