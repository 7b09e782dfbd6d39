"""Cost of QK-norm (Qwen3) in attention, on one GPU.

``--mode kernel``: the fused QK-norm + RoPE forward and backward (``transformer.cu:qk_norm_rope_kernel`` /
``qk_norm_rope_bwd_kernel``) against ``rope_qk_inplace`` alone (the pass it replaces) and against the fp32 torch
composition, at the Llama-3.2-3B (24/8 heads) and Qwen3-8B (32/8 heads) attention shapes, head dim 128, bf16, T = 8192
tokens.  CUDA events over many launches; bytes are what each pass must move (fused forward: read Q|K, write Q|K and the
saved pre-norm copy; fused backward: read dQ|dK and the copy, write dQ|dK; RoPE: read and write Q|K).

``--mode step --qk-norm {0,1}``: ``bench.py``'s default configuration (Llama-3.2-3B, ZeRO-3, sequence 4096, micro-batch 2,
bf16, the same optimizer and activation-recompute policy) with ``LlamaConfig.qk_norm`` set, one arm per process.

Without ``--mode`` it runs the kernel benchmark, then the step arms alternately, twice each (qk_norm 0, 1, 0, 1), each in
its own process.  Every result is one JSON line with the card name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"llama3.2-3b": (24, 8, 128), "qwen3-8b": (32, 8, 128)}


def _smi():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                               "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa
        return f"unavailable: {type(ex).__name__}"


def _time(torch, fn, reset, iters=50, warmup=5):
    """Mean milliseconds of ``fn`` over ``iters`` launches; ``reset`` restores the inputs (untimed, between launches)."""
    for _ in range(warmup):
        reset()
        fn()
    torch.cuda.synchronize()
    total = 0.0
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(iters):
        reset()
        s.record()
        fn()
        e.record()
        e.synchronize()
        total += s.elapsed_time(e)
    return total / iters


def kernel_bench(tokens):
    import torch
    from deepspeed_b200.ops.kernels import transformer_ops as T
    dev = "cuda"
    for name, (hq, hkv, d) in SHAPES.items():
        g = torch.Generator(device=dev).manual_seed(0)
        width = (hq + 2 * hkv) * d
        base = torch.randn(tokens, width, generator=g, device=dev).bfloat16()
        dbase = torch.randn(tokens, width, generator=g, device=dev).bfloat16()
        w_q = (1 + 0.1 * torch.randn(d, generator=g, device=dev)).bfloat16()
        w_k = (1 + 0.1 * torch.randn(d, generator=g, device=dev)).bfloat16()
        table = T.RotaryTable(d, 8192, 1e6, dev)
        qkv, dqkv = base.clone(), dbase.clone()
        raw = T.qk_norm_rope_inplace(qkv.clone(), hq, hkv, d, table, w_q, w_k, 1e-6, None, 4096)
        heads = T._qk_heads(qkv, hq, hkv, d)
        dheads = T._qk_heads(dqkv, hq, hkv, d)

        def reset():
            qkv.copy_(base)
            dqkv.copy_(dbase)

        qk_bytes = tokens * (hq + hkv) * d * 2
        arms = {
            "fused_fwd": (lambda: T.qk_norm_rope_inplace(qkv, hq, hkv, d, table, w_q, w_k, 1e-6, None, 4096), 3),
            "fused_bwd": (lambda: T.qk_norm_rope_bwd_inplace(dqkv, raw, hq, hkv, d, table, w_q, w_k, 1e-6, None, 4096),
                          3),
            "rope_fwd": (lambda: T.rope_qk_inplace(qkv, hq, hkv, d, table, None, 4096), 2),
            "rope_bwd": (lambda: T.rope_qk_inplace(dqkv, hq, hkv, d, table, None, 4096, backward=True), 2),
            "torch_fwd": (lambda: T._qk_norm_rope_torch(heads, hq, table, w_q, w_k, 1e-6, None, 4096), 3),
            "torch_bwd": (lambda: T._qk_norm_rope_bwd_torch(dheads, raw, hq, table, w_q, w_k, 1e-6, None, 4096), 3),
        }
        res = {}
        for arm, (fn, passes) in arms.items():
            ms = _time(torch, fn, reset)
            res[arm] = {"ms": round(ms, 4), "GB_per_s": round(passes * qk_bytes / ms / 1e6, 1)}
        # the fused kernels give what the unfused path gives: compare with the composition on the same inputs
        a, b = base.clone(), base.clone()
        T.qk_norm_rope_inplace(a, hq, hkv, d, table, w_q, w_k, 1e-6, None, 4096)
        T._qk_norm_rope_torch(T._qk_heads(b, hq, hkv, d), hq, table, w_q, w_k, 1e-6, None, 4096)
        diff = (a.float() - b.float()).abs().max().item()
        print(json.dumps({"mode": "kernel", "shape": name, "tokens": tokens, "hq": hq, "hkv": hkv, "head_dim": d,
                          "dtype": "bf16", "qk_mib": round(qk_bytes / 2**20, 1), **res,
                          "max_abs_diff_vs_composition": diff, "device": torch.cuda.get_device_name(0),
                          "nvidia_smi": _smi()}), flush=True)


def step_bench(qk_norm, model, seq, micro_batch, steps, warmup):
    import torch
    import deepspeed_b200 as ds
    from bench import pick_checkpoint_layers
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    ds.init_distributed(verbose=False)
    cfg = llama_config(model, qk_norm=bool(qk_norm))
    cfg.checkpoint_layers = pick_checkpoint_layers(torch, cfg, micro_batch, seq, 1, 3, None)
    config = {
        "train_micro_batch_size_per_gpu": micro_batch,
        "gradient_accumulation_steps": 1,
        "gradient_clipping": 0.0,
        "bf16": {"enabled": True},
        "optimizer": {"type": "AdamW", "params": {"lr": 1e-5, "betas": [0.9, 0.95], "eps": 1e-8, "weight_decay": 0.1}},
        "zero_optimization": {"stage": 3, "overlap_comm": True},
        "steps_per_print": 10**9,
    }
    torch.manual_seed(1234)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    with torch.device("cuda"):
        net = LlamaForCausalLM(cfg)
    torch.set_default_dtype(prev)
    engine = ds.initialize(model=net, config=config)[0]
    g = torch.Generator().manual_seed(0)
    batches = [torch.randint(0, cfg.vocab_size, (micro_batch, seq), generator=g).cuda() for _ in range(4)]

    def step(i):
        loss = engine(batches[i % 4], labels=batches[i % 4])
        engine.backward(loss)
        engine.step()
        return loss

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(steps):
        loss = step(warmup + i)
    e.record()
    torch.cuda.synchronize()
    sec = s.elapsed_time(e) / 1e3
    print(json.dumps({
        "mode": "step", "model": model, "qk_norm": bool(qk_norm), "seq": seq, "micro_batch": micro_batch,
        "zero_stage": 3, "checkpoint_layers": cfg.checkpoint_layers, "steps": steps, "warmup": warmup,
        "tokens_per_s": round(steps * micro_batch * seq / sec, 1), "step_ms": round(1e3 * sec / steps, 2),
        "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2), "loss_after": float(loss.detach()),
        "device": torch.cuda.get_device_name(0), "nvidia_smi": _smi()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["kernel", "step"], default=None)
    ap.add_argument("--qk-norm", type=int, choices=[0, 1], default=1)
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--model", default="llama3.2-3b")
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--micro-batch", type=int, default=2)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_qk_norm needs a CUDA device")
    torch.cuda.set_device(0)
    if args.mode == "kernel":
        kernel_bench(args.tokens)
    elif args.mode == "step":
        step_bench(args.qk_norm, args.model, args.seq, args.micro_batch, args.steps, args.warmup)
    else:
        kernel_bench(args.tokens)
        for qk in (0, 1, 0, 1):
            subprocess.run([sys.executable, os.path.abspath(__file__), "--mode", "step", "--qk-norm", str(qk), "--model",
                            args.model, "--seq", str(args.seq), "--micro-batch", str(args.micro_batch), "--steps",
                            str(args.steps), "--warmup", str(args.warmup)], check=True)


if __name__ == "__main__":
    main()
