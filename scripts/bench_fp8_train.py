"""Llama training step with or without FP8 projections: ``bench.py``'s default configuration (Llama-3.2-3B, ZeRO-3,
sequence 4096, micro-batch 2, bf16, the same optimizer and activation-recompute policy) with ``LlamaConfig.fp8`` set by
``--fp8``.  One arm per process: run ``--fp8 0`` and ``--fp8 1`` alternately, at least twice each, to see the spread.
Reports tokens/s over the timed steps (CUDA events), peak device memory, the loss after the timed steps, and the card
name and power limit.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fp8", type=int, choices=[0, 1], required=True)
    ap.add_argument("--model", default="llama3.2-3b")
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--micro-batch", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_train needs a CUDA device")
    torch.cuda.set_device(0)
    import deepspeed_b200 as ds
    from bench import pick_checkpoint_layers
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    ds.init_distributed(verbose=False)
    cfg = llama_config(args.model, fp8=bool(args.fp8))
    cfg.checkpoint_layers = pick_checkpoint_layers(torch, cfg, args.micro_batch, args.seq, 1, 3, None)
    config = {
        "train_micro_batch_size_per_gpu": args.micro_batch,
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
        model = LlamaForCausalLM(cfg)
    torch.set_default_dtype(prev)
    engine = ds.initialize(model=model, config=config)[0]
    g = torch.Generator().manual_seed(0)
    batches = [torch.randint(0, cfg.vocab_size, (args.micro_batch, args.seq), generator=g).cuda() for _ in range(4)]

    def step(i):
        loss = engine(batches[i % 4], labels=batches[i % 4])
        engine.backward(loss)
        engine.step()
        return loss

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(args.steps):
        loss = step(args.warmup + i)
    e.record()
    torch.cuda.synchronize()
    sec = s.elapsed_time(e) / 1e3
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa
        smi = f"unavailable: {type(ex).__name__}"
    print(json.dumps({
        "model": args.model, "fp8": bool(args.fp8), "seq": args.seq, "micro_batch": args.micro_batch, "zero_stage": 3,
        "checkpoint_layers": cfg.checkpoint_layers, "steps": args.steps, "warmup": args.warmup,
        "tokens_per_s": round(args.steps * args.micro_batch * args.seq / sec, 1), "step_ms": round(1e3 * sec / args.steps, 2),
        "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2), "loss_after": float(loss.detach()),
        "device": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)


if __name__ == "__main__":
    main()
