"""Tensorwise against blockwise FP8 scaling, kernels and training step.

Part ``kernels``: the products of one decoder layer of Llama-3.2-3B and Llama-3-8B at 8192 tokens (forward, dgrad and
wgrad of qkv, o, gate|up with SwiGLU, down with dSwiGLU on its dgrad).  For each, on operands already cast, the
tensorwise kernel (``fp8_matmul``) and the blockwise kernel (``fp8_matmul_block``); the casts the autograd node makes
for that product alone -- tensorwise an amax pass and a cast pass per operand, blockwise one pass per operand (forward:
x row-major + transposed and W; dgrad: dY row-major + transposed and W^T; wgrad reuses the transposed copies) -- and
kernel plus casts.  TFLOP/s count 2 M N K.  Every figure is the median of ``--repeats`` windows of ``--iters`` launches
between CUDA events, after a warm-up; the two recipes alternate window by window.

Part ``train``: ``bench_fp8_train.py``'s configuration (Llama-3.2-3B, ZeRO-3, sequence 4096, micro-batch 2) with three
arms -- bf16, tensorwise, blockwise -- one process per run, alternated ``--rounds`` times: tokens/s, peak memory and the
loss after the same number of steps.

The card's name and power limit are read in the same run and printed with the results.  Needs a CUDA device; prints one
JSON line per row and a closing JSON object."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

MODELS = {"llama3.2-3b": dict(H=3072, I=8192, qkv=5120), "llama3-8b": dict(H=4096, I=14336, qkv=6144)}
ARMS = {"bf16": dict(fp8=False), "tensorwise": dict(fp8=True, fp8_recipe="tensorwise"),
        "blockwise": dict(fp8=True, fp8_recipe="blockwise")}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.max_limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", "0"], capture_output=True, text=True, timeout=30)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or f"unavailable: {q.stderr.strip()[:80]}"}


def window(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def alternated(fns, warmup, iters, repeats):
    """Median ms per call of each function in ``fns`` (a dict), their timing windows interleaved."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    times = {k: [] for k in fns}
    for _ in range(repeats):
        for k, fn in fns.items():
            times[k].append(window(fn, iters))
    return {k: statistics.median(v) for k, v in times.items()}


def problems(T, H, I, qkv):
    out = []
    for name, n, k in (("qkv", qkv, H), ("o", H, H), ("gate_up", 2 * I, H), ("down", H, I)):
        out += [(name, "fwd", T, n, k), (name, "dgrad", T, k, n), (name, "wgrad", n, k, T)]
    return out


def bench_one(name, pas, M, N, Kd, args):
    """One product ``[M, Kd] x [N, Kd]^T``; for the gate|up forward ``N`` is ``2 I``."""
    from deepspeed_b200.ops import fp8 as F8
    from deepspeed_b200.ops.kernels import fp8_ops
    from deepspeed_b200.ops.kernels import gemm_sm100 as K
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    swiglu, dswiglu = name == "gate_up" and pas == "fwd", name == "down" and pas == "dgrad"
    afmt = F8.E4M3 if pas == "fwd" else F8.E5M2
    tw = lambda x, fmt, row, col: fp8_ops.fp8_cast(x, fp8_ops.fp8_amax(x), fmt, rowwise=row, colwise=col)
    bw = fp8_ops.fp8_cast_block
    if pas == "fwd":  # x [T, K] and W [N, K], both row-major sources
        a = torch.randn(M, Kd, generator=g, device=dev).bfloat16()
        b = (torch.randn(N, Kd, generator=g, device=dev) * 0.02).bfloat16()
        a8, _, sa = tw(a, afmt, True, False)
        b8, _, sb = tw(b, F8.E4M3, True, False)
        a8b, sab, _, _ = bw(a, afmt, row="strip")
        b8b, sbb, _, _ = bw(b, F8.E4M3, row="block")
        casts = {"tensorwise": lambda: (tw(a, afmt, True, True), tw(b, F8.E4M3, True, False)),
                 "blockwise": lambda: (bw(a, afmt, row="strip", col="block"), bw(b, F8.E4M3, row="block"))}
    elif pas == "dgrad":  # dY [T, K] and W [K, N]: B = W^T
        a = torch.randn(M, Kd, generator=g, device=dev).bfloat16()
        w = (torch.randn(Kd, N, generator=g, device=dev) * 0.02).bfloat16()
        a8, _, sa = tw(a, afmt, True, False)
        _, b8, sb = tw(w, F8.E4M3, False, True)
        a8b, sab, _, _ = bw(a, afmt, row="strip")
        _, _, b8b, sbb = bw(w, F8.E4M3, row=None, col="block")
        casts = {"tensorwise": lambda: (tw(a, afmt, True, True), tw(w, F8.E4M3, False, True)),
                 "blockwise": lambda: (bw(a, afmt, row="strip", col="strip"), bw(w, F8.E4M3, row=None, col="block"))}
    else:  # dW = dY^T X over T = Kd tokens: both operands are transposed copies made by the other two products' casts
        dy = torch.randn(Kd, M, generator=g, device=dev).bfloat16()
        x = torch.randn(Kd, N, generator=g, device=dev).bfloat16()
        _, a8, sa = tw(dy, afmt, False, True)
        _, b8, sb = tw(x, F8.E4M3, False, True)
        _, _, a8b, sab = bw(dy, afmt, row=None, col="strip")
        _, _, b8b, sbb = bw(x, F8.E4M3, row=None, col="block")
        casts = None
    kw = {}
    if swiglu:
        kw = dict(epi=K.EPI_SWIGLU, out2=torch.empty(M, N, dtype=torch.bfloat16, device=dev))
    elif dswiglu:
        kw = dict(epi=K.EPI_DSWIGLU, aux=torch.randn(M, 2 * N, generator=g, device=dev).bfloat16(),
                  out2=torch.empty(M, 2 * N, dtype=torch.bfloat16, device=dev))
    gemms = {"tensorwise": lambda: K.fp8_matmul(a8, b8, sa, sb, **kw), "blockwise": lambda: K.fp8_matmul_block(a8b, b8b, sab, sbb, **kw)}
    flops = 2.0 * M * N * Kd
    r = {"proj": name, "pass": pas, "M": M, "N": N, "K": Kd}
    t = alternated(gemms, args.warmup, args.iters, args.repeats)
    for k, ms in t.items():
        r[f"{k}_gemm_ms"], r[f"{k}_gemm_tflops"] = round(ms, 4), round(flops / ms / 1e9, 1)
    if casts is not None:
        t = alternated(casts, args.warmup, args.iters, args.repeats)
        both = alternated({k: (lambda k=k: (casts[k](), gemms[k]())) for k in casts}, args.warmup, args.iters, args.repeats)
        for k in casts:
            r[f"{k}_casts_ms"] = round(t[k], 4)
            r[f"{k}_gemm_cast_ms"], r[f"{k}_gemm_cast_tflops"] = round(both[k], 4), round(flops / both[k] / 1e9, 1)
    return r


def train_arm(args):
    import deepspeed_b200 as ds
    from bench import pick_checkpoint_layers
    from deepspeed_b200.models.llama import LlamaForCausalLM, llama_config
    torch.cuda.set_device(0)
    ds.init_distributed(verbose=False)
    cfg = llama_config(args.model, **ARMS[args.arm])
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

    for i in range(args.train_warmup):
        step(i)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(args.steps):
        loss = step(args.train_warmup + i)
    e.record()
    torch.cuda.synchronize()
    sec = s.elapsed_time(e) / 1e3
    print(json.dumps({"arm": args.arm, "model": args.model, "seq": args.seq, "micro_batch": args.micro_batch,
                      "checkpoint_layers": cfg.checkpoint_layers, "steps": args.steps, "warmup": args.train_warmup,
                      "tokens_per_s": round(args.steps * args.micro_batch * args.seq / sec, 1),
                      "step_ms": round(1e3 * sec / args.steps, 2),
                      "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
                      "loss_after": float(loss.detach()), **gpu_info()}), flush=True)


def train(args):
    rows = []
    for rnd in range(args.rounds):
        for arm in ARMS:
            cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--model", args.model, "--seq", str(args.seq),
                   "--micro-batch", str(args.micro_batch), "--steps", str(args.steps), "--train-warmup", str(args.train_warmup)]
            p = subprocess.run(cmd, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(f"arm {arm} failed:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            row = json.loads([l for l in p.stdout.splitlines() if l.startswith("{")][-1])
            row["round"] = rnd
            rows.append(row)
            print(json.dumps(row), flush=True)
    summary = {}
    for arm in ARMS:
        mine = [r for r in rows if r["arm"] == arm]
        summary[arm] = {"tokens_per_s_median": statistics.median(r["tokens_per_s"] for r in mine),
                        "tokens_per_s_runs": [r["tokens_per_s"] for r in mine], "peak_mem_gib": mine[-1]["peak_mem_gib"],
                        "loss_after": mine[-1]["loss_after"]}
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=["kernels", "train", "all"], default="all")
    ap.add_argument("--models", default="llama3.2-3b,llama3-8b")
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--model", default="llama3.2-3b")
    ap.add_argument("--seq", type=int, default=4096)
    ap.add_argument("--micro-batch", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--train-warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arm", choices=list(ARMS), help="run one training arm in this process (used by --part train)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_blockwise needs a CUDA device")
    if args.arm:
        return train_arm(args)
    out = {**gpu_info(), "tokens": args.tokens}
    if args.part in ("kernels", "all"):
        out["kernels"] = []
        for m in args.models.split(","):
            for name, pas, M, N, Kd in problems(args.tokens, **MODELS[m]):
                r = {"model": m, **bench_one(name, pas, M, N, Kd, args)}
                out["kernels"].append(r)
                print(json.dumps(r), flush=True)
    if args.part in ("train", "all"):
        out["train"] = train(args)
    out["nvidia_smi_after"] = gpu_info()["nvidia_smi"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
