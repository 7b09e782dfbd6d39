"""FP8 vs bf16 GEMMs at the Llama training step's projection shapes (8192 tokens): Llama-3.2-3B (qkv 5120 x 3072, o 3072 x
3072, gate|up + SwiGLU 2 x 8192 x 3072, down 3072 x 8192) and Llama-3-8B.  For each projection, forward, dgrad and wgrad
are timed on
  * own_bf16:    the in-tree bf16 wgmma GEMM with the step's layouts and epilogues (SwiGLU on the gate|up forward,
                 dSwiGLU on the down dgrad);
  * cublas_bf16: torch.mm (plain product, no epilogue);
  * own_fp8:     the in-tree FP8 GEMM on operands already cast (same epilogues as own_bf16);
  * own_fp8_cast: own_fp8 plus the casts the node makes for that product: forward casts x (row-major + transposed) and
                 W; dgrad casts dY (row-major + transposed) and W^T; wgrad reuses the transposed dY and x, so it adds none;
  * scaled_mm / scaled_mm_fast: torch._scaled_mm (cuBLASLt) with promoted / fast accumulation, plain product.
TFLOP/s count 2 M N K per product (the gate|up forward's N is 2 I; its row reports N = I, the SwiGLU output width).  CUDA events after a warm-up, mean of --iters launches;
the card name and power limit are recorded in the same run.  Prints one JSON object."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepspeed_b200.ops import fp8 as F8
from deepspeed_b200.ops.kernels import fp8_ops
from deepspeed_b200.ops.kernels import gemm_sm100 as K

MODELS = {"llama3.2-3b": dict(H=3072, I=8192, qkv=5120), "llama3-8b": dict(H=4096, I=14336, qkv=6144)}


def gpu_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.max_limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except Exception as ex:  # noqa
        info["nvidia_smi"] = f"unavailable: {type(ex).__name__}"
    return info


def timed(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def cast(x, fmt, row=True, col=False):
    return fp8_ops.fp8_cast(x, fp8_ops.fp8_amax(x), fmt, rowwise=row, colwise=col)


def problems(T, H, I, qkv):
    """(projection, pass, M, N, K, epilogue) of one decoder layer's products; N is the output width."""
    out = []
    for name, n, k in (("qkv", qkv, H), ("o", H, H), ("gate_up", 2 * I, H), ("down", H, I)):
        out.append((name, "fwd", T, n, k))
        out.append((name, "dgrad", T, k, n))
        out.append((name, "wgrad", n, k, T))
    return out


def bench_one(name, pas, M, N, Kd, T, warmup, iters):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    r = {"proj": name, "pass": pas, "M": M, "N": N, "K": Kd}
    flops = 2.0 * M * N * Kd * (2 if name == "gate_up" and pas == "fwd" else 1)
    swiglu = name == "gate_up" and pas == "fwd"
    dswiglu = name == "down" and pas == "dgrad"
    afmt = F8.E4M3 if pas == "fwd" else F8.E5M2
    # logical operands in the step's own layouts (bf16)
    if pas == "fwd":  # x [T, K], W [N, K]
        a = torch.randn(M, Kd, generator=g, device=dev).bfloat16()
        b = (torch.randn(2 * N if swiglu else N, Kd, generator=g, device=dev) * 0.02).bfloat16()
        own = lambda: K.matmul_2cta(a, b, False, False, epi=K.EPI_SWIGLU if swiglu else K.EPI_STORE,
                                    out2=gu_out if swiglu else None, inter=N if swiglu else 0)
        lib = lambda: torch.mm(a, b.t())
    elif pas == "dgrad":  # dY [T, N_out], W [N_out, K_out]: dX = dY W, here M = T, N = K_out, K = N_out
        a = torch.randn(M, Kd, generator=g, device=dev).bfloat16()
        w = (torch.randn(Kd, N, generator=g, device=dev) * 0.02).bfloat16()
        own = lambda: K.matmul_2cta(a, w, False, True, epi=K.EPI_DSWIGLU if dswiglu else K.EPI_STORE,
                                    aux=gu_aux if dswiglu else None, out=dgu_out[:, :N] if dswiglu else None,
                                    out2=dgu_out if dswiglu else None, inter=N if dswiglu else 0)
        lib = lambda: torch.mm(a, w)
    else:  # dW [N_out, K_in] = dY^T X: M = N_out, N = K_in, K = T
        dy = torch.randn(Kd, M, generator=g, device=dev).bfloat16()
        x = torch.randn(Kd, N, generator=g, device=dev).bfloat16()
        own = lambda: K.matmul_2cta(dy, x, True, True)
        lib = lambda: torch.mm(dy.t(), x)
    gu_out = torch.empty(M, 2 * N, dtype=torch.bfloat16, device=dev) if swiglu else None
    gu_aux = torch.randn(M, 2 * N, generator=g, device=dev).bfloat16() if dswiglu else None
    dgu_out = torch.empty(M, 2 * N, dtype=torch.bfloat16, device=dev) if dswiglu else None
    r["own_bf16_ms"] = timed(own, warmup, iters)
    r["cublas_bf16_ms"] = timed(lib, warmup, iters)
    # fp8 operands, K-major: A [M, K], B [N, K]
    if pas == "fwd":
        a_src, b_src = a, b
        a8, _, sa = cast(a_src, afmt)
        b8, _, sb = cast(b_src, F8.E4M3)
        casts = lambda: (cast(a_src, afmt, True, True), cast(b_src, F8.E4M3))
    elif pas == "dgrad":
        a8, _, sa = cast(a, afmt)
        _, b8, sb = cast(w, F8.E4M3, False, True)  # W^T [K_out, N_out]
        casts = lambda: (cast(a, afmt, True, True), cast(w, F8.E4M3, False, True))
    else:
        _, a8, sa = cast(dy, F8.E5M2, False, True)  # dY^T [N_out, T]
        _, b8, sb = cast(x, F8.E4M3, False, True)  # X^T [K_in, T]
        casts = lambda: None
    if swiglu:
        f8 = lambda: K.fp8_matmul(a8, b8, sa, sb, epi=K.EPI_SWIGLU, out2=gu_out)
    elif dswiglu:
        f8 = lambda: K.fp8_matmul(a8, b8, sa, sb, epi=K.EPI_DSWIGLU, aux=gu_aux, out2=dgu_out)
    else:
        f8 = lambda: K.fp8_matmul(a8, b8, sa, sb)
    r["own_fp8_ms"] = timed(f8, warmup, iters)
    r["own_fp8_cast_ms"] = timed(lambda: (casts(), f8()), warmup, iters)
    r["casts_ms"] = timed(casts, warmup, iters) if pas != "wgrad" else 0.0
    for key, fast in (("scaled_mm_ms", False), ("scaled_mm_fast_ms", True)):
        try:
            r[key] = timed(lambda: torch._scaled_mm(a8, b8.t(), scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16,
                                                    use_fast_accum=fast), warmup, iters)
        except RuntimeError as ex:
            r[key] = f"unavailable: {str(ex)[:120]}"
    for k in list(r):
        if k.endswith("_ms") and isinstance(r[k], float) and r[k] > 0 and k != "casts_ms":
            r[k.replace("_ms", "_tflops")] = round(flops / (r[k] * 1e-3) / 1e12, 1)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama3.2-3b,llama3-8b")
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_gemm needs a CUDA device")
    out = {**gpu_info(), "tokens": args.tokens, "rows": []}
    for m in args.models.split(","):
        for name, pas, M, N, Kd in problems(args.tokens, **MODELS[m]):
            r = bench_one(name, pas, M, N // 2 if (name == "gate_up" and pas == "fwd") else N, Kd, args.tokens,
                          args.warmup, args.iters)
            r["model"] = m
            out["rows"].append(r)
            print(json.dumps(r), flush=True)
    out["nvidia_smi_after"] = gpu_info()["nvidia_smi"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
