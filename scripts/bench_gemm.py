"""wgmma GEMM vs cuBLAS on the Llama-3-8B forward shapes (CUDA events, L2 flushed between iterations)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepspeed_b200.ops.kernels import gemm_sm100

shapes = [(8192, 6144, 4096, "qkv"), (8192, 4096, 4096, "o"), (8192, 28672, 4096, "gate_up"), (8192, 4096, 14336, "down"),
          (2048, 128256, 4096, "lm_head_chunk")]
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
rows = []
for M, N, K, name in shapes:
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)

    def t(fn, iters=10):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(iters):
            flush.zero_()
            s, e = torch.cuda.Event(True), torch.cuda.Event(True)
            s.record(); fn(); e.record(); torch.cuda.synchronize()
            ts.append(s.elapsed_time(e))
        ts.sort()
        return ts[len(ts) // 2]

    ok = gemm_sm100.self_check()
    t_lib = t(lambda: torch.matmul(a, b.t(), out=out))
    t_own = t(lambda: gemm_sm100.matmul_nt(a, b, out=out)) if ok else float("nan")
    try:
        t_2cta = t(lambda: gemm_sm100.matmul_nt_2cta(a, b, out=out))
        ok2 = bool((out.float() - torch.matmul(a, b.t()).float()).abs().max() < 0.05 * out.float().abs().max() + 0.5)
    except Exception as ex:
        t_2cta, ok2 = float("nan"), False
    fl = 2.0 * M * N * K
    rows.append({"shape": name, "M": M, "N": N, "K": K, "cublas_ms": t_lib, "sm100_ms": t_own,
                 "cublas_tflops": fl / t_lib / 1e9, "sm100_tflops": fl / t_own / 1e9 if ok else None,
                 "sm100_2cta_ms": t_2cta, "sm100_2cta_tflops": fl / t_2cta / 1e9 if ok2 else None, "2cta_correct": ok2})
    print(rows[-1], flush=True)
# backward shapes: dX = dY[M,N] @ W[N,K] (NN) and dW[N,K] = dY[M,N]^T @ X[M,K] (TN)
for M, N, K, name in shapes[:4]:
    dy = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    dx = torch.empty(M, K, device="cuda", dtype=torch.bfloat16)
    dw = torch.empty(N, K, device="cuda", dtype=torch.bfloat16)

    def t(fn, iters=10):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(iters):
            flush.zero_()
            s, e = torch.cuda.Event(True), torch.cuda.Event(True)
            s.record(); fn(); e.record(); torch.cuda.synchronize()
            ts.append(s.elapsed_time(e))
        ts.sort()
        return ts[len(ts) // 2]

    fl = 2.0 * M * N * K
    r = {"shape": name + "_bwd", "M": M, "N": N, "K": K,
         "dx_cublas_tflops": fl / t(lambda: torch.mm(dy, w, out=dx)) / 1e9,
         "dx_2cta_tflops": fl / t(lambda: gemm_sm100.matmul_nn(dy, w, out=dx)) / 1e9,
         "dw_cublas_tflops": fl / t(lambda: torch.mm(dy.t(), x, out=dw)) / 1e9,
         "dw_2cta_tflops": fl / t(lambda: gemm_sm100.matmul_tn(dy, x, out=dw)) / 1e9}
    rows.append(r)
    print(r, flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(rows, open("gpurun_out/gemm_bench.json", "w"), indent=1)
