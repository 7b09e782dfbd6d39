"""Weight-only-quantised linear at prefill / batched-decode sizes: the fused dequantise-in-smem wgmma kernel
(csrc/cuda/wq_tc_gemm.cu) vs dequantise-once + bf16 GEMM, per mode and row count.  CUDA events, rotating weights (> L2),
median of 20.  Writes gpurun_out/wq_tc_bench.json; the crossover feeds WQ_TC_MAX_ROWS in inference/quantization/layers.py."""
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from _clocks import Clocks

from deepspeed_b200.inference.quantization import layers as QL


def timeit(fn, n_rot, warm=4, iters=20):
    for i in range(warm):
        fn(i % n_rot)
    torch.cuda.synchronize()
    ts = []
    for i in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(i % n_rot)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    out = {"gpu": torch.cuda.get_device_name(0), "rows": []}
    clk = Clocks()
    N, K = 14336, 4096
    n_rot = 6  # 6 x 58 MB (int8) > 126 MB L2
    for mode in ("int8", "int4", "fp8", "fp6"):
        ws = [torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * 0.02 for _ in range(n_rot)]
        qws = [QL.quantize_weight(w, mode, 128) for w in ws]
        del ws
        for M in (64, 128, 256, 512, 1024):
            x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
            fused = lambda i: QL.wq_tc_linear(x, qws[i], max_rows=1 << 20)
            split = lambda i: torch.nn.functional.linear(x, qws[i].dequantize())
            y1, y2 = fused(0), split(0)
            err = (y1.float() - y2.float()).abs().max().item() / (y2.float().abs().max().item() + 1e-6)
            rec = {"mode": mode, "M": M, "N": N, "K": K, "fused_ms": timeit(fused, n_rot), "dequant_gemm_ms": timeit(split, n_rot),
                   "rel_err": err}
            rec["speedup"] = rec["dequant_gemm_ms"] / rec["fused_ms"]
            wbytes = qws[0].q.numel() * qws[0].q.element_size()
            rec["fused_weight_GBps"] = wbytes / rec["fused_ms"] / 1e6
            out["rows"].append(rec)
            print(json.dumps(rec))
    out["clocks"] = clk.stop()
    os.makedirs("gpurun_out", exist_ok=True)
    with open("gpurun_out/wq_tc_bench.json", "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
