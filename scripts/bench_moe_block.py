"""Mixtral-8x7B MoE block (H=4096, I=14336, 8 experts, top-2) on the ragged engine: grouped wgmma GEMM path vs the
per-expert / dense-all-experts paths.  Device-timed, L2 flushed between iterations."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepspeed_b200.inference.v2.model_implementations.arch import ArchSpec  # noqa: E402
from deepspeed_b200.inference.v2.model_implementations.ragged_transformer import LayerWeights, RaggedTransformer  # noqa: E402

H, I, E, K = 4096, 14336, 8, 2
spec = ArchSpec("mixtral", 32000, H, 1, 32, 8, 128, I, num_experts=E, top_k=K)
model = RaggedTransformer(spec, dtype=torch.bfloat16, device="cuda")
lw = LayerWeights()
torch.manual_seed(0)
lw.gate_w = (torch.randn(E, H, device="cuda") * 0.02).bfloat16()
lw.experts_up = (torch.randn(E, 2 * I, H, device="cuda") * 0.02).bfloat16()
lw.experts_down = (torch.randn(E, H, I, device="cuda") * 0.02).bfloat16()
flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")


def timed(fn, n=7):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        s, e = torch.cuda.Event(True), torch.cuda.Event(True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return sorted(ts)[n // 2]


rows = []
for T in (1, 8, 64, 512, 4096):
    x = (torch.randn(T, H, device="cuda") * 0.5).bfloat16()
    os.environ["DSB200_MOE_GROUPED"] = "1"
    yg = model._moe(lw, x)
    tg = timed(lambda: model._moe(lw, x))
    os.environ["DSB200_MOE_GROUPED"] = "0"
    yr = model._moe(lw, x)
    tr = timed(lambda: model._moe(lw, x))
    err = (yg.float() - yr.float()).abs().max().item() / max(1e-6, yr.float().abs().max().item())
    flops = 2 * T * K * 3 * H * I
    touched = min(E, T * K) * 3 * H * I * 2
    rows.append({"tokens": T, "grouped_ms": round(tg, 3), "baseline_ms": round(tr, 3), "speedup": round(tr / tg, 2),
                 "grouped_TFLOPs": round(flops / tg / 1e9, 1), "grouped_weight_GBps_lower_bound": round(touched / tg / 1e6),
                 "rel_err_vs_baseline": round(err, 4)})
    print(rows[-1], flush=True)
if len(sys.argv) > 1:
    json.dump({"config": "Mixtral-8x7B MoE block, bf16, top-2 of 8", "rows": rows}, open(sys.argv[1], "w"), indent=1)
