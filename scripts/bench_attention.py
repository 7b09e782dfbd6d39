"""Training-attention micro-benchmark at the Llama-3-8B shape: the in-tree wgmma kernel vs cuDNN / flash SDPA.
CUDA events, 5 warm-up + 20 timed iterations, inputs (100+ MB per call) rotate through 4 buffers so L2 does not help."""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from torch.nn.attention import SDPBackend, sdpa_kernel

from deepspeed_b200.ops.kernels import attention_sm100 as A

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=2)
ap.add_argument("--S", type=int, default=4096)
ap.add_argument("--hq", type=int, default=32)
ap.add_argument("--hkv", type=int, default=8)
ap.add_argument("--head-dim", type=int, default=128, choices=(64, 128))
ap.add_argument("--out", default="gpurun_out/attention_bench.json")
a = ap.parse_args()
B, S, hq, hkv, d = a.B, a.S, a.hq, a.hkv, a.head_dim
bufs = [torch.randn(B * S, (hq + 2 * hkv) * d, device="cuda", dtype=torch.bfloat16) for _ in range(4)]
flops_fwd = 4.0 * B * hq * S * S * d * 0.5  # causal


def timeit(fn, n=20):
    for i in range(5):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(n):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def own_fwd(i):
    q, k, v = A.split_packed(bufs[i % 4], hq, hkv, d)
    return A.fwd(q, k, v, B, S, hq, hkv, causal=True, head_dim=d)


def lib_fwd(i, backend=SDPBackend.CUDNN_ATTENTION):
    x = bufs[i % 4].view(B, S, hq + 2 * hkv, d)
    with sdpa_kernel([backend]):
        return F.scaled_dot_product_attention(x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2),
                                              x[:, :, hq + hkv:].transpose(1, 2), is_causal=True, enable_gqa=True)


res = {"shape": dict(B=B, S=S, hq=hq, hkv=hkv, d=d, causal=True), "fwd_tflop": flops_fwd / 1e12}
o, _ = own_fwd(0)
ref = lib_fwd(0).transpose(1, 2).reshape(B * S, hq * d)
res["max_abs_diff_vs_cudnn"] = (o.float() - ref.float()).abs().max().item()
t_own = timeit(own_fwd)
res["own_fwd_ms"], res["own_fwd_tflops"] = t_own, flops_fwd / t_own / 1e9
for name, be in (("cudnn", SDPBackend.CUDNN_ATTENTION), ("flash", SDPBackend.FLASH_ATTENTION)):
    try:
        t = timeit(lambda i: lib_fwd(i, be))
        res[f"{name}_fwd_ms"], res[f"{name}_fwd_tflops"] = t, flops_fwd / t / 1e9
    except Exception as ex:  # noqa
        res[f"{name}_fwd_ms"] = f"unavailable: {type(ex).__name__}"
if hasattr(A, "bwd"):
    try:
        x = bufs[0]
        q, k, v = A.split_packed(x, hq, hkv, d)
        o, lse = A.fwd(q, k, v, B, S, hq, hkv, causal=True, head_dim=d)
        do = torch.randn_like(o)
        t = timeit(lambda i: A.bwd(do, q, k, v, o, lse, B, S, hq, hkv, causal=True, head_dim=d))
        res["own_bwd_ms"], res["own_bwd_tflops"] = t, 2.5 * flops_fwd / t / 1e9
    except Exception as ex:  # noqa
        res["own_bwd_ms"] = f"failed: {type(ex).__name__}: {ex}"
xq = bufs[0].view(B, S, hq + 2 * hkv, d)
qq, kk, vv = (t.transpose(1, 2).detach().requires_grad_(True) for t in (xq[:, :, :hq], xq[:, :, hq:hq + hkv], xq[:, :, hq + hkv:]))
with sdpa_kernel([SDPBackend.CUDNN_ATTENTION]):
    oo = F.scaled_dot_product_attention(qq, kk, vv, is_causal=True, enable_gqa=True)
go = torch.randn_like(oo)
t = timeit(lambda i: torch.autograd.grad(oo, (qq, kk, vv), go, retain_graph=True))
res["cudnn_bwd_ms"], res["cudnn_bwd_tflops"] = t, 2.5 * flops_fwd / t / 1e9
print(json.dumps(res, indent=1))
os.makedirs(os.path.dirname(a.out), exist_ok=True)
json.dump(res, open(a.out, "w"), indent=1)
