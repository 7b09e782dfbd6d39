"""Packed-sequence (document-masked) training attention at the benchmark model's attention shape (hq 24, hkv 8, d 128,
8192 tokens = one micro-batch of bench.py: 2 rows of 4096), documents drawn from a seeded length mix.

Measures forward and forward + backward milliseconds of
  * the in-tree varlen wgmma kernel (one launch per pass over all documents),
  * the per-document cuDNN SDPA loop (the fallback path of ``ops.attention``),
  * dense causal attention over the same 2 x 4096 rows ignoring document boundaries (a reference cost).
TFLOP/s count only the useful work: sum over documents of the causal len^2 attention FLOPs.  CUDA events after a warm-up;
inputs rotate through 4 buffers so L2 does not help.  The card name and power limit are recorded with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.nn.functional as F
from torch.nn.attention import SDPBackend, sdpa_kernel

from deepspeed_b200.ops.kernels import attention_sm100 as A

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=2)
ap.add_argument("--row-len", type=int, default=4096)
ap.add_argument("--hq", type=int, default=24)
ap.add_argument("--hkv", type=int, default=8)
ap.add_argument("--head-dim", type=int, default=128, choices=(64, 128))
ap.add_argument("--min-len", type=int, default=16)
ap.add_argument("--max-len", type=int, default=4096)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "packed_attention"),
                help="directory the JSON result is written to")
a = ap.parse_args()

d = a.head_dim
hq, hkv = a.hq, a.hkv
rng = np.random.default_rng(a.seed)
lens = []
for _ in range(a.rows):
    left = a.row_len
    while left:
        n = min(int(rng.integers(a.min_len, a.max_len + 1)), left)
        lens.append(n)
        left -= n
T = a.rows * a.row_len
cu_host = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
cu = torch.from_numpy(cu_host).cuda()
spans = list(zip(cu_host[:-1].tolist(), cu_host[1:].tolist()))
max_len = max(lens)
useful_fwd = sum(4.0 * hq * n * n * d * 0.5 for n in lens)  # causal: half of QK^T and PV
dense_fwd = 4.0 * a.rows * hq * a.row_len**2 * d * 0.5

bufs = [torch.randn(T, (hq + 2 * hkv) * d, device="cuda", dtype=torch.bfloat16) for _ in range(4)]
d_o = torch.randn(T, hq * d, device="cuda", dtype=torch.bfloat16)


def timeit(fn, n=a.iters):
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


def native_fwd(i):
    q, k, v = A.split_packed(bufs[i % 4], hq, hkv, d)
    return A.fwd_varlen(q, k, v, cu, max_len, hq, hkv, causal=True, head_dim=d)


def native_fwd_bwd(i):
    q, k, v = A.split_packed(bufs[i % 4], hq, hkv, d)
    o, lse = A.fwd_varlen(q, k, v, cu, max_len, hq, hkv, causal=True, head_dim=d)
    A.bwd_varlen(d_o, q, k, v, o, lse, cu, max_len, hq, hkv, causal=True, head_dim=d)


def _heads(x2d, rows, S):
    x = x2d.view(rows, S, hq + 2 * hkv, d)
    return (x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2), x[:, :, hq + hkv:].transpose(1, 2))


def loop_fwd(i, grad=False):
    x = bufs[i % 4]
    outs = []
    with sdpa_kernel([SDPBackend.CUDNN_ATTENTION]):
        for s, e in spans:
            q, k, v = (t.detach().requires_grad_(grad) for t in _heads(x[s:e], 1, e - s))
            o = F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True)
            outs.append((q, k, v, o, s, e))
    return outs


def loop_fwd_bwd(i):
    for q, k, v, o, s, e in loop_fwd(i, grad=True):
        torch.autograd.grad(o, (q, k, v), d_o[s:e].view(1, e - s, hq, d).transpose(1, 2))


def dense_fwd_(i, grad=False):
    q, k, v = (t.detach().requires_grad_(grad) for t in _heads(bufs[i % 4], a.rows, a.row_len))
    with sdpa_kernel([SDPBackend.CUDNN_ATTENTION]):
        return q, k, v, F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True)


def dense_fwd_bwd(i):
    q, k, v, o = dense_fwd_(i, grad=True)
    torch.autograd.grad(o, (q, k, v), d_o.view(a.rows, a.row_len, hq, d).transpose(1, 2))


def gpu_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.max_limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except Exception as ex:  # noqa
        info["nvidia_smi"] = f"unavailable: {type(ex).__name__}"
    return info


res = {"shape": dict(T=T, rows=a.rows, row_len=a.row_len, hq=hq, hkv=hkv, d=d, causal=True, n_docs=len(lens),
                     max_len=max_len, seed=a.seed, len_range=[a.min_len, a.max_len]),
       "doc_lengths": lens, "useful_fwd_tflop": useful_fwd / 1e12, "dense_fwd_tflop": dense_fwd / 1e12, **gpu_info()}
# correctness against the per-document loop before timing
o_native, _ = native_fwd(0)
o_loop = torch.cat([o.transpose(1, 2).reshape(e - s, hq * d) for _, _, _, o, s, e in loop_fwd(0)])
res["max_abs_diff_native_vs_loop"] = (o_native.float() - o_loop.float()).abs().max().item()
for name, fwd_fn, both_fn in (("native_varlen", native_fwd, native_fwd_bwd), ("cudnn_per_doc_loop", loop_fwd, loop_fwd_bwd),
                              ("cudnn_dense_causal", dense_fwd_, dense_fwd_bwd)):
    tf = timeit(fwd_fn)
    tb = timeit(both_fn)
    res[name] = {"fwd_ms": tf, "fwd_bwd_ms": tb, "fwd_useful_tflops": useful_fwd / tf / 1e9,
                 "fwd_bwd_useful_tflops": 3.5 * useful_fwd / tb / 1e9}
res["speedup_native_vs_loop"] = {"fwd": res["cudnn_per_doc_loop"]["fwd_ms"] / res["native_varlen"]["fwd_ms"],
                                 "fwd_bwd": res["cudnn_per_doc_loop"]["fwd_bwd_ms"] / res["native_varlen"]["fwd_bwd_ms"]}
print(json.dumps(res, indent=1))
os.makedirs(a.out, exist_ok=True)
path = os.path.join(a.out, "bench_packed_attention.json")
with open(path, "w") as f:
    json.dump(res, f, indent=1)
print(f"wrote {path}")
