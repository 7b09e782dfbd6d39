"""Causal sliding-window training attention at Mistral-7B's attention shape (hq 32, hkv 8, d 128, window 4096), one
sequence of S = 4096 ... 32768 tokens.

Measures forward and forward + backward milliseconds of
  * the in-tree wgmma kernel with the window (it skips the tiles outside the band: O(S * W) work),
  * the in-tree kernel, full causal (a cost reference, not the same result),
  * cuDNN SDPA, full causal (a cost reference, not the same result),
  * the masked-SDPA fallback of ``ops.attention`` (an explicit [S, S] band mask; recorded as unavailable when it runs out
    of memory -- at 32 k the boolean mask alone is 1 GiB).
TFLOP/s count only the useful work: the visible (query, key) pairs of the window, 4 * hq * d FLOPs each forward and 3.5x
that forward + backward.  CUDA events after a warm-up; inputs rotate through 4 buffers so L2 does not help.  The card name
and power limit are recorded with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from torch.nn.attention import SDPBackend, sdpa_kernel

from deepspeed_b200.ops.attention import causal_attention
from deepspeed_b200.ops.kernels import attention_sm100 as A

ap = argparse.ArgumentParser()
ap.add_argument("--seq", type=int, nargs="+", default=[4096, 8192, 16384, 32768])
ap.add_argument("--window", type=int, default=4096)
ap.add_argument("--hq", type=int, default=32)
ap.add_argument("--hkv", type=int, default=8)
ap.add_argument("--head-dim", type=int, default=128, choices=(64, 128))
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "sliding_window_attention"),
                help="directory the JSON result is written to")
a = ap.parse_args()

d = a.head_dim
hq, hkv, W = a.hq, a.hkv, a.window


def visible_pairs(S, W):
    """sum over query rows i of min(i + 1, W)"""
    return S * (S + 1) // 2 if W >= S else S * W - W * (W - 1) // 2


def timeit(fn, n=a.iters):
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(n):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def gpu_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,power.max_limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        info["nvidia_smi"] = q.stdout.strip()
    except Exception as ex:  # noqa
        info["nvidia_smi"] = f"unavailable: {type(ex).__name__}"
    return info


def run_shape(S):
    bufs = [torch.randn(S, (hq + 2 * hkv) * d, device="cuda", dtype=torch.bfloat16) for _ in range(4)]
    d_o = torch.randn(S, hq * d, device="cuda", dtype=torch.bfloat16)

    def native(window):

        def fwd(i):
            q, k, v = A.split_packed(bufs[i % 4], hq, hkv, d)
            return A.fwd(q, k, v, 1, S, hq, hkv, causal=True, window=window, head_dim=d)

        def fwd_bwd(i):
            q, k, v = A.split_packed(bufs[i % 4], hq, hkv, d)
            o, lse = A.fwd(q, k, v, 1, S, hq, hkv, causal=True, window=window, head_dim=d)
            A.bwd(d_o, q, k, v, o, lse, 1, S, hq, hkv, causal=True, window=window, head_dim=d)

        return fwd, fwd_bwd

    def heads(x2d, grad):
        x = x2d.view(1, S, hq + 2 * hkv, d)
        return (t.detach().requires_grad_(grad)
                for t in (x[:, :, :hq].transpose(1, 2), x[:, :, hq:hq + hkv].transpose(1, 2),
                          x[:, :, hq + hkv:].transpose(1, 2)))

    def cudnn_fwd(i, grad=False):
        q, k, v = heads(bufs[i % 4], grad)
        with sdpa_kernel([SDPBackend.CUDNN_ATTENTION]):
            return q, k, v, F.scaled_dot_product_attention(q, k, v, is_causal=True, enable_gqa=True)

    def cudnn_fwd_bwd(i):
        q, k, v, o = cudnn_fwd(i, grad=True)
        torch.autograd.grad(o, (q, k, v), d_o.view(1, S, hq, d).transpose(1, 2))

    def masked_fwd(i):
        with torch.no_grad():
            return causal_attention(bufs[i % 4], 1, S, hq, hkv, d, backend="cudnn", sliding_window=W)

    def masked_fwd_bwd(i):
        x = bufs[i % 4].detach().requires_grad_(True)
        causal_attention(x, 1, S, hq, hkv, d, backend="cudnn", sliding_window=W).backward(d_o)

    useful = 4.0 * hq * d * visible_pairs(S, W)
    res = {"S": S, "visible_pairs": visible_pairs(S, W), "useful_fwd_tflop": useful / 1e12}
    nw_fwd, nw_both = native(W)
    o_native = nw_fwd(0)[0]
    try:
        o_masked = masked_fwd(0)
        res["max_abs_diff_native_vs_masked_sdpa"] = (o_native.float() - o_masked.float()).abs().max().item()
        del o_masked
    except torch.cuda.OutOfMemoryError:
        res["max_abs_diff_native_vs_masked_sdpa"] = None
    del o_native
    torch.cuda.empty_cache()
    nc_fwd, nc_both = native(None)
    for name, f_fn, b_fn in (("native_window", nw_fwd, nw_both), ("native_full_causal", nc_fwd, nc_both),
                             ("cudnn_full_causal", cudnn_fwd, cudnn_fwd_bwd),
                             ("masked_sdpa_window", masked_fwd, masked_fwd_bwd)):
        r = {}
        for key, fn, mult in (("fwd", f_fn, 1.0), ("fwd_bwd", b_fn, 3.5)):
            try:
                t = timeit(fn)
                r[f"{key}_ms"] = t
                r[f"{key}_useful_tflops"] = mult * useful / t / 1e9
            except torch.cuda.OutOfMemoryError:
                r[f"{key}_ms"] = None
                r[f"{key}_unavailable"] = "out of memory"
            torch.cuda.empty_cache()
        res[name] = r
    return res


res = {"shape": dict(B=1, hq=hq, hkv=hkv, d=d, window=W, causal=True, seq=a.seq), **gpu_info(), "runs": []}
for S in a.seq:
    r = run_shape(S)
    res["runs"].append(r)
    print(json.dumps(r), flush=True)
times = {r["S"]: r["native_window"]["fwd_bwd_ms"] for r in res["runs"]}
if 16384 in times and 32768 in times:
    res["native_window_fwd_bwd_ratio_32k_over_16k"] = times[32768] / times[16384]
    res["visible_pair_ratio_32k_over_16k"] = visible_pairs(32768, W) / visible_pairs(16384, W)
print(json.dumps({k: v for k, v in res.items() if k != "runs"}, indent=1))
os.makedirs(a.out, exist_ok=True)
path = os.path.join(a.out, "bench_sliding_window_attention.json")
with open(path, "w") as f:
    json.dump(res, f, indent=1)
print(f"wrote {path}")
