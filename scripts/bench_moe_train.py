"""Dropless MoE training cost at one Mixtral-8x7B MoE layer (H 4096, I 14336, 8 experts, top-2, bf16 weights) and 8192
tokens.

Routing is fixed per run from a seed, either uniform (two distinct experts per token) or skewed (expert 0 is one of each
token's two choices with probability 0.8, so it takes ~40 % of the assignments).  Every path starts from the same expert
ids and combine weights and covers dispatch, experts and combine; forward and forward + backward milliseconds of
  * ragged: 64-row aligned segments built on the device, one wgmma launch per projection and direction
    (``ops.linear._RaggedSwiGLUFn``), no host synchronisation;
  * padded_to_max: every expert padded to the largest expert's count and run through ``grouped_swiglu_mlp`` (the dropless
    path before the ragged kernels existed: bincount, ``.tolist()``, a Python fill loop and ``torch.cat``);
  * capacity_1.25: the capacity-factor path (``[E, C, H]`` with C = 1.25 x the mean load).  It drops tokens under skew, so
    it computes a different result: a cost reference only;
  * torch_grouped_mm: ``torch._grouped_mm`` on the ragged layout, where this torch build and its shape constraints allow;
  * fp8_tensorwise / fp8_blockwise: the ragged path with FP8 products (``ops.linear.fp8_ragged_swiglu_mlp``) on 128-row
    segments, the times including every cast the node makes.
Useful TFLOP/s count the true token-expert assignments only (6 H I FLOPs each forward, 3x that forward + backward).  CUDA
events after a warm-up.  The card name and power limit are recorded with the numbers."""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from deepspeed_b200.ops import gemm
from deepspeed_b200.ops.kernels import moe_ops
from deepspeed_b200.ops.linear import _RaggedSwiGLUFn, fp8_ragged_swiglu_mlp, fp8_ragged_swiglu_native, grouped_swiglu_mlp

ap = argparse.ArgumentParser()
ap.add_argument("--tokens", type=int, default=8192)
ap.add_argument("--hidden", type=int, default=4096)
ap.add_argument("--inter", type=int, default=14336)
ap.add_argument("--experts", type=int, default=8)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--iters", type=int, default=10)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "moe_train"), help="directory the JSON result is written to")
a = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_moe_train.py measures on a CUDA device; none is present")

T, H, I, E, k = a.tokens, a.hidden, a.inter, a.experts, 2
dev = "cuda"
g = torch.Generator(device=dev).manual_seed(a.seed)
w13 = (torch.randn(E, 2 * I, H, device=dev, generator=g) * H**-0.5).bfloat16().requires_grad_(True)
w2 = (torch.randn(E, H, I, device=dev, generator=g) * I**-0.5).bfloat16().requires_grad_(True)
x0 = (torch.randn(T, H, device=dev, generator=g) * 0.5).bfloat16()
dy = torch.randn(T, H, device=dev, generator=g).bfloat16()


def routing(kind):
    """-> (ids [T, 2] int32, weights [T, 2] fp32)."""
    gc = torch.Generator(device="cpu").manual_seed(a.seed + 1)
    if kind == "uniform":
        ids = torch.stack([torch.randperm(E, generator=gc)[:2] for _ in range(T)])
    else:
        ids = torch.empty(T, 2, dtype=torch.long)
        hot = torch.rand(T, generator=gc) < 0.8
        for t in range(T):
            rest = torch.randperm(E - 1, generator=gc) + 1
            ids[t] = torch.stack([torch.tensor(0), rest[0]]) if hot[t] else rest[:2]
    w = torch.rand(T, 2, generator=gc) + 0.1
    return ids.to(torch.int32).to(dev), (w / w.sum(1, keepdim=True)).to(dev)


def _counts(ids):
    return torch.zeros(E, dtype=torch.int32, device=dev).scatter_add_(0, ids.reshape(-1).long(),
                                                                       torch.ones(ids.numel(), dtype=torch.int32, device=dev))


def ragged(x, ids, w):
    pos, counts, _ = moe_ops.route(ids, E, counts=_counts(ids))
    seg = (counts + 63) // 64 * 64
    off = torch.cat([seg.new_zeros(1), torch.cumsum(seg, 0, dtype=torch.int32)])
    rows, slots = moe_ops.scatter(x, ids, pos, off, k, 0, T * k + E * 63)
    eo = _RaggedSwiGLUFn.apply(rows, off, w13, w2)
    return moe_ops.gather(eo, w, slots, T, k)


def fp8_ragged(recipe):
    def run(x, ids, w):
        pos, counts, _ = moe_ops.route(ids, E, counts=_counts(ids))
        seg = (counts + 127) // 128 * 128
        off = torch.cat([seg.new_zeros(1), torch.cumsum(seg, 0, dtype=torch.int32)])
        rows, slots = moe_ops.scatter(x, ids, pos, off, k, 0, -(-(T * k + E * 127) // 128) * 128)
        assert fp8_ragged_swiglu_native(rows, off, w13, w2), "the FP8 arm must run the wgmma kernels"
        eo = fp8_ragged_swiglu_mlp(rows, off, w13, w2, recipe=recipe)
        return moe_ops.gather(eo, w, slots, T, k)

    return run


def padded_to_max(x, ids, w):
    pos, counts, off = moe_ops.route(ids, E)  # torch.bincount
    rows, slots = moe_ops.scatter(x, ids, pos, off, k, 0, T * k)
    cl = counts.tolist()
    mx = max(cl)
    padded = rows.new_zeros(E, mx, H)
    for e, c in enumerate(rows.split(cl, dim=0)):
        padded[e, :c.shape[0]] = c
    po = grouped_swiglu_mlp(padded, w13, w2)
    eo = torch.cat([po[e, :n] for e, n in enumerate(cl)], dim=0)
    return moe_ops.gather(eo, w, slots, T, k)


C = int(math.ceil(T * k / E * 1.25))


def capacity(x, ids, w):
    pos, _, off = moe_ops.route(ids, E, counts=_counts(ids))
    rows, slots = moe_ops.scatter(x, ids, pos, off, k, C, E * C)
    eo = grouped_swiglu_mlp(rows.view(E, C, H), w13, w2)
    return moe_ops.gather(eo.reshape(E * C, H), w, slots, T, k)


def grouped_mm(x, ids, w):
    pos, counts, _ = moe_ops.route(ids, E, counts=_counts(ids))
    seg = (counts + 63) // 64 * 64
    off = torch.cat([seg.new_zeros(1), torch.cumsum(seg, 0, dtype=torch.int32)])
    rows, slots = moe_ops.scatter(x, ids, pos, off, k, 0, T * k + E * 63)
    ends = off[1:]
    gu = torch._grouped_mm(rows, w13.transpose(-2, -1), offs=ends)
    act = F.silu(gu[:, :I]) * gu[:, I:]
    eo = torch._grouped_mm(act, w2.transpose(-2, -1), offs=ends)
    return moe_ops.gather(eo, w, slots, T, k)


def timeit(fn, n):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
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


gemm.set_backend("own")  # the padded and capacity paths on the in-tree kernels, like the ragged one
useful_fwd = 6.0 * H * I * T * k
res = {"shape": dict(T=T, H=H, I=I, E=E, k=k, capacity=C, seed=a.seed), "gemm_backend": gemm.get_backend(),
       "useful_fwd_tflop": useful_fwd / 1e12, **gpu_info()}
paths = {"ragged": ragged, "padded_to_max": padded_to_max, "capacity_1.25": capacity, "torch_grouped_mm": grouped_mm,
         "fp8_tensorwise": fp8_ragged("tensorwise"), "fp8_blockwise": fp8_ragged("blockwise")}
for kind in ("uniform", "skewed"):
    ids, w = routing(kind)
    counts = torch.bincount(ids.reshape(-1).long(), minlength=E).tolist()
    r = {"counts": counts, "max_share": max(counts) / (T * k)}
    ref = None
    for name, fn in paths.items():
        try:
            x = x0.clone().requires_grad_(True)
            y = fn(x, ids, w)
            if name == "ragged":
                ref = y.float()
            elif name.startswith("fp8"):  # a different rounding of the same product: its size relative to the bf16 one
                r.setdefault("rel_l2_diff_vs_ragged", {})[name] = ((y.float() - ref).norm() / ref.norm()).item()
            elif name != "capacity_1.25":
                r.setdefault("max_abs_diff_vs_ragged", {})[name] = (y.float() - ref).abs().max().item()
            del y

            def fwd():
                with torch.no_grad():
                    fn(x0, ids, w)

            def fwd_bwd():
                xg = x0.detach().requires_grad_(True)
                fn(xg, ids, w).backward(dy)
                w13.grad = w2.grad = None

            tf, tb = timeit(fwd, a.iters), timeit(fwd_bwd, a.iters)
            r[name] = {"fwd_ms": tf, "fwd_bwd_ms": tb, "fwd_useful_tflops": useful_fwd / tf / 1e9,
                       "fwd_bwd_useful_tflops": 3 * useful_fwd / tb / 1e9}
        except Exception as ex:  # noqa: a path this torch build or shape cannot run is reported, not fatal
            r[name] = {"error": f"{type(ex).__name__}: {str(ex)[:300]}"}
        w13.grad = w2.grad = None
        torch.cuda.empty_cache()
    if "fwd_ms" in r.get("padded_to_max", {}) and "fwd_ms" in r["ragged"]:
        r["speedup_ragged_vs_padded"] = {p: r["padded_to_max"][p] / r["ragged"][p] for p in ("fwd_ms", "fwd_bwd_ms")}
    for name in ("fp8_tensorwise", "fp8_blockwise"):
        if "fwd_ms" in r.get(name, {}) and "fwd_ms" in r["ragged"]:
            r[f"speedup_{name}_vs_ragged"] = {p: r["ragged"][p] / r[name][p] for p in ("fwd_ms", "fwd_bwd_ms")}
    res[kind] = r
print(json.dumps(res, indent=1))
os.makedirs(a.out, exist_ok=True)
path = os.path.join(a.out, "bench_moe_train.json")
with open(path, "w") as f:
    json.dump(res, f, indent=1)
print(f"wrote {path}")
