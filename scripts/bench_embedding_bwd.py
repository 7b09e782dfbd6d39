"""Embedding backward into a bf16 ZeRO gradient view, on one GPU.

Native: ``transformer_ops.embedding_bwd_`` (the device sort of the ids plus ``transformer.cu:embedding_bwd_kernel`` /
``embedding_bwd_tail_kernel``), which adds into the view's touched rows only.  Torch: ``embedding_dense_backward`` into a
fresh dense ``[V, H]`` tensor plus the add of that tensor into the view -- what ``nn.Embedding`` and the post-accumulate
hook do for an untied embedding.  T = 8192 tokens at the ``llama3.2-1b`` (V 128256, H 2048) and ``qwen3-1.7b``
(V 151936, H 2048) shapes, bf16 gradient, with uniform, Zipf-like (rank^-1.1) and all-equal ids.  CUDA events over many
launches after warm-up; one JSON line per case with the card name and power limit.  The native pass moves ``T x H``
gradient rows and as many view rows; the torch pass writes, scatters into and re-reads the whole ``[V, H]`` tensor.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"llama3.2-1b": (128256, 2048), "qwen3-1.7b": (151936, 2048)}


def _smi():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                               "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa
        return f"unavailable: {type(ex).__name__}"


def _time(torch, fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def _ids(torch, kind, T, V, g):
    if kind == "uniform":
        return torch.randint(0, V, (T, ), generator=g, device="cuda")
    if kind == "zipf":
        w = torch.arange(1, V + 1, dtype=torch.float64, device="cuda").pow(-1.1)
        return torch.multinomial(w / w.sum(), T, replacement=True, generator=g)
    return torch.full((T, ), 7, dtype=torch.long, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_embedding_bwd.py needs a GPU")
    from deepspeed_b200.ops.kernels.transformer_ops import embedding_bwd_
    smi = _smi()
    T = args.tokens
    for model, (V, H) in SHAPES.items():
        view = torch.zeros(V, H, dtype=torch.bfloat16, device="cuda")
        for kind in ("uniform", "zipf", "all_equal"):
            g = torch.Generator(device="cuda").manual_seed(0)
            ids = _ids(torch, kind, T, V, g)
            dy = torch.randn(T, H, generator=g, device="cuda").bfloat16()

            def native():
                embedding_bwd_(dy, ids, view)

            def dense():
                view.add_(torch.ops.aten.embedding_dense_backward(dy, ids, V, -1, False))

            ms_n = _time(torch, native, args.iters)
            ms_t = _time(torch, dense, args.iters)
            print(json.dumps({"model": model, "V": V, "H": H, "tokens": T, "ids": kind,
                              "unique_ids": int(torch.unique(ids).numel()), "native_ms": round(ms_n, 4),
                              "torch_dense_plus_add_ms": round(ms_t, 4), "speedup": round(ms_t / ms_n, 2),
                              "gpu": smi}), flush=True)


if __name__ == "__main__":
    main()
