"""Build ``deepspeed_b200/ops/gemm_table.json``: the persisted per-shape choice between the in-tree wgmma GEMM ("own") and
cuBLASLt ("lib") for every GEMM problem of the benchmark models' training step.

Protocol per problem: candidates alternate (so clock drift hits them equally), 5 warm-up + ``--iters`` (>= 20) timed
iterations each, CUDA events, median; the operands of the Llama-3-8B problems (>= 64 MB each, together > L2) are re-read
from HBM every iteration.  ``nvidia-smi`` clocks are sampled during the whole run and stored in the table's ``meta``.

    python scripts/tune_gemm.py [--tokens 8192] [--iters 20] [--models llama3-8b,phi3-mini] [--out ...]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from deepspeed_b200.models.llama import llama_config
from deepspeed_b200.ops import gemm
from deepspeed_b200.ops.kernels import gemm_sm100 as K
from deepspeed_b200.ops.kernels import transformer_ops as T

ap = argparse.ArgumentParser()
ap.add_argument("--tokens", default="8192")
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--models", default="llama3-8b,phi3-mini,llama3-70b")
ap.add_argument("--loss-chunk", type=int, default=2048)
ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "deepspeed_b200",
                                              "ops", "gemm_table.json"))
ap.add_argument("--report", default="gpurun_out/gemm_tune_report.json")
ap.add_argument("--group-m", default="8")
a = ap.parse_args()
dev = "cuda"


class Clocks:

    def __init__(self):
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        self.lines = []
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "200", "-i",
                                       "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=lambda: [self.lines.append(l.strip()) for l in self.p.stdout], daemon=True).start()
        except Exception:
            self.p = None

    def stop(self):
        if self.p is None:
            return {"reasons": ["unavailable"]}
        self.p.terminate()
        sm, mx, pw, reasons = [], None, [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx = float(f[1]); pw.append(float(f[2]))
            except ValueError:
                continue
            for n, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz_median": statistics.median(sm) if sm else None, "sm_max_mhz": mx,
                "power_w_max": max(pw) if pw else None, "reasons": sorted(reasons), "samples": len(sm)}


def rnd(*shape):
    return (torch.randn(*shape, device=dev) * 0.05).bfloat16()


def problems(cfg, tokens, chunk):
    """(key, own_fn, lib_fn, flops) for every GEMM of one decoder layer + the chunked LM head, forward and backward."""
    H, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    qkv = cfg.q_size + 2 * cfg.kv_size
    out = []
    lin = [("qkv", qkv, H), ("o", H, cfg.q_size), ("down", H, I)]
    for name, n, k in lin:
        out.append(("nt", tokens, n, k))
        out.append(("nn", tokens, k, n))       # dX = dY[T, n] @ W[n, k]
        out.append(("tn", n, k, tokens))       # dW[n, k] = dY^T X
        out.append(("tn_acc", n, k, tokens))
    out.append(("nt_swiglu", tokens, I, H))
    out.append(("nn_dswiglu", tokens, I, H))
    out.append(("nn", tokens, H, 2 * I))       # dX of gate_up
    out.append(("tn", 2 * I, H, tokens))
    out.append(("tn_acc", 2 * I, H, tokens))
    c = min(chunk, tokens)
    out.append(("nt", c, V, H))                # LM head chunk
    out.append(("nn", c, H, V))
    out.append(("tn", V, H, c))
    out.append(("tn_acc", V, H, c))
    return out


def runner(kind, M, N, Kd, gm):
    """-> (own_fn, lib_fn) operating on private buffers."""
    if kind == "nt":
        x, w, o = rnd(M, Kd), rnd(N, Kd), torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        return (lambda: K.matmul_2cta(x, w, False, False, out=o, group_m=gm)), (lambda: torch.mm(x, w.t(), out=o))
    if kind == "nn":
        x, w, o = rnd(M, Kd), rnd(Kd, N), torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        return (lambda: K.matmul_2cta(x, w, False, True, out=o, group_m=gm)), (lambda: torch.mm(x, w, out=o))
    if kind in ("tn", "tn_acc"):
        dy, x, o = rnd(Kd, M), rnd(Kd, N), torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
        if kind == "tn":
            return (lambda: K.matmul_2cta(dy, x, True, True, out=o, group_m=gm)), (lambda: torch.mm(dy.t(), x, out=o))
        return (lambda: K.matmul_2cta(dy, x, True, True, out=o, epi=K.EPI_ACCUM, group_m=gm)), (lambda: o.addmm_(dy.t(), x, beta=1.0, alpha=1e-3))
    if kind == "nt_swiglu":
        x, w = rnd(M, Kd), rnd(2 * N, Kd)
        act, gu = torch.empty(M, N, device=dev, dtype=torch.bfloat16), torch.empty(M, 2 * N, device=dev, dtype=torch.bfloat16)

        def lib():
            torch.mm(x, w.t(), out=gu)
            T.gated_act_fwd_raw(gu)

        return (lambda: K.matmul_2cta(x, w, False, False, out=act, epi=K.EPI_SWIGLU, out2=gu, inter=N, group_m=gm)), lib
    if kind == "nn_dswiglu":
        dy, w, gu = rnd(M, Kd), rnd(Kd, N), rnd(M, 2 * N)
        dgu, dact = torch.empty(M, 2 * N, device=dev, dtype=torch.bfloat16), torch.empty(M, N, device=dev, dtype=torch.bfloat16)

        def lib():
            torch.mm(dy, w, out=dact)
            T.gated_act_bwd(dact, gu)

        return (lambda: K.matmul_2cta(dy, w, False, True, out=dgu[:, :N], epi=K.EPI_DSWIGLU, aux=gu, out2=dgu, inter=N,
                                      group_m=gm)), lib
    raise ValueError(kind)


clk = Clocks()
t_start = time.time()
shapes, report = {}, []
seen = set()
gms = [int(g) for g in a.group_m.split(",")]
for model in a.models.split(","):
    cfg = llama_config(model)
    for tokens in [int(t) for t in a.tokens.split(",")]:
        for (kind, M, N, Kd) in problems(cfg, tokens, a.loss_chunk):
            key = f"{kind}:{M}x{N}x{Kd}"
            if key in seen:
                continue
            seen.add(key)
            try:
                fns, lib = [], None
                for gm in gms:
                    own, lib = runner(kind, M, N, Kd, gm)
                    fns.append(own)
                ts = gemm._time_interleaved(fns + [lib], warm=5, iters=a.iters)
            except Exception as e:  # noqa
                print(f"{key}: FAILED {type(e).__name__}: {e}", flush=True)
                torch.cuda.empty_cache()
                continue
            t_own, t_lib = min(ts[:-1]), ts[-1]
            best_gm = gms[ts.index(t_own)]
            flops = 2.0 * M * N * Kd * (2 if kind == "nt_swiglu" else 1)
            choice = "own" if t_own <= t_lib * (1 + gemm._margin(key)) else "lib"
            shapes[key] = {"choice": choice, "own_ms": round(t_own, 4), "lib_ms": round(t_lib, 4),
                           "own_tflops": round(flops / t_own / 1e9, 1), "lib_tflops": round(flops / t_lib / 1e9, 1),
                           "group_m": best_gm, "model": model}
            report.append(dict(key=key, **shapes[key], per_group_m={str(g): round(t, 4) for g, t in zip(gms, ts[:-1])}))
            print(f"{key:34s} own {t_own:8.4f} ms ({flops / t_own / 1e9:7.1f} TF)  lib {t_lib:8.4f} ms "
                  f"({flops / t_lib / 1e9:7.1f} TF) -> {choice} (group_m {best_gm})", flush=True)
            del fns, lib, own
            torch.cuda.empty_cache()
meta = {"gpu": torch.cuda.get_device_name(0), "torch": torch.__version__, "iters": a.iters, "tie_margin": gemm.TIE_MARGIN,
        "protocol": "interleaved candidates, 5 warm-up + iters timed, CUDA events, median", "clocks": clk.stop(),
        "when": time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime()), "wall_s": round(time.time() - t_start, 1)}
blob = {"meta": meta, "shapes": shapes}
os.makedirs(os.path.dirname(a.report), exist_ok=True)
json.dump({"meta": meta, "rows": report}, open(a.report, "w"), indent=1)
json.dump(blob, open(a.out, "w"), indent=1)
n_own = sum(1 for v in shapes.values() if v["choice"] == "own")
print(f"wrote {a.out}: {n_own}/{len(shapes)} shapes -> own kernel; clocks {meta['clocks']}")
