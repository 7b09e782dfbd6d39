"""GEMM front door of the training hot path.

Every matrix product of the Llama-family step goes through one of

* :func:`matmul_nt` ``a[M,K] @ b[N,K]^T``            (``y = x W^T``)
* :func:`matmul_nn` ``a[M,K] @ b[K,N]``              (``dX = dY W``)
* :func:`matmul_tn` ``a[K,M]^T @ b[K,N]``            (``dW = dY^T X``), optionally *accumulating* into ``out``
* :func:`gate_up_swiglu`   ``silu(x Wg^T) * (x Wu^T)`` with the activation applied in the GEMM epilogue
* :func:`down_dx_dswiglu`  ``(dY Wd) (.) dSwiGLU(gate, up)`` with the activation backward applied in the GEMM epilogue

and is served either by the framework's own wgmma / TMA kernel (``csrc/cuda/gemm_sm90.cu``, "own") or by
cuBLASLt through ``torch.mm`` (+ the separate element-wise kernel for the fused forms, "lib").

Which one runs is decided **per problem shape by a persisted table** (``gemm_table.json`` next to this file, produced by
``scripts/tune_gemm.py`` on an H100 from >= 20 warm iterations per candidate with the clocks recorded).  A shape that is not
in the table is measured on first use with the same protocol (interleaved candidates, 5 warm-up + 20 timed iterations each,
median), and the own kernel is kept unless the library is more than ``TIE_MARGIN`` faster: inside a training step both are
power-capped, so an isolated few-percent edge of either does not survive, while the own kernel's fused epilogues do.
``DSB200_GEMM=own|lib|auto`` overrides (``sm100`` / ``cublas`` accepted as aliases).

Reference role: the cuBLAS algorithm sweep of ``csrc/includes/gemm_test.h:58`` + ``cublas_wrappers.cu:65``.
"""
import json
import os

import torch

_ALIASES = {"sm100": "own", "cublas": "lib", "auto": "auto", "own": "own", "lib": "lib"}
_backend = _ALIASES.get(os.environ.get("DSB200_GEMM", "auto").lower(), "auto")
TIE_MARGIN = 0.03
# fused-epilogue forms: the library alternative is a GEMM plus a separate element-wise pass over the [tokens, 2I]
# activations; timed alone that pass runs at full HBM bandwidth, inside a training step it shares HBM with the overlapped
# reduce-scatter / optimizer kernels (measured 0.23 ms alone vs 0.3-0.67 ms in-step), while the fused epilogue's traffic
# hides under the MMAs -- so the fused kernel is kept unless the library pair is clearly (> 10 %) faster in isolation
FUSED_TIE_MARGIN = 0.10
GROUP_M = int(os.environ.get("DSB200_GEMM_GROUP_M", "8"))
_TABLE_PATH = os.path.join(os.path.dirname(__file__), "gemm_table.json")

_table = None  # key -> "own" | "lib"
_table_gm = {}  # key -> rasterisation group size measured best for that shape
_table_meta = {}
_measured = {}  # key -> {"own_ms":, "lib_ms":} for shapes tuned online in this process
_own_ok = None


def set_backend(name: str):
    global _backend
    assert name in _ALIASES, name
    _backend = _ALIASES[name]


def get_backend():
    return _backend


def _load_table():
    global _table, _table_meta
    if _table is None:
        _table = {}
        try:
            with open(_TABLE_PATH) as f:
                blob = json.load(f)
            _table_meta = blob.get("meta", {})
            for k, v in blob.get("shapes", {}).items():
                _table[k] = v["choice"] if isinstance(v, dict) else v
                if isinstance(v, dict) and "group_m" in v:
                    _table_gm[k] = int(v["group_m"])
        except (OSError, ValueError):
            pass
    return _table


def tuning_table():
    """Choices made so far in this process (shipped-table hits and online measurements)."""
    return dict(_used)


def tuning_measurements():
    return dict(_measured)


_used = {}


def _own_available():
    """One-time numerical self check of the CTA-pair kernel on this device."""
    global _own_ok
    if _own_ok is None:
        if not torch.cuda.is_available() or _backend == "lib":
            _own_ok = False
            return False
        try:
            from deepspeed_b200.ops.kernels import gemm_sm100
            g = torch.Generator(device="cuda").manual_seed(0)
            a = torch.randn(640, 320, device="cuda", generator=g).bfloat16()
            b = torch.randn(768, 320, device="cuda", generator=g).bfloat16()
            c = gemm_sm100.matmul_2cta(a, b, False, False)
            ref = a.float() @ b.float().t()
            torch.cuda.synchronize()
            _own_ok = bool((c.float() - ref).abs().max() < 0.05 * ref.abs().max() + 0.5) and bool(torch.isfinite(c).all())
        except Exception:
            _own_ok = False
        if not _own_ok and _backend == "own":
            raise RuntimeError("DSB200_GEMM=own requested but the native wgmma GEMM failed its self check")
    return _own_ok


def _eligible(M, N, K, *tensors):
    """Own-kernel preconditions: bf16 CUDA row-major operands with 16-byte aligned rows, N % 8 == 0 (the kernel's
    16-byte column pairs; ``matmul_nt`` without ``out`` has no tensor whose rows are N long), at least one 256x128 tile."""
    if _backend == "lib" or M < 256 or N < 128 or K < 64 or N % 8:
        return False
    for t in tensors:
        if t is None:
            continue
        if not (t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 8 == 0
                and t.data_ptr() % 16 == 0 and t.shape[1] % 8 == 0):
            return False
    return _own_available()


def _time_interleaved(fns, warm=5, iters=20):
    """Median device time (ms) of each callable; candidates alternate so clock drift hits them equally."""
    for _ in range(warm):
        for f in fns:
            f()
    samples = [[] for _ in fns]
    for _ in range(iters):
        for i, f in enumerate(fns):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            e.synchronize()
            samples[i].append(s.elapsed_time(e))
    return [sorted(x)[len(x) // 2] for x in samples]


def _margin(key):
    return FUSED_TIE_MARGIN if key.startswith(("nt_swiglu", "nn_dswiglu")) else TIE_MARGIN


def _choose(key, own_fn, lib_fn):
    """-> "own" | "lib" for problem ``key``; ``own_fn`` / ``lib_fn`` run the problem on scratch outputs."""
    if _backend != "auto":
        choice = _backend
    else:
        choice = _used.get(key) or _load_table().get(key)
        if choice is None:
            if torch.cuda.is_current_stream_capturing():
                choice = "own"
            else:
                try:
                    t_own, t_lib = _time_interleaved([own_fn, lib_fn])
                    choice = "own" if t_own <= t_lib * (1.0 + _margin(key)) else "lib"
                    _measured[key] = {"own_ms": t_own, "lib_ms": t_lib}
                except Exception:
                    choice = "lib"
                release_scratch()  # tuning outputs can be hundreds of MB: never keep them next to a 150 GB model
    _used[key] = choice
    return choice


def _gm(key):
    _load_table()
    return _table_gm.get(key, GROUP_M)


def _report(macs):
    """Make the ctypes-launched GEMM visible to an active FlopsProfiler (ATen calls are counted by dispatch)."""
    from deepspeed_b200.profiling.flops_profiler import profiler as _p
    if _p._ACTIVE:
        _p.add_flops(2 * macs, macs)


def _k():
    from deepspeed_b200.ops.kernels import gemm_sm100
    return gemm_sm100


# ---------------------------------------------------------------------------------------------------------------------
def matmul_nt(a, b, out=None):
    """a [M, K] @ b[N, K]^T."""
    M, K = a.shape
    Nn = b.shape[0]
    if _eligible(M, Nn, K, a, b, out):
        key = f"nt:{M}x{Nn}x{K}"
        if _choose(key, lambda: _k().matmul_2cta(a, b, False, False, out=_scratch(M, Nn, a), group_m=GROUP_M),
                   lambda: torch.mm(a, b.t(), out=_scratch(M, Nn, a))) == "own":
            _report(M * Nn * K)
            return _k().matmul_2cta(a, b, False, False, out=out, group_m=_gm(key))
    return torch.mm(a, b.t(), out=out) if out is not None else torch.matmul(a, b.t())


def matmul_nn(a, b, out=None):
    """a [M, K] @ b [K, N]  (dX = dY @ W)."""
    M, K = a.shape
    Nn = b.shape[1]
    if out is None:
        out = torch.empty(M, Nn, dtype=a.dtype, device=a.device)
    if _eligible(M, Nn, K, a, b, out):
        key = f"nn:{M}x{Nn}x{K}"
        if _choose(key, lambda: _k().matmul_2cta(a, b, False, True, out=_scratch(M, Nn, a), group_m=GROUP_M),
                   lambda: torch.mm(a, b, out=_scratch(M, Nn, a))) == "own":
            _report(M * Nn * K)
            return _k().matmul_2cta(a, b, False, True, out=out, group_m=_gm(key))
    return torch.mm(a, b, out=out)


def matmul_tn(a, b, out=None, accumulate=False):
    """a[K, M]^T @ b[K, N]  (dW = dY^T @ X), written -- or with ``accumulate`` added -- straight into ``out`` (typically
    a view of the ZeRO flat gradient buffer: no AccumulateGrad, no bucket copy, no memset)."""
    K, M = a.shape
    Nn = b.shape[1]
    if out is None:
        assert not accumulate
        out = torch.empty(M, Nn, dtype=a.dtype, device=a.device)
    if _eligible(M, Nn, K, a, b, out) and M % 8 == 0:
        key = f"{'tn_acc' if accumulate else 'tn'}:{M}x{Nn}x{K}"
        epi = 1 if accumulate else 0

        def lib(o):
            return o.addmm_(a.t(), b) if accumulate else torch.mm(a.t(), b, out=o)

        if _choose(key, lambda: _k().matmul_2cta(a, b, True, True, out=_scratch(M, Nn, a), epi=epi, group_m=GROUP_M),
                   lambda: lib(_scratch(M, Nn, a))) == "own":
            _report(M * Nn * K)
            return _k().matmul_2cta(a, b, True, True, out=out, epi=epi, group_m=_gm(key))
    if accumulate:
        return out.addmm_(a.t(), b)
    return torch.mm(a.t(), b, out=out)


def _swiglu_key(x, w_gu):
    """Table key of the fused gate|up + SwiGLU problem, or None when the own kernel cannot take these operands."""
    T, H = x.shape
    I = w_gu.shape[0] // 2
    return f"nt_swiglu:{T}x{I}x{H}" if _eligible(T, I, H, x, w_gu) and I % 128 == 0 else None


def gate_up_swiglu_in_tree(x, w_gu) -> bool:
    """Whether :func:`gate_up_swiglu` of these operands ran the own fused kernel (valid after that call).  Its ``act`` then
    comes from the fp32 accumulators and differs from ``silu(gate) * up`` recomputed from the bf16 ``gate_up``; on the
    library path the two are bit-identical (:func:`down_dx_dswiglu` ``act_out``)."""
    key = _swiglu_key(x, w_gu)
    return key is not None and _used.get(key) == "own"


def gate_up_swiglu(x, w_gu, save_gate_up=True):
    """``x [T, H]``, ``w_gu [2I, H]`` (gate rows then up rows) -> ``(act [T, I], gate_up [T, 2I] | None)`` where
    ``act = silu(x Wg^T) * (x Wu^T)``.  Own path: ONE kernel (activation in the GEMM epilogue, gate|up saved for backward
    from the same accumulators); library path: :func:`matmul_nt` + the element-wise gated-activation kernel."""
    T, H = x.shape
    I = w_gu.shape[0] // 2
    key = _swiglu_key(x, w_gu)
    if key is not None:

        def own(scratch=True):
            act = _scratch(T, I, x, 1) if scratch else torch.empty(T, I, dtype=x.dtype, device=x.device)
            gu = None
            if save_gate_up:
                gu = _scratch(T, 2 * I, x, 2) if scratch else torch.empty(T, 2 * I, dtype=x.dtype, device=x.device)
            _k().matmul_2cta(x, w_gu, False, False, out=act, epi=2, out2=gu, inter=I, group_m=_gm(key))
            return act, gu

        def lib():
            from deepspeed_b200.ops.kernels import transformer_ops as T_
            gu = torch.mm(x, w_gu.t(), out=_scratch(T, 2 * I, x, 2))
            return T_.gated_act_fwd_raw(gu)

        if _choose(key, own, lib) == "own":
            _report(T * 2 * I * H)
            return own(scratch=False)
    from deepspeed_b200.ops.kernels import transformer_ops as T_
    gu = matmul_nt(x, w_gu)
    return T_.gated_act_fwd_raw(gu), (gu if save_gate_up else None)


def down_dx_dswiglu(dy, w_down, gate_up, act_out=None):
    """``dy [T, H]``, ``w_down [H, I]``, saved ``gate_up [T, 2I]`` -> ``dgate_up [T, 2I]``: the down-projection's input
    gradient ``dy @ w_down`` never reaches memory -- the SwiGLU backward is applied to the accumulators in the epilogue.
    ``act_out [T, I]`` (optional) receives ``silu(gate) * up`` of ``gate_up``, bit-identical to the library path of
    :func:`gate_up_swiglu`: written by the library path's dSwiGLU pass, or on the own path by a gated-activation pass
    after the fused kernel."""
    T, H = dy.shape
    I = w_down.shape[1]
    if _eligible(T, I, H, dy, w_down, gate_up):
        key = f"nn_dswiglu:{T}x{I}x{H}"

        def own(scratch=True):
            dgu = _scratch(T, 2 * I, dy, 3) if scratch else torch.empty(T, 2 * I, dtype=dy.dtype, device=dy.device)
            _k().matmul_2cta(dy, w_down, False, True, out=dgu[:, :I], epi=3, aux=gate_up, out2=dgu, inter=I, group_m=_gm(key))
            return dgu

        def lib():
            from deepspeed_b200.ops.kernels import transformer_ops as T_
            d_act = torch.mm(dy, w_down, out=_scratch(T, I, dy, 1))
            return T_.gated_act_bwd(d_act, gate_up, "silu")

        if _choose(key, own, lib) == "own":
            _report(T * I * H)
            dgu = own(scratch=False)
            if act_out is not None:
                from deepspeed_b200.ops.kernels import transformer_ops as T_
                T_.gated_act_fwd_raw(gate_up, "silu", out=act_out)
            return dgu
    from deepspeed_b200.ops.kernels import transformer_ops as T_
    return T_.gated_act_bwd(matmul_nn(dy, w_down), gate_up, "silu", act_out=act_out)


_scratch_bufs = {}


def _scratch(m, n, like, slot=0):
    """Tuning-time output buffers (never used for results)."""
    key = (m, n, like.device, slot)
    t = _scratch_bufs.get(key)
    if t is None:
        if len(_scratch_bufs) > 8:
            _scratch_bufs.clear()
        t = torch.empty(m, n, dtype=like.dtype, device=like.device)
        _scratch_bufs[key] = t
    return t


def release_scratch():
    _scratch_bufs.clear()
