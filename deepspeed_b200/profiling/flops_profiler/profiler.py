"""FLOPs / MACs / latency / parameter profiler with a per-module tree.

API parity: reference ``profiling/flops_profiler/profiler.py`` (``FlopsProfiler :30``, ``get_model_profile
:1131``, ``print_model_profile``).  Mechanism differs: the reference monkey-patches ``torch.nn.functional`` and
``torch.Tensor`` methods; here a ``TorchDispatchMode`` counts at the ATen level (every matmul / conv / SDPA that
actually runs, including those issued from custom autograd functions), module pre/post hooks attribute the
counts to the innermost active module, and this framework's own ctypes kernels report through
``add_flops`` (see ``ops/gemm.py``).  Latency per module comes from CUDA events on GPU (host clock on CPU).
"""
import time
from collections import defaultdict
from functools import partial
from typing import List, Optional

import torch
from torch import nn
from torch.utils._python_dispatch import TorchDispatchMode

_ACTIVE: List["FlopsProfiler"] = []


def add_flops(flops: int, macs: Optional[int] = None):
    """Called by native (non-ATen) kernels so they are visible to an active profiler."""
    for p in _ACTIVE:
        p._add(flops, flops // 2 if macs is None else macs)


def _prod(xs):
    r = 1
    for x in xs:
        r *= int(x)
    return r


def _mm(a, b):
    return _prod(a.shape) * b.shape[-1]


def _count(func, args, out):
    """-> (flops, macs) of one ATen call (0,0 for everything that is not counted)."""
    name = func.__name__ if hasattr(func, "__name__") else str(func)
    pkt = str(getattr(func, "_overloadpacket", func))
    op = pkt.split(".")[-1]
    try:
        if op in ("mm", "matmul"):
            m = _mm(args[0], args[1])
            return 2 * m, m
        if op == "addmm":
            m = _mm(args[1], args[2])
            return 2 * m + _prod(out.shape), m
        if op == "bmm":
            m = _prod(args[0].shape) * args[1].shape[-1]
            return 2 * m, m
        if op == "baddbmm":
            m = _prod(args[1].shape) * args[2].shape[-1]
            return 2 * m + _prod(out.shape), m
        if op == "linear":
            m = _prod(args[0].shape) * args[1].shape[0]
            return 2 * m, m
        if op in ("convolution", "_convolution", "cudnn_convolution"):
            x, w = args[0], args[1]
            o = out if torch.is_tensor(out) else out[0]
            m = _prod(o.shape) * _prod(w.shape[1:])
            return 2 * m, m
        if op.startswith("_scaled_dot_product") or op == "scaled_dot_product_attention":
            q, k = args[0], args[1]
            B, H, Sq, D = q.shape[-4] if q.dim() == 4 else 1, q.shape[-3], q.shape[-2], q.shape[-1]
            Sk = k.shape[-2]
            bwd = "backward" in op
            m = B * H * Sq * Sk * D * 2
            m = int(m * (2.5 if bwd else 1.0))
            return 2 * m, m
        if op in ("native_layer_norm", "native_group_norm", "native_batch_norm", "_native_batch_norm_legit"):
            return 5 * _prod(args[0].shape), 0
        if op in ("_softmax", "_log_softmax"):
            return 3 * _prod(args[0].shape), 0
        if op in ("gelu", "silu", "relu", "tanh", "sigmoid", "mul", "add", "sub", "div"):
            o = out if torch.is_tensor(out) else None
            return (_prod(o.shape) if o is not None else 0), 0
        if op in ("embedding", ):
            return 0, 0
    except Exception:
        return 0, 0
    return 0, 0


class _Counter(TorchDispatchMode):

    def __init__(self, prof):
        super().__init__()
        self.prof = prof

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        f, m = _count(func, args, out)
        if f:
            self.prof._add(f, m)
        return out


class FlopsProfiler:

    def __init__(self, model, ds_engine=None, recompute_fwd_factor=0.0):
        self.model = model
        self.ds_engine = ds_engine
        self.recompute_fwd_factor = recompute_fwd_factor
        self.started = False
        self.func_patched = False
        self._hooks = []
        self._stack = []
        self._mode = None
        self._done = False
        self._t0 = None

    # ---- counting plumbing
    def _add(self, flops, macs):
        if self._stack:
            m = self._stack[-1]
            m.__flops__ += flops
            m.__macs__ += macs
        else:
            self.model.__flops__ = getattr(self.model, "__flops__", 0) + flops
            self.model.__macs__ = getattr(self.model, "__macs__", 0) + macs

    def _now(self):
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        return time.perf_counter()

    def start_profile(self, ignore_list=None):
        self.reset_profile()
        ignore = tuple(ignore_list or ())

        def pre(mod, inp):
            self._stack.append(mod)
            mod.__start_time__ = self._now() if self._timed(mod) else None

        def post(mod, inp, out):
            if mod.__start_time__ is not None:
                mod.__duration__ += self._now() - mod.__start_time__
            if self._stack and self._stack[-1] is mod:
                self._stack.pop()

        for mod in self.model.modules():
            if ignore and isinstance(mod, ignore):
                continue
            self._hooks.append(mod.register_forward_pre_hook(pre))
            self._hooks.append(mod.register_forward_hook(post))
        self._mode = _Counter(self)
        self._mode.__enter__()
        _ACTIVE.append(self)
        self.started = True
        self._done = False
        self._t0 = self._now()

    def _timed(self, mod):
        # synchronising around every leaf would distort totals; time containers with children + the root only
        return mod is self.model or len(list(mod.children())) > 0

    def stop_profile(self):
        if not self.started:
            return
        self._total_duration = self._now() - self._t0
        if self._mode is not None:
            self._mode.__exit__(None, None, None)
            self._mode = None
        if self in _ACTIVE:
            _ACTIVE.remove(self)
        for h in self._hooks:
            h.remove()
        self._hooks.clear()
        self.started = False
        self._done = True

    def reset_profile(self):
        for mod in self.model.modules():
            mod.__flops__ = 0
            mod.__macs__ = 0
            mod.__duration__ = 0.0
            mod.__start_time__ = None
            mod.__params__ = sum(getattr(p, "ds_numel", p.numel()) for p in mod.parameters(recurse=False))
        self._stack = []

    def end_profile(self):
        if self.started:
            self.stop_profile()
        for mod in self.model.modules():
            for a in ("__flops__", "__macs__", "__duration__", "__start_time__", "__params__"):
                if hasattr(mod, a):
                    delattr(mod, a)
        self._done = False

    def has_result(self):
        return self._done

    # ---- aggregation
    @staticmethod
    def _sum(mod, attr):
        return getattr(mod, attr, 0) + sum(FlopsProfiler._sum(c, attr) for c in mod.children())

    def get_total_flops(self, as_string=False):
        v = self._sum(self.model, "__flops__")
        return flops_to_string(v) if as_string else v

    def get_total_macs(self, as_string=False):
        v = self._sum(self.model, "__macs__")
        return macs_to_string(v) if as_string else v

    def get_total_duration(self, as_string=False):
        v = getattr(self.model, "__duration__", 0.0) or getattr(self, "_total_duration", 0.0)
        return duration_to_string(v) if as_string else v

    def get_total_params(self, as_string=False):
        v = self._sum(self.model, "__params__")
        return params_to_string(v) if as_string else v

    def is_expert_tensor_parallelism_enabled(self):
        return False

    def print_model_profile(self, profile_step=1, module_depth=-1, top_modules=1, detailed=True, output_file=None):
        if not self._done and not self.started:
            return
        import sys
        out = open(output_file, "w") if output_file else sys.stdout
        p = partial(print, file=out)
        total_flops, total_macs = self.get_total_flops(), self.get_total_macs()
        total_dur, total_params = self.get_total_duration(), self.get_total_params()
        p("\n-------------------------- DeepSpeed-H100 Flops Profiler --------------------------")
        p(f"Profile Summary at step {profile_step}:")
        p("Notations:\n  data parallel size (dp_size), model parallel size(mp_size),\n  number of parameters (params), "
          "number of multiply-accumulate operations(MACs),\n  number of floating-point operations (flops), "
          "floating-point operations per second (FLOPS),\n  fwd latency (forward propagation latency), bwd latency "
          "(backward propagation latency),\n  step (weights update latency), iter latency (sum of fwd, bwd and step "
          "latency)\n")
        eng = self.ds_engine
        if eng is not None:
            p(f"{'world size: ':<60}  {eng.world_size}")
            p(f"{'data parallel size: ':<60}  {eng.dp_world_size}")
            p(f"{'model parallel size: ':<60}  {eng.mp_world_size}")
            p(f"{'batch size per GPU: ':<60}  {eng.train_micro_batch_size_per_gpu()}")
        p(f"{'params per GPU: ':<60}  {params_to_string(total_params)}")
        p(f"{'fwd MACs per GPU: ':<60}  {macs_to_string(total_macs)}")
        p(f"{'fwd flops per GPU: ':<60}  {number_to_string(total_flops)}")
        p(f"{'fwd latency: ':<60}  {duration_to_string(total_dur)}")
        if total_dur > 0:
            p(f"{'fwd FLOPS per GPU = fwd flops per GPU / fwd latency: ':<60}  {flops_to_string(total_flops / total_dur)}")
        if eng is not None and getattr(eng, "wall_clock_breakdown", lambda: False)():
            from deepspeed_b200.utils.timer import BACKWARD_GLOBAL_TIMER, STEP_GLOBAL_TIMER
            bwd = eng.timers(BACKWARD_GLOBAL_TIMER).elapsed(reset=False) / 1000.0
            stp = eng.timers(STEP_GLOBAL_TIMER).elapsed(reset=False) / 1000.0
            f = 2.0 + self.recompute_fwd_factor
            if bwd > 0:
                p(f"{'bwd latency: ':<60}  {duration_to_string(bwd)}")
                p(f"{'bwd FLOPS per GPU = ' + str(f) + ' * fwd flops per GPU / bwd latency: ':<60}  "
                  f"{flops_to_string(f * total_flops / bwd)}")
                p(f"{'fwd+bwd FLOPS per GPU: ':<60}  {flops_to_string((1 + f) * total_flops / (total_dur + bwd))}")
            p(f"{'step latency: ':<60}  {duration_to_string(stp)}")
            it = total_dur + bwd + stp
            p(f"{'iter latency: ':<60}  {duration_to_string(it)}")
            if it > 0:
                p(f"{'FLOPS per GPU = (1 + f) * fwd flops per GPU / iter latency: ':<60}  "
                  f"{flops_to_string((1 + f) * total_flops / it)}")
                p(f"{'samples/second: ':<60}  {eng.train_micro_batch_size_per_gpu() / it:.2f}")
        if detailed:
            self.print_model_aggregated_profile(module_depth=module_depth, top_modules=top_modules, file=out)
            p("\n------------------------------ Detailed Profile per GPU ------------------------------")
            p("Each module profile is listed after its name in the following order: \nparams, percentage of total "
              "params, MACs, percentage of total MACs, fwd latency, percentage of total fwd latency, fwd FLOPS\n")
            self._print_tree(self.model, type(self.model).__name__, 0, module_depth, total_params, total_macs, total_dur, p)
        p("------------------------------------------------------------------------------")
        if output_file:
            out.close()

    def _line(self, mod, total_params, total_macs, total_dur):
        params, macs = self._sum(mod, "__params__"), self._sum(mod, "__macs__")
        flops, dur = self._sum(mod, "__flops__"), getattr(mod, "__duration__", 0.0)
        items = [params_to_string(params), f"{params / total_params:.2%} Params" if total_params else "0% Params",
                 macs_to_string(macs), f"{macs / total_macs:.2%} MACs" if total_macs else "0% MACs"]
        if dur:
            items += [duration_to_string(dur), f"{dur / total_dur:.2%} latency" if total_dur else "",
                      flops_to_string(flops / dur)]
        return ", ".join(items)

    def _print_tree(self, mod, name, depth, max_depth, tp, tm, td, p):
        p("  " * depth + f"{name}: {type(mod).__name__}({self._line(mod, tp, tm, td)})")
        if max_depth >= 0 and depth >= max_depth:
            return
        for n, c in mod.named_children():
            self._print_tree(c, n, depth + 1, max_depth, tp, tm, td, p)

    def print_model_aggregated_profile(self, module_depth=-1, top_modules=1, file=None):
        import sys
        p = partial(print, file=file or sys.stdout)
        info = defaultdict(lambda: defaultdict(lambda: [0, 0, 0.0]))

        def walk(mod, d):
            e = info[d][type(mod).__name__]
            e[0] += self._sum(mod, "__macs__")
            e[1] += self._sum(mod, "__params__")
            e[2] += getattr(mod, "__duration__", 0.0)
            for c in mod.children():
                walk(c, d + 1)

        walk(self.model, 0)
        depths = sorted(info)
        if module_depth >= 0:
            depths = [d for d in depths if d <= module_depth]
        elif module_depth == -1 and depths:
            depths = [depths[-1]]
        p("\n----------------------------- Aggregated Profile per GPU -----------------------------")
        p(f"Top {top_modules} modules in terms of params, MACs or fwd latency at different model depths:")
        for d in depths:
            n = min(top_modules, len(info[d]))
            p(f"depth {d}:")
            for key, idx, fmt in (("params", 1, params_to_string), ("MACs", 0, macs_to_string), ("fwd latency", 2,
                                                                                                   duration_to_string)):
                top = sorted(info[d].items(), key=lambda kv: kv[1][idx], reverse=True)[:n]
                p(f"    {key:<12}- " + str({k: fmt(v[idx]) for k, v in top}))


# ---------------------------------------------------------------------------------------------------------- formatting
def number_to_string(num, units=None, precision=2):
    if units is None:
        for u, s in (("T", 1e12), ("G", 1e9), ("M", 1e6), ("K", 1e3)):
            if abs(num) >= s:
                return f"{num / s:.{precision}f} {u}"
        return f"{num:.{precision}f} "
    s = {"T": 1e12, "G": 1e9, "M": 1e6, "K": 1e3, "": 1, "m": 1e-3, "u": 1e-6}[units]
    return f"{num / s:.{precision}f} {units}"


def flops_to_string(flops, units=None, precision=2):
    return number_to_string(flops, units, precision) + "FLOPS"


def macs_to_string(macs, units=None, precision=2):
    return number_to_string(macs, units, precision) + "MACs"


def bytes_to_string(b, units=None, precision=2):
    return number_to_string(b, units, precision) + "B"


def params_to_string(n, units=None, precision=2):
    return number_to_string(n, units, precision).strip()


def duration_to_string(d, units=None, precision=2):
    if units is None:
        if d >= 1:
            return f"{d:.{precision}f} s"
        if d >= 1e-3:
            return f"{d * 1e3:.{precision}f} ms"
        return f"{d * 1e6:.{precision}f} us"
    return number_to_string(d, units, precision) + "s"


def get_model_profile(model, input_shape=None, args=(), kwargs=None, print_profile=True, detailed=True, module_depth=-1,
                      top_modules=1, warm_up=1, as_string=True, output_file=None, ignore_modules=None, mode="forward"):
    """One-shot profile of ``model(*args, **kwargs)`` (or a ones tensor of ``input_shape``).
    Returns ``(flops, macs, params)``."""
    assert isinstance(model, nn.Module), "model must be a PyTorch module"
    kwargs = dict(kwargs or {})
    args = list(args)
    if input_shape is not None:
        assert isinstance(input_shape, tuple) and len(input_shape) >= 1, "input_shape must be a non-empty tuple"
        try:
            p = next(model.parameters())
            inp = torch.ones((), dtype=p.dtype, device=p.device).new_empty(input_shape)
        except StopIteration:
            inp = torch.ones(()).new_empty(input_shape)
        args = [inp]
    fn = model.generate if mode == "generate" else model
    model.eval()
    with torch.no_grad():
        for _ in range(warm_up):
            fn(*args, **kwargs)
    prof = FlopsProfiler(model)
    prof.start_profile(ignore_list=ignore_modules)
    with torch.no_grad():
        fn(*args, **kwargs)
    prof.stop_profile()
    flops, macs, params = prof.get_total_flops(), prof.get_total_macs(), prof.get_total_params()
    if print_profile:
        prof.print_model_profile(profile_step=warm_up, module_depth=module_depth, top_modules=top_modules,
                                 detailed=detailed, output_file=output_file)
    prof.end_profile()
    if as_string:
        return number_to_string(flops), macs_to_string(macs), params_to_string(params)
    return flops, macs, params


# --- per-module aggregation helpers (reference ``profiler.py:1171-1192``) -----------------------------------------------
def get_module_flops(module):
    """FLOPs counted under ``module`` including all descendants."""
    return FlopsProfiler._sum(module, "__flops__")


def get_module_macs(module):
    return FlopsProfiler._sum(module, "__macs__")


def get_module_duration(module):
    """Wall time attributed to ``module``; untimed containers (e.g. ``ModuleList``) report the sum of their children."""
    own = getattr(module, "__duration__", 0.0) or 0.0
    return own if own else sum(get_module_duration(c) for c in module.children())


def wrapFunc(func, funcFlopCompute):
    """Wrap a functional op that is invisible to the dispatch-mode counter (a native kernel binding): the wrapper calls
    ``funcFlopCompute(*args, **kw) -> (flops, macs)`` and reports to whichever profiler is active (reference ``:866``)."""
    import functools

    @functools.wraps(func)
    def counted(*args, **kwds):
        if _ACTIVE:
            flops, macs = funcFlopCompute(*args, **kwds)
            add_flops(int(flops), int(macs) if macs else 0)
        return func(*args, **kwds)

    counted.__wrapped_for_flops__ = func
    return counted
