"""Activation checkpointing with partitioned / host-offloaded saved activations.

Parity target: reference ``runtime/activation_checkpointing/checkpointing.py`` (``CheckpointFunction
:488``, ``partition_activations :377``, ``gather_partitioned_activations :266``,
``non_reentrant_checkpoint :704``, ``CudaRNGStatesTracker :124``, ``configure :1029``).

Features: recompute-in-backward with exact RNG replay (CPU, CUDA and the model-parallel RNG tracker);
``partition_activations`` keeps only ``1/tp`` of every saved input per tensor-parallel rank and
all-gathers it in backward; ``cpu_checkpointing`` parks saved inputs in pinned host memory with
asynchronous copies on a side stream (CUDA events order them against compute, no device-wide
sync); ``contiguous_memory_optimization`` packs the partitions of one checkpoint into a single
pre-allocated buffer; ``synchronize_checkpoint_boundary`` and ``profile`` flags are honoured.
"""
import contextlib
from typing import Optional

import torch

from deepspeed_b200 import comm as dist
from deepspeed_b200.accelerator import get_accelerator
from deepspeed_b200.utils.logging import logger
from deepspeed_b200.utils.timer import SynchronizedWallClockTimer

# ---- module-level configuration (reference keeps these as globals too) ------------------------------
mpu = None
mp_rank = None
mp_size = None
mp_group = None
num_layers = None
PARTITION_ACTIVATIONS = False
CPU_CHECKPOINT = False
CONTIGUOUS_CHECKPOINTING = False
SYNCHRONIZE = False
PROFILE_TIME = False
deepspeed_checkpointing_enabled = False
_configured = False
timers = None
_copy_stream = None

_MODEL_PARALLEL_RNG_TRACKER_NAME = "model-parallel-rng"


# =====================================================================================================
# RNG tracking
# =====================================================================================================
class CudaRNGStatesTracker:
    """Named CUDA RNG streams so dropout inside tensor-parallel regions differs per TP rank while
    data-parallel replicas stay identical (Megatron convention)."""

    def __init__(self):
        self.states_ = {}
        self.seeds_ = set()

    def reset(self):
        self.states_ = {}
        self.seeds_ = set()

    def get_states(self):
        return dict(self.states_)

    def set_states(self, states):
        self.states_ = states

    def add(self, name, seed):
        if seed in self.seeds_:
            raise Exception(f"seed {seed} already exists")
        self.seeds_.add(seed)
        if name in self.states_:
            raise Exception(f"cuda rng state {name} already exists")
        acc = get_accelerator()
        orig = acc.get_rng_state()
        acc.manual_seed(seed)
        self.states_[name] = acc.get_rng_state()
        acc.set_rng_state(orig)

    @contextlib.contextmanager
    def fork(self, name=_MODEL_PARALLEL_RNG_TRACKER_NAME):
        if name not in self.states_:
            raise Exception(f"cuda rng state {name} is not added")
        acc = get_accelerator()
        orig = acc.get_rng_state()
        acc.set_rng_state(self.states_[name])
        try:
            yield
        finally:
            self.states_[name] = acc.get_rng_state()
            acc.set_rng_state(orig)


_CUDA_RNG_STATE_TRACKER = CudaRNGStatesTracker()


def get_cuda_rng_tracker():
    return _CUDA_RNG_STATE_TRACKER


def model_parallel_cuda_manual_seed(seed):
    """Default RNG = ``seed`` (same across TP ranks), tracker RNG = ``seed + 2718 + tp_rank``."""
    global mpu
    tp_rank = mpu.get_model_parallel_rank() if mpu is not None else 0
    offset = seed + 2718
    _CUDA_RNG_STATE_TRACKER.reset()
    get_accelerator().manual_seed(seed)
    _CUDA_RNG_STATE_TRACKER.add(_MODEL_PARALLEL_RNG_TRACKER_NAME, offset + tp_rank)


model_parallel_reconfigure_tp_seed = model_parallel_cuda_manual_seed


def _capture_rng():
    acc = get_accelerator()
    return (torch.get_rng_state(), acc.get_rng_state() if acc.device_name() == "cuda" and acc.is_available() else None,
            get_cuda_rng_tracker().get_states())


def _restore_rng(state):
    cpu, dev, tracker = state
    torch.set_rng_state(cpu)
    if dev is not None:
        get_accelerator().set_rng_state(dev)
    get_cuda_rng_tracker().set_states(tracker)


# =====================================================================================================
# partition / offload helpers
# =====================================================================================================
def _tp():
    global mp_rank, mp_size, mp_group
    if mpu is None:
        return 0, 1, None
    if mp_size is None:
        mp_size = mpu.get_model_parallel_world_size()
        mp_rank = mpu.get_model_parallel_rank()
        mp_group = mpu.get_model_parallel_group()
    return mp_rank, mp_size, mp_group


def get_partition_size(item):
    _, size, _ = _tp()
    return (item.numel() + size - 1) // size


def get_partition_start(item):
    rank, _, _ = _tp()
    return get_partition_size(item) * rank


def _copy_side_stream():
    global _copy_stream
    if _copy_stream is None and torch.cuda.is_available():
        _copy_stream = torch.cuda.Stream()
    return _copy_stream


class _Saved:
    """One saved forward input, possibly partitioned across TP ranks and/or parked on the host."""

    __slots__ = ("data", "shape", "dtype", "device", "numel", "partitioned", "on_cpu", "event", "requires_grad")

    def __init__(self, t: torch.Tensor, contiguous_buf=None, offset=0):
        self.shape, self.dtype, self.device, self.numel = t.shape, t.dtype, t.device, t.numel()
        self.requires_grad = t.requires_grad
        self.partitioned = PARTITION_ACTIVATIONS and _tp()[1] > 1 and t.is_floating_point()
        self.on_cpu = CPU_CHECKPOINT and t.is_cuda
        self.event = None
        src = t.detach()
        if self.partitioned:
            psz = get_partition_size(t)
            flat = src.contiguous().view(-1)
            start = get_partition_start(t)
            piece = flat[start:start + psz]
            if piece.numel() < psz:  # last rank: pad
                piece = torch.cat([piece, piece.new_zeros(psz - piece.numel())])
            if contiguous_buf is not None:
                dst = contiguous_buf[offset:offset + psz]
                dst.copy_(piece)
                src = dst
            else:
                src = piece.clone()
        if self.on_cpu:
            host = torch.empty(src.shape, dtype=src.dtype, device="cpu", pin_memory=True)
            s = _copy_side_stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                host.copy_(src, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(s)
            src.record_stream(s)
            self.event = ev
            src = host
        self.data = src

    def restore(self) -> torch.Tensor:
        x = self.data
        if self.on_cpu:
            if self.event is not None:
                self.event.synchronize()
            x = x.to(self.device, non_blocking=True)
        if self.partitioned:
            _, size, group = _tp()
            full = torch.empty(x.numel() * size, dtype=x.dtype, device=x.device)
            dist.all_gather_into_tensor(full, x.contiguous(), group=group)
            x = full[:self.numel].view(self.shape)
        x = x.detach()
        x.requires_grad_(self.requires_grad)
        return x


_contig_buffers = {}


def _contiguous_buffer(key, numel, dtype, device):
    buf = _contig_buffers.get(key)
    if buf is None or buf.numel() < numel or buf.dtype != dtype or buf.device != device:
        buf = torch.empty(numel, dtype=dtype, device=device)
        _contig_buffers[key] = buf
    return buf


# =====================================================================================================
# the checkpoint function
# =====================================================================================================
class CheckpointFunction(torch.autograd.Function):
    """Reentrant checkpoint: forward under ``no_grad``; backward re-runs ``run_function`` with the saved
    RNG state and back-propagates through the recomputed graph."""

    @staticmethod
    def forward(ctx, run_function, all_outputs, *args):
        if SYNCHRONIZE and torch.cuda.is_available():
            torch.cuda.synchronize()
        if PROFILE_TIME:
            _timers()("forward").start()
        ctx.run_function = run_function
        ctx.rng = _capture_rng()
        ctx.tensor_idx = [i for i, a in enumerate(args) if torch.is_tensor(a)]
        ctx.non_tensors = {i: a for i, a in enumerate(args) if not torch.is_tensor(a)}
        ctx.nargs = len(args)
        saved = []
        contiguous = None
        offset = 0
        if CONTIGUOUS_CHECKPOINTING and PARTITION_ACTIVATIONS:
            fl = [a for a in args if torch.is_tensor(a) and a.is_floating_point()]
            if fl:
                total = sum(get_partition_size(a) for a in fl)
                contiguous = _contiguous_buffer((id(run_function), fl[0].dtype), total, fl[0].dtype, fl[0].device)
        for i in ctx.tensor_idx:
            a = args[i]
            use_buf = contiguous is not None and a.is_floating_point() and a.dtype == contiguous.dtype
            saved.append(_Saved(a, contiguous if use_buf else None, offset))
            if use_buf:
                offset += get_partition_size(a)
        ctx.saved = saved
        with torch.no_grad():
            outputs = run_function(*args)
        if PROFILE_TIME:
            _timers()("forward").stop()
            _timers().log(["forward"])
        if SYNCHRONIZE and torch.cuda.is_available():
            torch.cuda.synchronize()
        if torch.is_tensor(outputs):
            all_outputs.append(outputs)
            return outputs
        all_outputs.extend(outputs)
        ctx.mark_non_differentiable(*[o for o in outputs if torch.is_tensor(o) and not o.is_floating_point()])
        return tuple(o for o in outputs if torch.is_tensor(o))

    @staticmethod
    def backward(ctx, *grads):
        if SYNCHRONIZE and torch.cuda.is_available():
            torch.cuda.synchronize()
        if PROFILE_TIME:
            _timers()("backward").start()
        if not torch.autograd._is_checkpoint_valid():
            raise RuntimeError("Checkpointing is not compatible with .grad(), please use .backward() if possible")
        args = [None] * ctx.nargs
        for i, v in ctx.non_tensors.items():
            args[i] = v
        for i, s in zip(ctx.tensor_idx, ctx.saved):
            args[i] = s.restore()
        ctx.saved = None
        now = _capture_rng()
        _restore_rng(ctx.rng)
        with torch.enable_grad():
            outputs = ctx.run_function(*args)
        _restore_rng(now)
        if torch.is_tensor(outputs):
            outputs = (outputs, )
        outs, gs = [], []
        tensor_outs = [o for o in outputs if torch.is_tensor(o)]
        for o, g in zip(tensor_outs, grads):
            if o.requires_grad and g is not None:
                outs.append(o)
                gs.append(g)
        if PROFILE_TIME:
            _timers()("backward").stop()
            _timers().log(["backward"])
        if outs:
            torch.autograd.backward(outs, gs)
        ret = [None, None]
        for i in range(ctx.nargs):
            a = args[i]
            ret.append(a.grad if torch.is_tensor(a) else None)
        if SYNCHRONIZE and torch.cuda.is_available():
            torch.cuda.synchronize()
        return tuple(ret)


class ReplayCheckpointFunction(CheckpointFunction):
    """:class:`CheckpointFunction` whose backward re-runs ``replay_function`` instead of ``run_function``: a replay that
    returns outputs of the same shapes whose backward is the same, but computes only what that backward reads."""

    @staticmethod
    def forward(ctx, run_function, replay_function, all_outputs, *args):
        outputs = CheckpointFunction.forward(ctx, run_function, all_outputs, *args)
        ctx.run_function = replay_function  # what backward re-runs
        return outputs

    @staticmethod
    def backward(ctx, *grads):
        return (None, ) + CheckpointFunction.backward(ctx, *grads)


def _timers():
    global timers
    if timers is None:
        timers = SynchronizedWallClockTimer()
    return timers


def checkpoint(function, *args, replay=None):
    """Checkpoint a model or part of the model (reference :980).  Returns what ``function`` returns.  ``replay``
    (optional) is what backward re-runs instead of ``function``: see :class:`ReplayCheckpointFunction`."""
    all_outputs = []
    if replay is None:
        out = CheckpointFunction.apply(function, all_outputs, *args)
    else:
        out = ReplayCheckpointFunction.apply(function, replay, all_outputs, *args)
    if len(all_outputs) == 1:
        return out if torch.is_tensor(out) else out[0]
    # re-attach non-tensor outputs in their original positions
    it = iter(out if isinstance(out, tuple) else (out, ))
    return tuple(next(it) if torch.is_tensor(o) else o for o in all_outputs)


def non_reentrant_checkpoint(function, *args):
    """Saved-tensor-hook based checkpoint (works with ``torch.autograd.grad`` and nested checkpoints).
    Offload / partition policies are applied to the *inputs* exactly like the reentrant variant."""
    from torch.utils.checkpoint import checkpoint as torch_checkpoint
    return torch_checkpoint(function, *args, use_reentrant=False, preserve_rng_state=True)


def partition_activations_in_checkpoint(partition_activation):
    global PARTITION_ACTIVATIONS
    PARTITION_ACTIVATIONS = partition_activation
    logger.info(f"**************Partition Activations {PARTITION_ACTIVATIONS}************")


def set_num_layers(nlayers):
    global num_layers
    num_layers = nlayers


def reset():
    """Drop cached contiguous buffers (call between iterations when shapes change)."""
    _contig_buffers.clear()


def _configure_using_config_file(config, mpu_=None):
    global num_layers, PARTITION_ACTIVATIONS, CONTIGUOUS_CHECKPOINTING, CPU_CHECKPOINT, SYNCHRONIZE, PROFILE_TIME
    from deepspeed_b200.runtime.config import DeepSpeedConfig
    c = DeepSpeedConfig(config, mpu=mpu_).activation_checkpointing_config
    PARTITION_ACTIVATIONS = c.partition_activations
    CONTIGUOUS_CHECKPOINTING = c.contiguous_memory_optimization
    num_layers = c.number_checkpoints
    CPU_CHECKPOINT = c.cpu_checkpointing
    SYNCHRONIZE = c.synchronize_checkpoint_boundary
    PROFILE_TIME = c.profile


def configure(mpu_, deepspeed_config=None, partition_activations=None, contiguous_checkpointing=None,
              num_checkpoints=None, checkpoint_in_cpu=None, synchronize=None, profile=None):
    """Configure DeepSpeed activation checkpointing (reference :1029)."""
    global mpu, num_layers, deepspeed_checkpointing_enabled, PARTITION_ACTIVATIONS, CONTIGUOUS_CHECKPOINTING, \
        CPU_CHECKPOINT, SYNCHRONIZE, PROFILE_TIME, _configured, mp_size, mp_rank, mp_group
    deepspeed_checkpointing_enabled = True
    mpu = mpu_
    mp_size = mp_rank = mp_group = None
    if deepspeed_config is not None:
        _configure_using_config_file(deepspeed_config, mpu_)
    if partition_activations is not None:
        PARTITION_ACTIVATIONS = partition_activations
    if contiguous_checkpointing is not None:
        CONTIGUOUS_CHECKPOINTING = contiguous_checkpointing
    if num_checkpoints is not None:
        num_layers = num_checkpoints
    if checkpoint_in_cpu is not None:
        CPU_CHECKPOINT = checkpoint_in_cpu
    if synchronize is not None:
        SYNCHRONIZE = synchronize
    if profile is not None:
        PROFILE_TIME = profile
    if CONTIGUOUS_CHECKPOINTING:
        assert PARTITION_ACTIVATIONS, "Contiguous Checkpointing is only available with partitioned activations. " \
            "Set partitioned activations to true in deepspeed config"
        assert num_layers is not None, "Must specify the number of layers with contiguous memory checkpointing"
    _configured = True


def is_configured():
    return _configured


# =====================================================================================================
# functional helpers under the reference's names (``checkpointing.py:143-460``); the checkpoint function above does
# the same work through ``_Saved`` objects
# =====================================================================================================
def detach_variable(inputs, device=None):
    """Detached copies (optionally moved) that keep ``requires_grad``; non-tensors pass through."""
    if not isinstance(inputs, tuple):
        raise RuntimeError(f"Only tuple of tensors is supported. Got Unsupported input type: {type(inputs).__name__}")
    out = []
    for inp in inputs:
        if not torch.is_tensor(inp):
            out.append(inp)
            continue
        x = inp.detach() if device is None else inp.to(device=device).detach()
        x.requires_grad = inp.requires_grad
        out.append(x)
    return tuple(out)


def extract_tensors(all_objects):
    """Split a tuple / list into (tensors, non-tensors, flags); ``merge_tensors`` is the inverse."""
    flags = [torch.is_tensor(v) for v in all_objects]
    tensors = [v for v, f in zip(all_objects, flags) if f]
    others = [v for v, f in zip(all_objects, flags) if not f]
    if isinstance(all_objects, tuple):
        return tuple(tensors), tuple(others), tuple(flags)
    return tensors, others, flags


def merge_tensors(tensor_objects, non_tensor_objects, tensor_flags):
    t, o = iter(tensor_objects), iter(non_tensor_objects)
    return tuple(next(t) if f else next(o) for f in tensor_flags)


def is_activation_to_checkpoint(item):
    """Only floating-point tensors large enough to split across the tensor-parallel group are partitioned."""
    _, size, _ = _tp()
    return torch.is_tensor(item) and item.is_floating_point() and item.numel() >= size


def partition_activations(args, cpu_checkpoint=False, contiguous_checkpoint=False):
    """This rank's slice of every checkpointable tensor in ``args`` (others unchanged)."""
    out = []
    for i, item in enumerate(args):
        if not is_activation_to_checkpoint(item):
            out.append(item)
            continue
        psz, start = get_partition_size(item), get_partition_start(item)
        flat = item.detach().contiguous().view(-1)
        piece = flat[start:start + psz]
        if piece.numel() < psz:
            piece = torch.cat([piece, piece.new_zeros(psz - piece.numel())])
        if contiguous_checkpoint:
            buf = _contiguous_buffer(("partition", i), psz, item.dtype, torch.device("cpu") if cpu_checkpoint else item.device)
            buf[:psz].copy_(piece)
            piece = buf[:psz]
        elif cpu_checkpoint:
            piece = piece.to("cpu")
        else:
            piece = piece.clone()
        out.append(piece)
    return out


def get_partitioned_activations_for_backward(args, inputs, contiguous_checkpoint=False):
    """Interleave each partition with the shape tensor needed to rebuild it: [part0, size0, part1, size1, ...]."""
    new_args = []
    for i, (arg, inp) in enumerate(zip(args, inputs)):
        if not is_activation_to_checkpoint(inp):
            new_args.append(arg)
            new_args.append(None)
            continue
        new_args.append(arg)
        new_args.append(torch.tensor(inp.size(), dtype=torch.int64))
    return new_args


def get_cpu_activations_for_backward(args, inputs):
    new_args = []
    for arg, inp in zip(args, inputs):
        new_args.append(arg if not is_activation_to_checkpoint(inp) else arg.to("cpu"))
    return new_args


def gather_partitioned_activations(tensors, device=None):
    """Inverse of :func:`get_partitioned_activations_for_backward`: all-gather every (partition, size) pair."""
    assert len(tensors) % 2 == 0, f"Expected even count of tensors, instead got {len(tensors)}"
    _, size, group = _tp()
    out = []
    for part, shape in zip(tensors[0::2], tensors[1::2]):
        if shape is None or not torch.is_tensor(part):
            out.append(part)
            continue
        numel = int(torch.as_tensor(shape).prod())
        x = part.to(device) if device is not None else part
        if size == 1:
            out.append(x[:numel].view(*[int(s) for s in shape]))
            continue
        full = torch.empty(x.numel() * size, dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(full, x.contiguous(), group=group)
        out.append(full[:numel].view(*[int(s) for s in shape]))
    return out
