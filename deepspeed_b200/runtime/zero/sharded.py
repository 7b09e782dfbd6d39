"""ZeRO stages 0-3 as ONE sharded-state engine over a static unit plan.

Capability parity with the reference ``runtime/zero/stage_1_and_2.py`` (P5), ``stage3.py`` (P6),
``partition_parameters.py`` (P7), ``partitioned_param_coordinator.py`` (P8),
``parameter_offload.py`` (P9), ``bf16_optimizer.py`` (P13) and ``fp16/fused_optimizer.py`` (P14),
but a different architecture (see SURVEY.md 7.1):

* **Static plan** (``units.py``): unit-flat buffers sharded contiguously across the DP group, so
  all-gather / reduce-scatter are zero-copy on both ends.
* **Rank-local arenas**: one flat tensor each for the low-precision shard, the fp32 master, every
  optimizer state and (when needed) the accumulated gradient shard.  The optimizer step is a few
  fused-kernel launches over arena segments, not a Python loop over parameters.
* **Stage is a parameter, not a class**: stage 0 = no sharding (all-reduce), stage 1/2 = sharded
  optimizer state + reduce-scatter'd gradients with persistently gathered parameters, stage 3 =
  transient parameters gathered per unit with prefetch.
* **Streams**: gathers run on ``ag_stream``, reductions (+ fused accumulate / Adam) on
  ``rs_stream``; buffers come from fixed rotating pools so no allocator/stream hazards exist.
* **Collective back-ends**: NCCL through ``deepspeed_b200.comm`` (baseline / multi-node / host),
  or the in-kernel NVLink peer-memory path from ``deepspeed_b200.comm.symm`` when the symmetric
  arena is available (``b200_fused_collectives``).
* **No host syncs in the step** for bf16: grad-norm, clip coefficient and overflow flag live on
  the device and are consumed by the fused optimizer kernel directly.
"""
import math
import weakref
from typing import Dict, List, Optional

import torch
from torch import nn

from deepspeed_b200 import comm as dist
from deepspeed_b200.accelerator import get_accelerator
from deepspeed_b200.ops.kernels import flat_ops
from deepspeed_b200.runtime.base_optimizer import ZeROOptimizer
from deepspeed_b200.runtime.fp16.loss_scaler import CreateLossScaler
from deepspeed_b200.runtime.zero.flat_optimizers import (FlatOptimizer, TorchOptimizerAdapter, build_flat_optimizer)
from deepspeed_b200.runtime.zero.units import (Segment, Unit, arena_segments, build_units, param_fragments)
from deepspeed_b200.utils.logging import logger, log_dist
from deepspeed_b200.utils.nvtx import instrument_w_nvtx

NOT_GATHERED, INFLIGHT, GATHERED = 0, 1, 2


class _InnerOptimizerView:
    """Read-only face of the flat optimizer in the shape user code expects from ``engine.optimizer.optimizer``."""

    def __init__(self, zo):
        self._zo = zo

    @property
    def param_groups(self):
        return self._zo.param_groups

    @property
    def state(self):
        zo = self._zo
        st = {k: v for k, v in (zo.flat_opt.state_tensors() or {}).items() if torch.is_tensor(v)}
        st["step"] = max(zo.group_steps) if zo.group_steps else 0
        key = zo.master if torch.is_tensor(zo.master) else 0
        return {key: st}

    def state_dict(self):
        groups = [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]
        return {"state": {0: next(iter(self.state.values()))}, "param_groups": groups}


def tag_reference_class(opt):
    """Give an engine-built optimizer the reference's class for its stage so ``isinstance(engine.optimizer,
    DeepSpeedZeroOptimizer_Stage3)`` style checks in user code keep working (the subclasses only add the reference's
    constructor signature)."""
    if opt.stage == 3:
        from deepspeed_b200.runtime.zero.stage3 import DeepSpeedZeroOptimizer_Stage3 as cls
    elif opt.stage in (1, 2):
        from deepspeed_b200.runtime.zero.stage_1_and_2 import DeepSpeedZeroOptimizer as cls
    elif opt.model_dtype == torch.float16:
        from deepspeed_b200.runtime.fp16.fused_optimizer import FP16_Optimizer as cls
    elif opt.model_dtype == torch.bfloat16:
        from deepspeed_b200.runtime.bf16_optimizer import BF16_Optimizer as cls
    else:
        return _tag_basic_class(opt)
    if type(opt) is ZeroShardedOptimizer:
        opt.__class__ = cls
    return opt


_BASIC_TAGGED = {}


def _tag_basic_class(opt):
    """Stage 0 + fp32: the reference wraps nothing and hands the *basic* optimizer back from ``initialize`` (engine.py
    ``_configure_optimizer``: ``FusedAdam`` for a config-named Adam, the client's own object / class otherwise), and user
    code checks ``isinstance(opt, FusedAdam)`` / ``opt == client_optimizer``.  The flat optimizer here also is that
    class: a (cached) subclass of both, with this implementation first in the MRO."""
    client = getattr(opt, "client_optimizer", None)
    if client is not None:
        basic = type(client)
    else:
        name = (getattr(opt, "optimizer_name", None) or "").lower()
        if name in ("adam", "adamw"):
            from deepspeed_b200.ops.adam import FusedAdam as basic
        elif name == "lamb":
            from deepspeed_b200.ops.lamb import FusedLamb as basic
        elif name == "lion":
            from deepspeed_b200.ops.lion import FusedLion as basic
        elif name == "adagrad":
            basic = torch.optim.Adagrad
        elif name == "sgd":
            basic = torch.optim.SGD
        else:
            return opt
    base = type(opt)
    if not isinstance(basic, type) or issubclass(base, basic) or type(opt) is not ZeroShardedOptimizer:
        return opt
    key = (base, basic)
    if key not in _BASIC_TAGGED:
        def __eq__(self, other):
            return other is self or (other is not None and other is getattr(self, "client_optimizer", None))

        try:
            _BASIC_TAGGED[key] = type(basic.__name__, (base, basic), {"__eq__": __eq__, "__hash__": object.__hash__,
                                                                      "__module__": basic.__module__})
        except TypeError:  # incompatible layouts (a C-extension optimizer class)
            _BASIC_TAGGED[key] = None
    cls = _BASIC_TAGGED[key]
    if cls is not None:
        try:
            opt.__class__ = cls
        except TypeError:
            pass
    return opt


def _param_status():
    from deepspeed_b200.runtime.zero.partition_parameters import ZeroParamStatus
    return ZeroParamStatus


class _Slot:
    """One buffer of a rotating pool plus the event that marks it reusable."""

    def __init__(self, buf):
        self.buf = buf
        self.free_event = None  # recorded on the stream that last read/wrote it
        self.owner = None


class _UnitRT:
    """Runtime (mutable) companion of a plan :class:`Unit`."""

    def __init__(self, unit: Unit):
        self.u = unit
        self.state = NOT_GATHERED
        self.full: Optional[torch.Tensor] = None
        self.slot: Optional[_Slot] = None
        self.gather_event = None
        self.grad_slot: Optional[_Slot] = None
        self.grad_full: Optional[torch.Tensor] = None
        self.pending = 0
        self.n_trainable = 0
        self.reduced_this_micro = False
        self.dense_grads = False  # set by model integrations that write every gradient view
        self.temp_refs = 0  # GatheredParameters / external users holding the unit
        self.home = None  # buffer used by this iteration's forward gather (backward MUST reuse it)
        self.borrow_home = None  # ... and by the forward gather for a module sharing the unit's weight
        self.running = 0  # forward passes of the unit's module currently executing (re-entrancy counter)
        self.unsynced = None  # local gradient parked by backward passes under engine.no_sync()
        self.fwd_calls = 0  # grad-enabled forward invocations of the module since the last backward finished
        self.bwd_calls = 0  # ... and how many of them have been back-propagated
        self.consumed = False  # a module hook actually used the gathered copy (vs. a speculative prefetch)
        self.skip_bwd_fetch = False  # module's backward does not read its weights (embedding, fused LM head)
        self.own_grad_slot: Optional[_Slot] = None  # units with borrowers: a gradient buffer outside the pool


class ZeroShardedOptimizer(ZeROOptimizer):
    """Sharded model-state manager + optimizer.  See module docstring."""

    def __init__(self,
                 module: nn.Module,
                 stage: int,
                 *,
                 client_optimizer=None,
                 optimizer_name: Optional[str] = None,
                 optimizer_params: Optional[dict] = None,
                 param_groups: Optional[List[dict]] = None,
                 zero_config=None,
                 dp_group=None,
                 model_dtype=torch.bfloat16,
                 grad_accum_dtype=None,
                 gradient_accumulation_steps: int = 1,
                 gradient_clipping: float = 0.0,
                 loss_scale_config: Optional[dict] = None,
                 communication_data_type=None,
                 prescale_gradients=False,
                 gradient_predivide_factor=1.0,
                 device=None,
                 mpu=None,
                 broadcast_init=True,
                 timers=None,
                 param_filter=None,
                 name="dense",
                 aio_config=None,
                 replica_group=None):
        self.aio_config = aio_config
        self.replica_group = replica_group  # MiCS: model-state replicas across shard groups
        from deepspeed_b200.runtime.zero.config import DeepSpeedZeroConfig
        self.param_filter = param_filter
        self.name = name
        self.module = module
        self.stage = int(stage)
        self.zc = zero_config or DeepSpeedZeroConfig(stage=self.stage)
        self.dp_group = dp_group
        self.dp_world = dist.get_world_size(dp_group)
        self.dp_rank = dist.get_rank(dp_group)
        self.shard_world = self.dp_world if self.stage >= 1 else 1
        self.shard_rank = self.dp_rank if self.stage >= 1 else 0
        self.accel = get_accelerator()
        self.device = torch.device(device if device is not None else self.accel.current_device_name())
        self.on_cuda = self.device.type == "cuda"
        self.model_dtype = model_dtype
        self.master_dtype = torch.float32
        self.gas = max(1, int(gradient_accumulation_steps))
        self.clip = float(gradient_clipping or 0.0)
        self.grad_accum_dtype = grad_accum_dtype or model_dtype
        self.comm_dtype = communication_data_type or model_dtype
        self.prescale = prescale_gradients
        self.predivide = float(gradient_predivide_factor)
        self.mpu = mpu
        self.timers = timers
        self.micro_step = 0
        self.global_step = 0
        self.overflow = False
        self.skipped_steps = 0
        self._global_grad_norm = None
        self.custom_loss_scaler = False
        self.external_loss_scale = None

        # ---- offload tiers -------------------------------------------------------------
        oo = self.zc.offload_optimizer
        op = self.zc.offload_param
        self.offload_optimizer = bool(oo and str(getattr(oo.device, "value", oo.device)) != "none")
        self.offload_param = bool(op and str(getattr(op.device, "value", op.device)) != "none") and self.stage == 3
        self.offload_param_nvme = self.offload_param and str(getattr(op.device, "value", op.device)) == "nvme"
        self.offload_pin = bool(oo.pin_memory) if oo else False
        self.offload_ratio = float(oo.ratio) if oo else 1.0
        self.grad_allreduce_enabled = lambda: True
        from deepspeed_b200.runtime.zero.partitioned_param_profiler import PartitionedParameterProfiler
        self.param_profiler = PartitionedParameterProfiler() if PartitionedParameterProfiler.enabled() else None
        self.replica_world = dist.get_world_size(replica_group) if replica_group is not None else 1
        # ---- ZeRO++ -----------------------------------------------------------------------
        self.qwz = bool(getattr(self.zc, "zero_quantized_weights", False)) and self.stage == 3 and self.shard_world > 1
        self.qgz = bool(getattr(self.zc, "zero_quantized_gradients", False)) and self.shard_world > 1
        self.loco = getattr(self.zc, "zeropp_loco_param", None) if self.qgz else None
        hpz = int(getattr(self.zc, "zero_hpz_partition_size", 1) or 1)
        self.hpz = hpz if (hpz > 1 and self.stage == 3 and self.shard_world > hpz and self.shard_world % hpz == 0) else 1
        self.hpz_group = None
        if self.hpz > 1:
            from deepspeed_b200.utils import groups as _g
            if not _g._zero_param_parallel_is_initialized():
                _g._create_zero_param_parallel_group(self.hpz)
            self.hpz_group = _g._get_zero_param_intra_parallel_group()
        self.offload_nvme = self.offload_optimizer and str(getattr(oo.device, "value", oo.device)) == "nvme"
        self.state_swapper = None

        # ---- loss scaling ----------------------------------------------------------------
        lsc = loss_scale_config or {}
        self.loss_scaler = CreateLossScaler(dtype=model_dtype,
                                            static_loss_scale=lsc.get("static_loss_scale", 1.0),
                                            dynamic_scaling=lsc.get("dynamic", False),
                                            dynamic_loss_args=lsc.get("dynamic_args"))
        self.dynamic_loss_scale = self.loss_scaler.dynamic

        # ---- param groups ------------------------------------------------------------------
        self.client_optimizer = client_optimizer
        self.optimizer_name = optimizer_name
        self.flat_opt: FlatOptimizer = build_flat_optimizer(optimizer_name, optimizer_params, client_optimizer)
        self.param_groups = self._make_param_groups(client_optimizer, param_groups, optimizer_params)
        p2g = {}
        for gi, g in enumerate(self.param_groups):
            for p in g["params"]:
                p2g[id(p)] = gi
        if isinstance(self.flat_opt, TorchOptimizerAdapter):
            # the client optimizer reads ITS group dicts at step time: expose those very objects so LR
            # schedulers (which mutate ``optimizer.param_groups[i]["lr"]``) reach it
            self.param_groups = client_optimizer.param_groups
        for p in module.parameters():
            if id(p) not in p2g and (param_filter is None or param_filter(p)):
                p2g[id(p)] = -1  # frozen / unmanaged: sharded but never stepped
        self.group_steps = [0 for _ in self.param_groups]

        # ---- plan ------------------------------------------------------------------------------
        thresh = int(self.zc.param_persistence_threshold) if self.stage == 3 else 0
        self.units: List[Unit] = build_units(module, self.shard_world, p2g, persistence_threshold=0,
                                             param_filter=param_filter)
        assert self.units, f"ZeroShardedOptimizer[{name}]: no parameters to manage"
        self.rts: List[_UnitRT] = [_UnitRT(u) for u in self.units]
        self.unit_of_param: Dict[int, _UnitRT] = {}
        self.slot_of_param = {}
        for rt in self.rts:
            for s in rt.u.slots:
                self.unit_of_param[id(s.param)] = rt
                self.slot_of_param[id(s.param)] = s
            rt.n_trainable = sum(1 for s in rt.u.slots if s.param.requires_grad)
            rt.layout_sig = (rt.u.full_numel, tuple((s.offset, s.numel) for s in rt.u.slots))
            # whole-unit persistence (small units stay gathered, like the reference's
            # param_persistence_threshold but at unit granularity)
            rt.u.persistent = self.stage < 3 or self.shard_world == 1 or rt.u.raw_numel <= thresh
        self.arena_numel = sum(u.shard_numel for u in self.units)
        self.segments: List[Segment] = arena_segments(self.units, self.shard_rank)
        # pieces = segments split at unit boundaries: (unit_rt, group, start, end)
        self.pieces = []
        for rt in self.rts:
            a, b = rt.u.arena_offset, rt.u.arena_offset + rt.u.shard_numel
            for seg in self.segments:
                s0, e0 = max(seg.start, a), min(seg.end, b)
                if s0 < e0:
                    self.pieces.append((rt, seg.group, s0, e0))
        self.max_full = max(u.full_numel for u in self.units)

        # ---- streams ---------------------------------------------------------------------------
        overlap = bool(self.zc.overlap_comm) and self.on_cuda
        self.ag_stream = torch.cuda.Stream() if overlap else None
        self.rs_stream = torch.cuda.Stream() if overlap else None
        self.prefetch_depth = max(0, int(self.zc.b200_unit_prefetch))
        # host-offload tier: reduced gradient shards leave the GPU on ``d2h_stream`` (pinned cudaMemcpyAsync, nothing on
        # the compute stream waits for them) and updated parameters come back on ``h2d_stream`` while the CPU optimizer is
        # already working on the next unit (reference stage3.py:1466-1527 async D2H of reduced shards,
        # swap_tensor/pipelined_optimizer_swapper.py:52)
        if self.offload_optimizer:
            from deepspeed_b200.ops.adam import cpu_adam as _cpu_adam
            n_thr = _cpu_adam.configure_threads()
            log_dist(f"host optimizer: {n_thr} threads per rank", ranks=[0])
        off_cuda = self.offload_optimizer and self.on_cuda
        self.d2h_stream = torch.cuda.Stream() if off_cuda else None
        self.h2d_stream = torch.cuda.Stream() if off_cuda else None
        self._d2h_slots, self._d2h_i, self._d2h_adds, self._grad_stage = None, 0, [], None
        self._h2d_slots, self._h2d_i = None, 0

        # ---- fusion policy ------------------------------------------------------------------------
        self._fib_request = self.zc.b200_fused_optimizer_in_backward
        self._forced_boundary = None
        self._accum = 0  # micro steps accumulated since the last optimizer step
        self.fused_in_backward = self._fusion_policy()
        # host tier analogue of the fused-in-backward step: each unit's CPU optimizer step starts as soon as its reduced
        # gradient shard has landed in pinned memory, on a worker thread, while backward is still running on the GPU
        self.host_step_in_backward = self._host_overlap_policy()
        self._host_worker = None

        self._allocate(broadcast_init)
        self._register_hooks()
        self.stats = flat_ops.GradStats(self.device if not self.offload_optimizer else "cpu")
        self._dev_stats = flat_ops.GradStats(self.device) if self.offload_optimizer else self.stats
        self._trace: List[int] = []
        self._borrow_pos = set()  # positions in _trace that are borrows (fetches for a module sharing the unit's weight)
        self._trace_done = False
        self._order_pos: Dict[int, int] = {}
        self._in_backward = False
        self._symm = None
        self._maybe_enable_symm()
        self._verify_left = int(getattr(self.zc, "b200_verify_collectives", 0) or 0) if self._symm is not None else 0
        from deepspeed_b200.runtime.zero import _stage_helpers
        if _stage_helpers.pg_correctness_test and self._symm is not None:
            self._verify_left = 1 << 60  # the reference's global switch: verify for the whole run
        self.verify_report = {"all_gather": 0, "reduce_scatter": 0, "max_rel_err": 0.0}
        log_dist(
            f"ZeroShardedOptimizer: stage={self.stage} units={len(self.units)} arena={self.arena_numel:,} elems/rank "
            f"shard_world={self.shard_world} fused_in_backward={self.fused_in_backward} "
            f"offload_opt={self.offload_optimizer} host_step_in_backward={self.host_step_in_backward} "
            f"symm={'on' if self._symm else 'off'}",
            ranks=[0])

    # =========================================================================================
    # construction
    # =========================================================================================
    def _fusion_policy(self) -> bool:
        """May the optimizer step run unit by unit inside backward (no gradient arena at all)?  Only when nothing
        needs the *whole* gradient first: no clipping, no accumulation, no loss scaling of any kind (fp16 always
        unscales + checks overflow, reference ``stage3.py:2086-2130``), no offload, a flat fused optimizer."""
        scaled = (self.model_dtype == torch.float16 or self.dynamic_loss_scale
                  or float(self.loss_scaler.cur_scale) != 1.0)
        can_fuse = (self.flat_opt.fused and not getattr(self.flat_opt, "per_tensor", False) and self.clip == 0.0
                    and self.gas == 1 and not scaled and not self.offload_optimizer
                    and not getattr(self, "_no_fuse_reason", None))
        fib = self._fib_request
        return bool(can_fuse if fib is None else (fib and can_fuse))

    def _host_overlap_policy(self) -> bool:
        """Same preconditions as :meth:`_fusion_policy` (nothing may need the whole gradient first), for the CPU tier."""
        scaled = (self.model_dtype == torch.float16 or self.dynamic_loss_scale
                  or float(self.loss_scaler.cur_scale) != 1.0)
        ok = (self.offload_optimizer and not self.offload_nvme and self.d2h_stream is not None and self.flat_opt.fused
              and not getattr(self.flat_opt, "per_tensor", False) and self.clip == 0.0 and self.gas == 1 and not scaled
              and not self.offload_param and not getattr(self, "_no_fuse_reason", None))
        want = self._fib_request
        return bool(ok if want is None else (want and ok))

    def disable_fused_in_backward(self, reason: str):
        """Fall back to the two-phase step (reduce + accumulate, then one fused step); allocates the gradient arena
        if the fused path had elided it.  Used when something discovered after construction needs whole gradients
        (gradient accumulation turned on, tied weights across pipeline stages, ...)."""
        self._no_fuse_reason = reason
        if getattr(self, "host_step_in_backward", False):
            self._join_host_worker()
            self.host_step_in_backward = False
            log_dist(f"ZeroShardedOptimizer[{self.name}]: host step inside backward disabled ({reason})", ranks=[0])
        if not self.fused_in_backward:
            return
        self.fused_in_backward = False
        self._ensure_grad_arena()
        log_dist(f"ZeroShardedOptimizer[{self.name}]: fused-in-backward step disabled ({reason})", ranks=[0])

    def _apply_pending_defuse(self):
        reason = getattr(self, "_defuse_after_step", None)
        if reason and (self.fused_in_backward or self.host_step_in_backward):
            self.disable_fused_in_backward(reason)

    def _ensure_grad_arena(self):
        if self.grad_arena is None:
            st_dev = "cpu" if self.offload_optimizer else self.device
            gdt = torch.float32 if (self.offload_optimizer or not self.flat_opt.fused) else self.grad_accum_dtype
            self.grad_arena = self._empty(self.arena_numel, gdt, st_dev, pin=True)
            self.grad_arena.zero_()

    def set_gradient_accumulation_steps(self, gas: int):
        """Change GAS after construction (``engine.set_train_batch_size``): re-evaluates the fusion policy."""
        self.gas = max(1, int(gas))
        if self.gas > 1:
            self.disable_fused_in_backward(f"gradient_accumulation_steps={self.gas}")

    def _make_param_groups(self, client_optimizer, param_groups, defaults):
        keep = self.param_filter or (lambda p: True)
        if client_optimizer is not None:
            groups = []
            for g in client_optimizer.param_groups:
                ng = {k: v for k, v in g.items() if k != "params"}
                ng["params"] = [p for p in g["params"] if keep(p)]
                groups.append(ng)
            return groups
        if param_groups is None:
            param_groups = [{"params": [p for p in self.module.parameters() if p.requires_grad and keep(p)]}]
        elif len(param_groups) and not isinstance(param_groups[0], dict):
            param_groups = [{"params": list(param_groups)}]
        out = []
        base = dict(self.flat_opt.defaults)
        for g in param_groups:
            ng = dict(base)
            ng.update({k: v for k, v in g.items() if k != "params"})
            ng["params"] = [p for p in g["params"] if p.requires_grad and keep(p)]
            ng.setdefault("lr", base.get("lr", 1e-3))
            out.append(ng)
        return out

    def _empty(self, n, dtype, device=None, pin=False):
        dev = device or self.device
        if pin and torch.device(dev).type == "cpu" and torch.cuda.is_available():
            # page-locked from the start: `.pin_memory()` on a pageable tensor would hold BOTH copies for a moment, which at
            # Llama-70B scale is an extra ~70 GB of host memory per arena and rank
            # (and not through torch's pinned allocator for big arenas: it rounds sizes up to a power of two)
            from deepspeed_b200.ops.pinned import pinned_empty
            return pinned_empty(n, dtype)
        return torch.empty(n, dtype=dtype, device=dev)

    def _allocate(self, broadcast_init):
        dev = self.device
        lp = self.model_dtype
        S3 = self.stage == 3 and self.shard_world > 1
        self.transient = S3
        # ---- low-precision storage ------------------------------------------------------------
        if S3:
            if self.offload_param_nvme:
                # ZeRO-Infinity parameter tier: this rank's low-precision shards live in a swap file; a unit's shard passes
                # through a pinned window on its way to the all-gather and on its way back from the optimizer (reference
                # swap_tensor/partitioned_param_swapper.py:36 AsyncPartitionedParameterSwapper)
                import os as _os
                from deepspeed_b200.runtime.swap_tensor.aio_config import make_handle
                from deepspeed_b200.runtime.swap_tensor.optimizer_utils import SwappedFlatState
                opc = self.zc.offload_param
                folder = _os.path.join(str(opc.nvme_path or "/tmp"), "zero_stage_3", f"{str(lp).split('.')[-1]}params",
                                       f"rank{dist.get_rank()}")
                self.lp_arena = SwappedFlatState("lp_params", self.arena_numel, lp, folder, make_handle(self.aio_config or {}),
                                                 max(u.shard_numel for u in self.units), max(3, int(opc.buffer_count or 3)))
            elif self.offload_param:
                self.lp_arena = self._empty(self.arena_numel, lp, "cpu", pin=True)
            else:
                self.lp_arena = self._symm_or_empty(self.arena_numel, lp)  # peers gather straight from it
            n_slots = 2 + self.prefetch_depth
            self.param_pool = [_Slot(self._symm_or_empty(self.max_full, lp)) for _ in range(n_slots)]
            self.full_arena = None
        else:
            total_full = sum(u.full_numel for u in self.units)
            self.full_arena = self._symm_or_empty(total_full, lp)
            self.full_arena.zero_()
            self.param_pool = []
            self.lp_arena = None  # shards are views of full_arena
        self.grad_pool = [_Slot(self._symm_or_empty(self.max_full, self.comm_dtype)) for _ in range(2)]
        for rt in self.rts:
            if rt.u.borrowers:
                # a tied LM head writes its dW into the shared weight's gradient view in forward and the embedding's
                # backward adds to it at the very end: held through the whole backward, the view gets a buffer of its
                # own rather than one of the two the other units take turns on
                rt.own_grad_slot = _Slot(self._symm_or_empty(rt.u.full_numel, self.comm_dtype))
        self._rs_tmp = [self._empty(max(u.shard_numel for u in self.units), self.comm_dtype) for _ in range(2)] \
            if self.shard_world > 1 else []

        # ---- materialise parameter data ---------------------------------------------------------
        foff = 0
        src_rank = dist.get_global_rank(self.dp_group, 0) if self.dp_group is not None else 0
        for rt in self.rts:
            u = rt.u
            if S3:
                tmp = torch.zeros(u.full_numel, dtype=lp, device=dev)
                self._pack_unit(u, tmp)
                if broadcast_init and self.dp_world > 1:
                    dist.broadcast(tmp, src=src_rank, group=self.dp_group)
                if broadcast_init and self.replica_world > 1:  # MiCS: replicas start from replica 0's values
                    dist.broadcast(tmp, src=dist.get_global_rank(self.replica_group, 0), group=self.replica_group)
                lo, hi = u.shard_range(self.shard_rank)
                self._lp_shard(u).copy_(tmp[lo:hi])
                if u.persistent:
                    rt.full = tmp
                    rt.state = GATHERED
                    self._point_params(rt, tmp)
                else:
                    self._detach_params(rt)
                    del tmp
            else:
                full = self.full_arena[foff:foff + u.full_numel]
                self._pack_unit(u, full)
                rt.full = full
                rt.state = GATHERED
                self._point_params(rt, full)
                foff += u.full_numel
        if not S3 and broadcast_init and self.dp_world > 1:
            dist.broadcast(self.full_arena, src=src_rank, group=self.dp_group)
        if not S3 and broadcast_init and self.replica_world > 1:
            dist.broadcast(self.full_arena, src=dist.get_global_rank(self.replica_group, 0), group=self.replica_group)

        # ---- master + optimizer state ---------------------------------------------------------------
        st_dev = "cpu" if self.offload_optimizer else dev
        nvme = self.offload_nvme and not isinstance(self.flat_opt, TorchOptimizerAdapter)
        if nvme:
            # NVMe tier: fp32 master weights and optimizer moments live in per-rank swap files and stream through pinned
            # windows (reference swap_tensor/optimizer_utils.py:117, partitioned_optimizer_swapper.py:27)
            from deepspeed_b200.runtime.swap_tensor import FlatStateSwapper
            oo = self.zc.offload_optimizer
            self.state_swapper = FlatStateSwapper(oo, self.aio_config or {}, str(oo.nvme_path or "/tmp"),
                                                  dist.get_rank())
        if lp == torch.float32 and not self.offload_optimizer:
            self.master = None  # fp32 training: the lp shard *is* the master
        else:
            if nvme and getattr(self.zc.offload_optimizer, "b200_swap_master", True) and self.master_dtype == torch.float32:
                self.master = self.state_swapper.wrap_master(self.arena_numel, self.master_dtype)
            else:
                self.master = self._empty(self.arena_numel, self.master_dtype, st_dev, pin=True)
            for rt in self.rts:
                a = rt.u.arena_offset
                self.master[a:a + rt.u.shard_numel].copy_(self._lp_shard(rt.u))
        if nvme:
            self.state_swapper.wrap(self.flat_opt, self.arena_numel)
        else:
            self.flat_opt.init_state(self.arena_numel, st_dev, torch.float32, pin=True)
        if isinstance(self.flat_opt, TorchOptimizerAdapter):
            self.flat_opt.bind([(g, s0, e0, self._piece_master(rt, s0, e0)) for (rt, g, s0, e0) in self.pieces],
                               len(self.param_groups))
        # accumulated gradient shard: only allocated when the fused-in-backward path is off
        self.grad_arena = None
        if not self.fused_in_backward:
            self._ensure_grad_arena()
        self._lp_stage = self._empty(max(u.shard_numel for u in self.units), lp, "cpu", pin=True) \
            if self.offload_optimizer else None

    def _symm_or_empty(self, n, dtype):
        """Allocate from the symmetric (peer-mapped) arena when available, else a plain tensor."""
        from deepspeed_b200.comm import symm
        t = symm.maybe_alloc(n, dtype, self.device, self.dp_group) if (self.on_cuda and self.shard_world > 1
                                                                       and self._want_symm()) else None
        return t if t is not None else torch.empty(n, dtype=dtype, device=self.device)

    def _want_symm(self):
        f = self.zc.b200_fused_collectives
        if f is False or self.replica_world > 1 or self.qwz or self.qgz or self.hpz > 1:
            return False
        from deepspeed_b200.comm import symm
        return symm.is_supported(self.dp_group, explicit=bool(f))

    def _maybe_enable_symm(self):
        if not (self.on_cuda and self.shard_world > 1 and self._want_symm()):
            return
        from deepspeed_b200.comm import symm
        self._symm = symm.get_context(self.dp_group)

    def _piece_master(self, rt, s0, e0):
        """fp32 (or native-precision) master slice for arena range [s0, e0) inside unit ``rt``."""
        if self.master is not None:
            return self.master[s0:e0]
        a = rt.u.arena_offset
        return self._lp_shard(rt.u)[s0 - a:e0 - a]

    def _piece_lp(self, rt, s0, e0):
        a = rt.u.arena_offset
        return self._lp_shard(rt.u)[s0 - a:e0 - a]

    def _lp_shard(self, u: Unit) -> torch.Tensor:
        if self.lp_arena is not None:
            return self.lp_arena[u.arena_offset:u.arena_offset + u.shard_numel]
        rt = self.rts[u.index]
        lo, hi = u.shard_range(self.shard_rank)
        return rt.full[lo:hi]

    @torch.no_grad()
    def _pack_unit(self, u: Unit, flat: torch.Tensor):
        """Copy current parameter values into the unit's flat layout."""
        for s in u.slots:
            p = s.param
            src = getattr(p, "ds_full_data", None)
            if src is None:
                src = p.data
            if src.numel() != s.numel:
                from deepspeed_b200.runtime.zero.partition_parameters import materialize_full
                src = materialize_full(p)
            flat[s.offset:s.offset + s.numel].copy_(src.reshape(-1))

    def _point_params(self, rt: _UnitRT, full: torch.Tensor):
        for s in rt.u.slots:
            s.param.data = full[s.offset:s.offset + s.numel].view(s.shape)
            s.param.ds_status = _param_status().AVAILABLE

    def _detach_params(self, rt: _UnitRT):
        for s in rt.u.slots:
            p = s.param
            p.ds_shape = s.shape
            p.ds_numel = s.numel
            if rt.skip_bwd_fetch:
                # Units whose backward never reads the weights are not re-gathered, but autograd still
                # validates incoming gradients against the parameter's *shape*: keep the logical shape
                # with a stride-0 one-element placeholder (no memory).
                p.data = torch.empty(1, dtype=p.dtype, device=self.device).expand(s.shape)
            else:
                p.data = torch.empty(0, dtype=p.dtype, device=self.device)
            p.ds_status = _param_status().NOT_AVAILABLE

    # =========================================================================================
    # hooks
    # =========================================================================================
    def _register_hooks(self):
        self._hook_handles = []
        for rt in self.rts:
            for s in rt.u.slots:
                p = s.param
                p.ds_unit_index = rt.u.index
                p._ds_zero = weakref.ref(self)
                self._tag_param(rt, s)
                if p.requires_grad:
                    self._hook_handles.append(p.register_post_accumulate_grad_hook(self._make_grad_hook(rt, s)))
            if self.transient and not rt.u.persistent:
                for _, b in rt.u.borrowers:
                    self._hook_borrower(rt, b)
            m = rt.u.module
            if m is None or not self.transient or rt.u.persistent:
                continue
            self._hook_handles.append(m.register_forward_pre_hook(self._make_pre_fwd(rt)))
            self._hook_handles.append(m.register_forward_hook(self._make_post_fwd(rt)))
            rt.skip_bwd_fetch = bool(getattr(m, "ds_skip_backward_fetch", False))
            if not rt.skip_bwd_fetch:
                self._hook_handles.append(m.register_full_backward_pre_hook(self._make_pre_bwd(rt)))
                if bool(getattr(self.zc, "b200_multi_forward", True)):
                    self._hook_handles.append(m.register_full_backward_hook(self._make_post_bwd(rt)))

    def _hook_borrower(self, rt, m):
        """ZeRO-3 hooks on a module outside unit ``rt`` that uses one of its parameters (a tied LM head): gather the unit
        for the module's forward and release it after; the same around its backward unless the module is
        ``ds_skip_backward_fetch`` (its backward reads no weight).  The forward fetch is recorded in the trace as a borrow,
        so once the order is known the unit is prefetched ahead of the borrower like any other unit."""

        def pre_fwd(module, args):
            self.fetch_unit(rt, forward=not self._in_backward, borrow=True)
            rt.running += 1

        def post_fwd(module, args, output):
            rt.running = max(0, rt.running - 1)
            if not self._in_backward and rt.running == 0:
                self.release_unit(rt)

        def pre_bwd(module, grad_output):
            self._in_backward = True
            self.fetch_unit(rt, forward=False, borrow=True)

        def post_bwd(module, grad_input, grad_output):
            self.release_unit(rt)

        self._hook_handles.append(m.register_forward_pre_hook(pre_fwd))
        self._hook_handles.append(m.register_forward_hook(post_fwd))
        if not getattr(m, "ds_skip_backward_fetch", False):
            self._hook_handles.append(m.register_full_backward_pre_hook(pre_bwd))
            self._hook_handles.append(m.register_full_backward_hook(post_bwd))

    def _tag_param(self, rt, s):
        """Reference-style per-parameter introspection attributes (``partition_parameters.py:1111``): ``ds_id``,
        ``ds_persist`` and ``ds_tensor``. The shard layout here is per *unit*, so ``ds_tensor`` is the (possibly empty)
        piece of this parameter that falls inside this rank's slice of the unit, not a ``ceil(numel / world)`` block."""
        p = s.param
        if not hasattr(p, "ds_id"):
            from deepspeed_b200.runtime.zero.partition_parameters import _next_id
            p.ds_id = _next_id()
        p.ds_persist = bool(rt.u.persistent)
        if self.stage < 3:
            return
        if not hasattr(p, "ds_numel"):
            p.ds_numel, p.ds_shape = s.numel, s.shape
        if not hasattr(p, "ds_status"):
            p.ds_status = _param_status().AVAILABLE
        if not hasattr(p, "ds_summary"):
            from deepspeed_b200.runtime.zero.partition_parameters import _attach_methods
            _attach_methods(p)
        try:
            shard = self._lp_shard(rt.u)
        except Exception:
            return
        if not torch.is_tensor(shard):
            return
        lo, hi = rt.u.shard_range(self.shard_rank)
        a, b = max(s.offset, lo), min(s.offset + s.numel, hi)
        # also drops a zero.Init piece (its value was packed into the unit arena; keeping it would double the lp shard)
        p.ds_tensor = shard[a - lo:b - lo] if a < b else shard[:0]

    def _make_pre_fwd(self, rt):

        def hook(module, args):
            self.fetch_unit(rt, forward=not self._in_backward)
            rt.running += 1
            if not self._in_backward and torch.is_grad_enabled():
                rt.fwd_calls += 1

        return hook

    def _make_post_fwd(self, rt):

        def hook(module, args, output):
            rt.running = max(0, rt.running - 1)
            if self._in_backward:
                return  # recompute inside backward: released by the gradient path
            if torch.is_grad_enabled() and rt.u.index == self._last_forward_unit() and not rt.skip_bwd_fetch:
                return  # its backward is next: keep it
            self.release_unit(rt)

        return hook

    def _make_pre_bwd(self, rt):

        def hook(module, grad_output):
            self._in_backward = True
            self.fetch_unit(rt, forward=False)

        return hook

    def _make_post_bwd(self, rt):
        """A module that ran MORE THAN ONCE in forward (two passes feeding one loss) is back-propagated once per invocation,
        and its parameter gradients -- hence the usual release on gradient completion -- only arrive after the last one.
        Free the gather buffer between invocations so the units of the other pass can use it (every weight-dependent node of
        this invocation has run once its input gradients exist); the next invocation's pre-backward hook gathers it back."""

        def hook(module, grad_input, grad_output):
            rt.bwd_calls += 1  # invocations are back-propagated last-to-first; the first one (possibly un-hooked) needs no release
            if rt.fwd_calls > 1 and rt.bwd_calls < rt.fwd_calls and rt.temp_refs == 0:
                self.release_unit(rt)

        return hook

    def _last_forward_unit(self):
        if self._trace_done and self._trace:
            return next((u for i, u in reversed(list(enumerate(self._trace))) if i not in self._borrow_pos),
                        self.units[-1].index)
        return self.units[-1].index

    def _make_grad_hook(self, rt, slot):

        def hook(p):
            g = p.grad
            if g is None:
                return
            self._in_backward = True
            if g.is_sparse:
                # nn.Embedding(sparse=True) / `sparse_gradients`: the unit's gradient lives in one flat dense buffer that is
                # reduced as a whole over NVLink, so a sparse gradient is densified on arrival (the reference's CSR
                # all-reduce, engine.py:2530 sparse_allreduce, trades bandwidth that NVSwitch does not lack)
                g = g.to_dense()
            view = self._grad_view(rt, slot)
            if getattr(slot, "_written", False):
                view.add_(g.reshape(-1))
            else:
                view.copy_(g.reshape(-1))
                slot._written = True
            p.grad = None
            self._param_grad_ready(rt)

        return hook

    # ---- gradient buffers ------------------------------------------------------------------------
    def _acquire_grad_buf(self, rt: _UnitRT):
        if rt.grad_full is not None:
            return
        # round-robin over the pool; wait until the previous reduce that used the slot is done
        slot = rt.own_grad_slot or self.grad_pool[rt.u.index % len(self.grad_pool)]
        if slot.owner is not None and slot.owner is not rt and slot.owner.grad_full is not None:
            # previous owner still accumulating (out-of-order graph): fall back to a private buffer
            slot = _Slot(torch.empty(self.max_full, dtype=self.comm_dtype, device=self.device))
        if slot.free_event is not None and self.on_cuda:
            self._stall_wait("reduce", lambda: torch.cuda.current_stream().wait_event(slot.free_event))
        slot.owner = rt
        rt.grad_slot = slot
        rt.grad_full = slot.buf[:rt.u.full_numel]
        # No blanket memset: every parameter slot is either written before the reduce or zeroed in the
        # flush path (unused parameters).  Only the alignment gaps must be zero, and they already are
        # when the buffer last held a unit with the same layout (all transformer blocks share one).
        sig = rt.layout_sig
        if getattr(slot, "layout_sig", None) != sig:
            rt.grad_full.zero_()
            slot.layout_sig = sig
        rt.pending = rt.n_trainable
        for s in rt.u.slots:
            s._written = False

    def _grad_view(self, rt: _UnitRT, slot) -> torch.Tensor:
        self._acquire_grad_buf(rt)
        return rt.grad_full[slot.offset:slot.offset + slot.numel]

    def grad_view_for(self, p: nn.Parameter) -> torch.Tensor:
        """Public: the flat-gradient view a custom autograd function should write ``p``'s gradient
        into (then call :meth:`mark_grad_ready`).  Avoids AccumulateGrad + copy entirely."""
        rt = self.unit_of_param[id(p)]
        s = self.slot_of_param[id(p)]
        return self._grad_view(rt, s).view(s.shape)

    def grad_is_fresh(self, p: nn.Parameter) -> bool:
        return not getattr(self.slot_of_param[id(p)], "_written", False)

    def note_grad_written(self, p: nn.Parameter):
        """Public: ``p``'s gradient view holds a contribution of this micro step, but ``p`` has another producer still
        to come (a tied LM head before the embedding's backward): the next producer accumulates instead of storing,
        and its :meth:`mark_grad_ready` is the one readiness event."""
        self._in_backward = True
        self.slot_of_param[id(p)]._written = True

    def mark_grad_ready(self, p: nn.Parameter):
        self._in_backward = True
        s = self.slot_of_param[id(p)]
        s._written = True
        self._param_grad_ready(self.unit_of_param[id(p)])

    def _param_grad_ready(self, rt: _UnitRT):
        rt.pending -= 1
        if rt.pending == 0:
            self._reduce_unit(rt)

    # =========================================================================================
    # gather / release (stage 3)
    # =========================================================================================
    def _position(self, rt):
        return self._order_pos.get(rt.u.index, rt.u.index)

    @instrument_w_nvtx
    def fetch_unit(self, rt: _UnitRT, forward=True, prefetch=True, borrow=False):
        """Make ``rt``'s parameters available on the compute stream; kick off prefetches.  ``borrow``: for a module
        outside the unit that shares one of its parameters (see :meth:`_hook_borrower`)."""
        if not self.transient or rt.u.persistent:
            return
        if forward and not self._trace_done:
            if borrow:
                self._borrow_pos.add(len(self._trace))
            self._trace.append(rt.u.index)
        prof = self.param_profiler
        if rt.state == NOT_GATHERED:
            if prof is not None:
                prof.count("fetch_miss", rt.u.full_numel)   # not prefetched: the gather is issued on demand
            self._launch_gather(rt, borrow=borrow)
        elif prof is not None:
            prof.count("fetch_hit", rt.u.full_numel)
        if rt.state == INFLIGHT:
            if rt.gather_event is not None and self.on_cuda:
                self._stall_wait("all_gather", lambda: torch.cuda.current_stream().wait_event(rt.gather_event))
            rt.state = GATHERED
        rt.consumed = True
        if prefetch and self.prefetch_depth > 0:
            for nxt, nxt_borrow in self._upcoming(rt, forward, borrow):
                if nxt.state == NOT_GATHERED and not nxt.u.persistent and (forward or not nxt.skip_bwd_fetch):
                    self._launch_gather(nxt, borrow=nxt_borrow)

    # ---- exposed-communication accounting (bench / profiling aid) -----------------------------------
    def measure_exposed(self, on=True):
        """While on, every point where the COMPUTE stream has to wait for a collective (a gather that did not
        finish in time, the reduction stream at the end of backward, a buffer still in use by a reduce) is bracketed
        with CUDA events; the bracket contains no kernels, so its elapsed time is exactly the stall."""
        self._exposed = [] if on else None

    def _stall_wait(self, what, wait_fn):
        if getattr(self, "_exposed", None) is None or not self.on_cuda:
            wait_fn()
            return
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        wait_fn()
        b.record()
        self._exposed.append((what, a, b))

    def exposed_ms(self):
        """-> {"all_gather": ms, "reduce": ms, "total": ms} since measure_exposed(True); synchronises."""
        if not getattr(self, "_exposed", None):
            return {"all_gather": 0.0, "reduce": 0.0, "total": 0.0}
        torch.cuda.synchronize()
        out = {"all_gather": 0.0, "reduce": 0.0}
        import os
        dbg = os.environ.get("DSB200_EXPOSED_DEBUG")
        for i, (what, a, b) in enumerate(self._exposed):
            ms = a.elapsed_time(b)
            out[what] += ms
            if dbg and ms > 0.05:
                print(f"[exposed] #{i} {what} {ms:.3f} ms", flush=True)
        out["total"] = out["all_gather"] + out["reduce"]
        self._exposed = []
        return out

    def _upcoming(self, rt, forward, borrow=False):
        """-> [(unit, is a borrow)] the next ``prefetch_depth`` entries of the unit order after this fetch."""
        traced = self._trace_done and self._trace
        order = self._trace if traced else [u.index for u in self.units]
        borrows = self._borrow_pos if traced else ()
        # a unit appears once as itself and once per borrow: the position of this fetch's kind
        at = [i for i, u in enumerate(order) if u == rt.u.index and (i in borrows) == borrow]
        if not at:
            return []
        pos = at[0] if forward else at[-1]
        out = []
        step = 1 if forward else -1
        for k in range(1, self.prefetch_depth + 1):
            q = pos + step * k
            if 0 <= q < len(order):
                out.append((self.rts[order[q]], q in borrows))
        return out

    def _launch_gather(self, rt: _UnitRT, borrow=False):
        """``borrow``: a gather for a module sharing the unit's weight, which runs after the unit's own module and
        typically after every other unit (a tied LM head).  It has a home of its own (``rt.borrow_home``), first the pool
        buffer that follows the last unit's: the unit's own home may be held by a unit still live at that point."""
        u = rt.u
        # Autograd may hold *views* of the gathered weights saved during forward, so the backward
        # re-gather must land in the very same memory: ``rt.home`` remembers the forward buffer.
        home = rt.borrow_home if borrow else rt.home
        if home is not None:
            slot = home
        else:
            slot = self.param_pool[(len(self.units) if borrow else u.index) % len(self.param_pool)]
        occ = slot.owner
        if occ is not None and occ is not rt and occ.state != NOT_GATHERED and not occ.consumed \
                and occ.temp_refs == 0:
            # speculative prefetch that nobody used (e.g. a module skipped by this forward): evict it
            self._detach_params(occ)
            occ.full, occ.state, occ.gather_event, occ.home = None, NOT_GATHERED, None, None
        if occ is not None and occ is not rt and occ.state != NOT_GATHERED and not self._in_backward \
                and occ.running == 0 and occ.temp_refs == 0 and not occ.u.persistent:
            # a second forward pass before backward (siamese / contrastive losses, evaluation between micro steps): the
            # unit cached in this buffer -- typically the last unit of the previous pass, kept for its backward -- is idle;
            # release it (it keeps its home: its own backward gathers it back into the same memory)
            self.release_unit(occ)
        if occ is not None and occ is not rt and occ.state != NOT_GATHERED:
            if home is not None:
                raise RuntimeError(
                    f"ZeRO-3 unit '{u.name}' must be re-gathered into the buffer it used in forward, but that "
                    f"buffer still holds live unit '{occ.u.name}'.  Increase zero_optimization.b200_unit_prefetch "
                    f"(pool size) or mark the enclosing module as a z3 leaf module.")
            slot = _Slot(self._symm_or_empty(self.max_full, self.model_dtype))  # irregular graph: private buffer
        if borrow and (self._in_backward is False or rt.borrow_home is None):
            rt.borrow_home = slot
        elif not borrow and (self._in_backward is False or rt.home is None):
            rt.home = slot
        stream = self.ag_stream
        cur = torch.cuda.current_stream() if self.on_cuda else None
        if stream is not None:
            if slot.free_event is not None:
                stream.wait_event(slot.free_event)
            if getattr(self, "_step_event", None) is not None:
                stream.wait_event(self._step_event)
        elif slot.free_event is not None and self.on_cuda:
            cur.wait_event(slot.free_event)
        full = slot.buf[:u.full_numel]
        shard = self._lp_shard(u)
        ctx = torch.cuda.stream(stream) if stream is not None else _nullctx()
        with ctx:
            if self.offload_param:
                lo, hi = u.shard_range(self.shard_rank)
                # (NVMe tier: the pinned window behind `shard` is recycled by the next unit -- finish the copy first)
                full[lo:hi].copy_(shard, non_blocking=not self.offload_param_nvme)
                shard = full[lo:hi]
            self._all_gather(full, shard, u, rt=rt)
            if self.on_cuda:
                ev = torch.cuda.Event()
                ev.record()
                rt.gather_event = ev
        slot.owner = rt
        rt.slot = slot
        rt.full = full
        rt.state = INFLIGHT
        rt.consumed = False
        self._point_params(rt, full)

    def _all_gather(self, full, shard, u: Unit, rt=None):
        if rt is not None and self.hpz > 1:
            if self._hpz_gather(full, rt):
                return
        if self.qwz:
            self._quantized_gather(full, shard, u)
            if rt is not None and self.hpz > 1:
                self._hpz_save(full, rt)
            return
        if rt is not None and self.hpz > 1:
            w = dist.all_gather_into_tensor(full, shard, group=self.dp_group, async_op=self.on_cuda)
            if w is not None and hasattr(w, "wait"):
                w.wait()
            self._hpz_save(full, rt)
            return
        if self._symm is not None and self._symm.owns(full) and self._symm.owns(shard):
            self._symm.all_gather(full, shard, u.shard_numel)
            if self._verify_left > 0:
                self._verify_all_gather(full, shard, u)
            return
        mg = getattr(self, "mics_groups", None)
        if mg is not None and mg.param_inter_node_shard_group is not None:
            from deepspeed_b200.runtime.zero.mics import hierarchical_all_gather
            hierarchical_all_gather(full, shard, mg)
            return
        w = dist.all_gather_into_tensor(full, shard, group=self.dp_group, async_op=self.on_cuda)
        if w is not None and hasattr(w, "wait"):
            w.wait()

    # ---- ZeRO++ helpers -------------------------------------------------------------------------
    def _quantized_gather(self, full, shard, u: Unit):
        """qwZ: all-gather int8 block-quantised shards (+ fp32 scales) and dequantise into ``full``; this rank's
        own range keeps its exact values (reference ``partition_parameters.py`` quantised all-gather)."""
        from deepspeed_b200.ops.quantizer import quantizer as Q
        n = u.shard_numel
        gs = Q.aligned_group_size(n)       # the device kernels want groups of a multiple of 8 elements:
        padded = (n + gs - 1) // gs * gs   # quantise a zero-padded copy of the shard when its length is not one
        g = padded // gs
        src = shard.contiguous()
        if padded != n:
            src = torch.nn.functional.pad(src, (0, padded - n))
        q, params = Q.quantize(src, g, 8, Q.Symmetric)
        qs = torch.empty(self.shard_world * q.numel(), dtype=q.dtype, device=q.device)
        ps = torch.empty(self.shard_world * params.numel(), dtype=params.dtype, device=params.device)
        dist.all_gather_into_tensor(qs, q.reshape(-1), group=self.dp_group)
        dist.all_gather_into_tensor(ps, params.reshape(-1), group=self.dp_group)
        deq = Q.dequantize(qs, ps, g * self.shard_world, 8, Q.Symmetric, dtype=full.dtype)
        deq = deq.view(self.shard_world, padded)[:, :n].reshape(-1)
        full.copy_(deq[:full.numel()])
        lo, hi = u.shard_range(self.shard_rank)
        full[lo:hi].copy_(shard)

    def _hpz_save(self, full, rt):
        """hpZ: keep this rank's slice of the freshly gathered unit as the *secondary* shard."""
        k = full.numel() // self.hpz
        hr = dist.get_rank(self.hpz_group)
        if getattr(rt, "sec", None) is None:
            rt.sec = torch.empty(k, dtype=full.dtype, device=full.device)
        rt.sec.copy_(full[hr * k:(hr + 1) * k])
        rt.sec_valid = True

    def _hpz_gather(self, full, rt) -> bool:
        """Backward re-gather inside the small (NVLink-local) group from the secondary shards."""
        if not (self._in_backward and getattr(rt, "sec_valid", False)):
            return False
        w = dist.all_gather_into_tensor(full, rt.sec, group=self.hpz_group, async_op=self.on_cuda)
        if w is not None and hasattr(w, "wait"):
            w.wait()
        return True

    @instrument_w_nvtx
    def release_unit(self, rt: _UnitRT):
        if not self.transient or rt.u.persistent or rt.state == NOT_GATHERED or rt.temp_refs > 0:
            return
        if self.on_cuda and rt.slot is not None:
            ev = torch.cuda.Event()
            ev.record()
            rt.slot.free_event = ev
        self._detach_params(rt)
        rt.full = None
        rt.state = NOT_GATHERED
        rt.gather_event = None

    def gather_all(self):
        """Gather every unit (used by state-dict export / GatheredParameters on the whole model)."""
        for rt in self.rts:
            self._ensure_ready(rt)
            if self.transient and not rt.u.persistent and rt.state == NOT_GATHERED:
                buf = torch.empty(rt.u.full_numel, dtype=self.model_dtype, device=self.device)
                shard = self._lp_shard(rt.u)
                if self.offload_param:
                    lo, hi = rt.u.shard_range(self.shard_rank)
                    buf[lo:hi].copy_(shard)
                    shard = buf[lo:hi]
                dist.all_gather_into_tensor(buf, shard, group=self.dp_group)
                rt.full = buf
                rt.slot = None
                rt.state = GATHERED
                rt.temp_refs += 1
                self._point_params(rt, buf)

    def release_all(self):
        for rt in self.rts:
            if self.transient and not rt.u.persistent and rt.state != NOT_GATHERED:
                rt.temp_refs = 0
                self._detach_params(rt)
                rt.full = None
                rt.state = NOT_GATHERED

    # =========================================================================================
    # gradient reduction
    # =========================================================================================
    def is_gradient_accumulation_boundary(self):
        """Will the micro step in flight be followed by an optimizer step?  The engine may force the answer
        (``engine.set_gradient_accumulation_boundary``, reference ``engine.py:2160``)."""
        if self._forced_boundary is not None:
            return bool(self._forced_boundary)
        return (self._accum + 1) % self.gas == 0

    def set_forced_boundary(self, is_boundary):
        """``None`` returns to counting micro steps against ``gradient_accumulation_steps``."""
        self._forced_boundary = is_boundary
        if is_boundary is not None and self.fused_in_backward:
            # the fused path needs to know *before* backward whether this micro step ends in a step; a caller that
            # drives boundaries by hand may also accumulate, which needs the gradient arena
            self.disable_fused_in_backward("gradient accumulation boundary is driven by the caller")

    def _first_micro(self, rt=None) -> bool:
        """True when this reduction must OVERWRITE the accumulated gradient (first micro step after an optimizer
        step and the unit has not been reduced yet in this micro step); a second reduction of the same unit inside
        one backward (weight used inside and outside a re-entrant checkpoint region) accumulates."""
        return self._accum == 0 and not (rt is not None and rt.reduced_this_micro)

    @instrument_w_nvtx
    def set_no_sync(self, on: bool):
        """``engine.no_sync()``: backward passes keep their gradients local (no reduction, no step); the next synchronised
        backward reduces them together with its own (reference ``engine.py:2065``)."""
        self._no_sync = bool(on)

    def _reduce_unit(self, rt: _UnitRT):
        u = rt.u
        full_g = rt.grad_full
        if getattr(self, "_no_sync", False):
            if rt.unsynced is None:
                rt.unsynced = full_g[:u.full_numel].clone()
            else:
                rt.unsynced.add_(full_g[:u.full_numel])
            if self.on_cuda:
                ev2 = torch.cuda.Event()
                ev2.record()
                rt.grad_slot.free_event = ev2
            rt.grad_full = None
            rt.grad_slot.owner = None if rt.grad_slot.owner is rt else rt.grad_slot.owner
            if self.transient and not u.persistent:
                self.release_unit(rt)
            return
        if rt.unsynced is not None:
            full_g[:u.full_numel].add_(rt.unsynced)
            rt.unsynced = None
        cur = torch.cuda.current_stream() if self.on_cuda else None
        stream = self.rs_stream
        if stream is not None:
            ev = torch.cuda.Event()
            ev.record(cur)
            stream.wait_event(ev)
        ctx = torch.cuda.stream(stream) if stream is not None else _nullctx()
        with ctx:
            scale = 1.0
            if self.dp_world > 1 or self.replica_world > 1:
                if self.prescale and self.predivide != 1.0:
                    full_g.mul_(1.0 / self.predivide)
                    scale = self.predivide / self.dp_world
                else:
                    scale = 1.0 / self.dp_world
            if self.shard_world > 1:
                lo, hi = u.shard_range(self.shard_rank)
                if self._symm is not None and self._symm.owns(full_g):
                    res = self._symm_reduce(rt, full_g, scale)
                    if res is None:
                        scale = None  # consumed inside the fused kernel
                    else:
                        shard_g, scale = res
                elif self.qgz:
                    from deepspeed_b200.runtime.comm.coalesced_collectives import all_to_all_quant_reduce
                    red = all_to_all_quant_reduce([full_g], {"local": self.dp_group})[0]  # already the shard-group mean
                    shard_g = self._rs_tmp[u.index % 2][:u.shard_numel]
                    shard_g.zero_()
                    shard_g[:red.numel()].copy_(red)
                    scale = scale * self.shard_world
                else:
                    shard_g = self._rs_tmp[u.index % 2][:u.shard_numel]
                    w = dist.reduce_scatter_tensor(shard_g, full_g, group=self.dp_group, async_op=self.on_cuda)
                    if w is not None and hasattr(w, "wait"):
                        w.wait()
                if self.replica_world > 1 and scale is not None:
                    # MiCS: sum the partial results of the model-state replicas (hierarchical all-reduce)
                    w = dist.all_reduce(shard_g, group=self.replica_group, async_op=self.on_cuda)
                    if w is not None and hasattr(w, "wait"):
                        w.wait()
                    scale = scale / self.replica_world
            else:
                if self.dp_world > 1:  # stage 0: plain data parallel
                    if self.grad_allreduce_enabled():
                        w = dist.all_reduce(full_g, group=self.dp_group, async_op=self.on_cuda)
                        if w is not None and hasattr(w, "wait"):
                            w.wait()
                    else:  # a communication-compressing optimizer (1-bit family) exchanges momentum itself
                        scale = 1.0
                shard_g = full_g
            if scale is not None:
                self._consume_shard_grad(rt, shard_g, scale)
            if self.on_cuda:
                ev2 = torch.cuda.Event()
                ev2.record()
                rt.grad_slot.free_event = ev2
        rt.grad_full = None
        rt.grad_slot.owner = None if rt.grad_slot.owner is rt else rt.grad_slot.owner
        rt.reduced_this_micro = True
        if self.transient and not u.persistent:
            self.release_unit(rt)

    def _consume_shard_grad(self, rt: _UnitRT, shard_g: torch.Tensor, scale: float):
        """Either run the fused optimizer now (boundary, no clipping) or accumulate into the arena."""
        u = rt.u
        a, b = u.arena_offset, u.arena_offset + u.shard_numel
        if self.fused_in_backward and self.is_gradient_accumulation_boundary():
            if rt.reduced_this_micro:
                raise RuntimeError(
                    f"ZeRO unit '{u.name}' produced gradients twice in one backward (a weight used both inside and "
                    f"outside a re-entrant activation-checkpoint region) while the optimizer step is fused into "
                    f"backward; set zero_optimization.b200_fused_optimizer_in_backward=false for this model")
            self._step_range(a, b, shard_g, grad_offset=a, grad_scale=scale)
            return
        first = self._first_micro(rt)
        dst = self.grad_arena[a:b]
        if dst.device != shard_g.device:  # optimizer offload: asynchronous D2H into the pinned arena
            if self.host_step_in_backward and self.is_gradient_accumulation_boundary():
                if rt.reduced_this_micro:
                    raise RuntimeError(
                        f"ZeRO unit '{u.name}' produced gradients twice in one backward while the host optimizer step "
                        f"overlaps backward; set zero_optimization.b200_fused_optimizer_in_backward=false for this model")
                done = self._offload_grad(a, b, shard_g, scale, True)
                self._host_submit(a, b, done)
                return
            self._offload_grad(a, b, shard_g, scale, first)
            return
        flat_ops.scale_cast(shard_g, dst, scale=scale, accumulate=not first)

    # ---- runtime cross-check of the in-kernel collectives against NCCL (zero_optimization.b200_verify_collectives) ---------
    def _verify_all_gather(self, full, shard, u):
        ref = torch.empty(u.full_numel, dtype=full.dtype, device=full.device)
        dist.all_gather_into_tensor(ref, shard.contiguous(), group=self.dp_group)
        if not torch.equal(ref, full[:u.full_numel]):
            bad = int((ref != full[:u.full_numel]).sum())
            raise RuntimeError(f"b200_verify_collectives: symmetric all-gather of unit '{u.name}' differs from NCCL in "
                               f"{bad} of {u.full_numel} elements")
        self.verify_report["all_gather"] += 1

    def _verify_reduce_scatter(self, rt, full_g, scale):
        """Reduce ``full_g`` twice -- NCCL and the NVLink kernel (into scratch) -- before the real kernel consumes it."""
        u = rt.u
        ref = torch.empty(u.shard_numel, dtype=full_g.dtype, device=full_g.device)
        dist.reduce_scatter_tensor(ref, full_g[:u.full_numel].clone(), group=self.dp_group)
        got = torch.empty(u.shard_numel, dtype=torch.float32, device=full_g.device)
        self._symm.reduce_scatter_accumulate(full_g, got, u.shard_numel, 1.0, accumulate=False)
        refs = ref.float()
        denom = float(refs.abs().max().clamp(min=1e-6))
        err = float((got - refs).abs().max()) / denom
        # bf16 rounding of the NCCL / switch sums bounds the disagreement
        if not (err < 2e-2):
            raise RuntimeError(f"b200_verify_collectives: symmetric reduce-scatter of unit '{u.name}' deviates from NCCL "
                               f"(max rel err {err:.3e})")
        self.verify_report["reduce_scatter"] += 1
        self.verify_report["max_rel_err"] = max(self.verify_report["max_rel_err"], err)

    # ---- host-offload pipeline -------------------------------------------------------------------------------------------
    def _offload_grad(self, a, b, shard_g, scale, first):
        """Scale the reduced shard to fp32 on the device and copy it to the pinned host gradient arena on ``d2h_stream``.
        Later micro steps land in a pinned staging arena and are added on the host in :meth:`end_backward` (the copy
        engine cannot accumulate); nothing here blocks the host or the compute stream."""
        n = b - a
        if self.d2h_stream is None:  # no CUDA: plain host path
            t = shard_g.float().mul_(scale).cpu()
            self.grad_arena[a:b].copy_(t) if first else self.grad_arena[a:b].add_(t)
            return
        if self._d2h_slots is None:
            cap = max(u.shard_numel for u in self.units)
            self._d2h_slots = [_Slot(torch.empty(cap, dtype=torch.float32, device=self.device)) for _ in range(2)]
        slot = self._d2h_slots[self._d2h_i % 2]
        self._d2h_i += 1
        cur = torch.cuda.current_stream()
        if slot.free_event is not None:
            cur.wait_event(slot.free_event)  # the copy that last read this staging buffer has finished
        tmp = slot.buf[:n]
        flat_ops.scale_cast(shard_g, tmp, scale=scale)
        ev = torch.cuda.Event()
        ev.record(cur)
        self.d2h_stream.wait_event(ev)
        if first:
            host = self.grad_arena[a:b]
        else:
            if self._grad_stage is None:
                self._grad_stage = self._empty(self.arena_numel, torch.float32, "cpu", pin=True)
            host = self._grad_stage[a:b]
            self._d2h_adds.append((a, b))
        with torch.cuda.stream(self.d2h_stream):
            host.copy_(tmp, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
        slot.free_event = done
        return done

    # ---- CPU optimizer step overlapped with backward -------------------------------------------------------------------------
    def _host_submit(self, a, b, landed):
        """Queue "step arena range [a, b) once its gradient has landed" for the worker thread (started lazily)."""
        import queue
        import threading
        if self._host_worker is None:
            self._host_q = queue.Queue()
            self._host_err = []
            dev = torch.cuda.current_device()

            def run():
                torch.cuda.set_device(dev)
                while True:
                    job = self._host_q.get()
                    try:
                        if job is None:
                            return
                        a_, b_, ev = job
                        ev.synchronize()  # the D2H copy of this shard has finished (host-side wait, no GPU stall)
                        # native CPU Adam (the ctypes call releases the GIL) + pinned bf16 staging + H2D on h2d_stream
                        self._step_range(a_, b_, self.grad_arena, 0, 1.0, join_upload=False)
                    except BaseException as e:  # surfaced by _join_host_worker on the training thread
                        self._host_err.append(e)
                    finally:
                        self._host_q.task_done()

            self._host_worker = threading.Thread(target=run, name="dsb200-host-step", daemon=True)
            self._host_worker.start()
        self._host_q.put((a, b, landed))

    def _join_host_worker(self):
        if self._host_worker is None:
            return
        self._host_q.join()
        if self._host_err:
            err = self._host_err.pop()
            self._host_err.clear()
            raise err

    def _drain_offloaded_grads(self):
        """Host-side join of the gradient D2H copies + the accumulation of later micro steps."""
        if self.d2h_stream is None:
            return
        self.d2h_stream.synchronize()
        for (a, b) in self._d2h_adds:
            self.grad_arena[a:b].add_(self._grad_stage[a:b])
        self._d2h_adds.clear()

    def _lp_upload_slot(self, n):
        """Pinned low-precision staging for one piece of updated parameters (two rotate so the CPU optimizer of piece
        k+1 overlaps the H2D copy of piece k)."""
        if self._h2d_slots is None:
            cap = max(u.shard_numel for u in self.units)
            self._h2d_slots = [_Slot(self._empty(cap, self.model_dtype, "cpu", pin=True)) for _ in range(2)]
        slot = self._h2d_slots[self._h2d_i % 2]
        self._h2d_i += 1
        if slot.free_event is not None:
            slot.free_event.synchronize()
        return slot

    def _symm_reduce(self, rt: _UnitRT, full_g, scale):
        """In-kernel reduce-scatter over NVLink peer memory, fused with scale + (Adam | accumulate).
        Returns ``None`` when the kernel consumed the gradient, else ``(shard_grad, remaining_scale)``."""
        u = rt.u
        a, b = u.arena_offset, u.arena_offset + u.shard_numel
        if self._verify_left > 0:
            self._verify_reduce_scatter(rt, full_g, scale)
        boundary = self.is_gradient_accumulation_boundary()
        # the unit that forward visited first is reduced last: nothing is left to overlap with, so it gets every SM
        tail = bool(self._trace_done and self._trace and u.index == self._trace[0])
        if self.fused_in_backward and boundary and isinstance(self.flat_opt, _adam_cls()) and self.master is not None \
                and not rt.reduced_this_micro:
            self._symm.reduce_scatter_adam(self, rt, full_g, scale, tail=tail)
            return None
        if self.grad_arena is not None and self.grad_arena.is_cuda and not self.fused_in_backward:
            first = self._first_micro(rt)
            self._symm.reduce_scatter_accumulate(full_g, self.grad_arena[a:b], u.shard_numel, scale,
                                                 accumulate=not first, tail=tail)
            return None
        tmp = self._rs_tmp[u.index % 2][:u.shard_numel]
        self._symm.reduce_scatter_accumulate(full_g, tmp, u.shard_numel, scale, accumulate=False)
        return tmp, 1.0

    def end_backward(self):
        """Flush units whose gradients are partially populated (unused parameters) and close the
        micro step.  Called by the engine after ``loss.backward()`` returns."""
        for rt in self.rts:
            if rt.grad_full is not None and rt.pending > 0:
                for sl in rt.u.slots:  # parameters that received no gradient this micro step
                    if not getattr(sl, "_written", False):
                        rt.grad_full[sl.offset:sl.offset + sl.numel].zero_()
                rt.pending = 0
                self._reduce_unit(rt)
        if self.offload_optimizer:
            self._drain_offloaded_grads()
        if self.grad_arena is not None and self._accum == 0:
            # units that produced no gradient at all this micro step must not keep stale values
            for rt in self.rts:
                if not rt.reduced_this_micro and rt.n_trainable:
                    a = rt.u.arena_offset
                    self.grad_arena[a:a + rt.u.shard_numel].zero_()
        for rt in self.rts:
            rt.reduced_this_micro = False
        if self.transient:
            for rt in self.rts:
                if not rt.u.persistent and rt.state != NOT_GATHERED and rt.grad_full is None:
                    self.release_unit(rt)
                rt.home = rt.borrow_home = None
                rt.fwd_calls = rt.bwd_calls = 0
        self._in_backward = False
        if not self._trace_done and self._trace:
            self._trace_done = True
            # keep first occurrence order, of a unit and of each unit's borrows
            seen, order, borrows = set(), [], set()
            for pos, i in enumerate(self._trace):
                key = (i, pos in self._borrow_pos)
                if key not in seen:
                    seen.add(key)
                    if key[1]:
                        borrows.add(len(order))
                    order.append(i)
            self._trace, self._borrow_pos = order, borrows
            if self.shard_world > 1:
                # every rank must walk the units in the same order or the prefetched collectives would mismatch
                # (reference coordinator.py:237 assert_ints_same_as_other_ranks)
                from deepspeed_b200.runtime.zero.utils import assert_ints_same_as_other_ranks
                assert_ints_same_as_other_ranks(order, self.dp_group)
        self.micro_step += 1
        self._accum += 1
        if self._accum % self.gas != 0 and self._forced_boundary is None:
            # more micro batches follow before the step: parameters are unchanged, so the first units of the next forward
            # can be gathered right away (with GAS > 1 every micro step would otherwise start with a cold all-gather)
            self._prefetch_next_forward()

    # =========================================================================================
    # backward / step API (reference-compatible)
    # =========================================================================================
    @property
    def loss_scale(self):
        if self.custom_loss_scaler:
            return self.external_loss_scale
        return self.loss_scaler.cur_scale

    cur_scale = loss_scale

    # ---- small reference-named conveniences (``stage3.py:563-571, :2079``; ``stage_1_and_2.py``) -----------------------
    def set_lr(self, lr):
        for g in self.param_groups:
            g["lr"] = lr

    def get_lr(self):
        return self.param_groups[0]["lr"]

    def override_loss_scale(self, loss_scale):
        """Use ``loss_scale`` (e.g. from an outer trainer) instead of the internal scaler from now on."""
        if loss_scale != self.external_loss_scale:
            logger.info(f"[deepspeed] setting loss scale from {self.external_loss_scale} -> {loss_scale}")
        self.custom_loss_scaler = True
        self.external_loss_scale = loss_scale

    def has_overflow(self, partition_gradients=True):
        """Did the last ``step`` skip because of inf/nan gradients?  (The check itself is fused into the step kernel.)"""
        return bool(self.overflow)

    def get_param_id(self, param):
        return id(param)

    def is_moe_group(self, group):
        return bool(group.get("moe", False))

    def reset_cpu_buffers(self):
        """Host staging buffers are owned by the offload runtime and reused across steps; nothing to reset per step."""

    def get_grad_norm_direct(self, gradients=None, params=None, norm_type=2):
        """Global gradient norm of the current (already reduced) gradient arena over the DP group."""
        import math
        g = self.grad_arena
        if g is None or self.fused_in_backward:
            # the step was applied unit by unit during backward: gradients no longer exist as a whole
            n = self.get_global_grad_norm()
            return float(n) if n is not None else 0.0
        if norm_type == math.inf:
            t = g.abs().max().float().reshape(1)
            if self.shard_world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.dp_group)
            return float(t.item())
        t = g.float().norm(norm_type).pow(norm_type).reshape(1)
        if self.shard_world > 1:  # the arena holds this rank's shard for every sharded stage (1, 2 and 3)
            dist.all_reduce(t, group=self.dp_group)
        return float(t.item()**(1.0 / norm_type))

    @staticmethod
    def defragment(tensors):
        """Move ``tensors`` into ONE contiguous flat buffer (each becomes a view of it) going through the host so the
        device allocator can release the scattered originals before the flat buffer is allocated; returns the buffer."""
        assert len({t.dtype for t in tensors}) == 1 and len({t.device for t in tensors}) == 1
        dev = tensors[0].device
        host = torch.empty(sum(t.numel() for t in tensors), dtype=tensors[0].dtype,
                           pin_memory=dev.type == "cuda" and torch.cuda.is_available())
        off = []
        pos = 0
        for t in tensors:
            n = t.numel()
            host[pos:pos + n].copy_(t.data.reshape(-1))
            off.append(pos)
            t.data = torch.empty(0, dtype=t.dtype, device=dev)  # drop the scattered storage
            pos += n
        if dev.type == "cuda":
            torch.cuda.empty_cache()
        flat = host.to(dev)
        sizes = [off[i + 1] - off[i] for i in range(len(off) - 1)] + [host.numel() - off[-1]]
        for t, o, n in zip(tensors, off, sizes):
            t.data = flat[o:o + n]
        return flat

    def backward(self, loss, retain_graph=False):
        self._in_backward = True
        if self.custom_loss_scaler:
            (loss * self.external_loss_scale).backward(retain_graph=retain_graph)
        else:
            self.loss_scaler.backward(loss.float(), retain_graph=retain_graph)
        self.end_backward()

    def zero_grad(self, set_to_none=True):
        for p in self.module.parameters():
            p.grad = None
        for rt in self.rts:
            rt.unsynced = None  # gradients parked under engine.no_sync()

    def _group_hyper(self, gi):
        return self.param_groups[gi]

    def _step_range(self, a, b, grad, grad_offset, grad_scale, d_gscale=None, d_skip=None, join_upload=True):
        """Run the flat optimizer over arena range [a, b).  ``grad`` holds arena coordinates
        ``[grad_offset, ...)``."""
        write_lp = self.master is not None and not self.offload_optimizer
        work = []
        win = self.state_swapper.window_elems if self.state_swapper is not None else None
        for (rt, gi, s0, e0) in self.pieces:
            s1, e1 = max(s0, a), min(e0, b)
            if s1 >= e1 or gi < 0:
                continue
            if win is None:
                work.append((rt, gi, s1, e1))
            else:  # NVMe tier: never touch more than one swap window of state at a time
                for c in range(s1, e1, win):
                    work.append((rt, gi, c, min(c + win, e1)))
        upload = self.offload_optimizer and self.h2d_stream is not None and self.master is not None \
            and not self.offload_param
        for i, (rt, gi, s1, e1) in enumerate(work):
            if self.state_swapper is not None and i + 1 < len(work):
                self.state_swapper.prefetch(self.flat_opt, work[i + 1][2], work[i + 1][3])
            p = self._piece_master(rt, s1, e1)
            g = grad[s1 - grad_offset:e1 - grad_offset]
            out = self._piece_lp(rt, s1, e1) if write_lp else None
            slot = None
            if upload:
                # the CPU optimizer writes the low-precision copy of this piece into pinned staging in the same pass;
                # its H2D copy then overlaps the CPU work on the next piece
                slot = self._lp_upload_slot(e1 - s1)
                out = slot.buf[:e1 - s1]
            self.flat_opt.step_segment(s1, e1, p, g, out, self.param_groups[gi], self._peek_step(gi),
                                       grad_scale=grad_scale, d_gscale=d_gscale, d_skip=d_skip)
            if slot is not None:
                with torch.cuda.stream(self.h2d_stream):
                    self._piece_lp(rt, s1, e1).copy_(out, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record()
                slot.free_event = ev
        if upload:
            if join_upload:
                torch.cuda.current_stream().wait_stream(self.h2d_stream)
            self._uploaded_lp = True
        if self.state_swapper is not None:
            self.state_swapper.flush(self.flat_opt)

    # ---- reference-style introspection (stage3.py / stage_1_and_2.py attribute names) ---------------------------------
    @property
    def fp32_partitioned_groups_flat(self):
        """This rank's fp32 master partition(s). The reference keeps one flat tensor per sub-group; here every unit's
        shard lives in ONE arena, exposed as a single-entry list."""
        return [self.master] if torch.is_tensor(self.master) else []

    single_partition_of_fp32_groups = fp32_partitioned_groups_flat

    @property
    def optimizer(self):
        """The wrapped optimizer as the reference exposes it (``engine.optimizer.optimizer``): ``param_groups``,
        ``state`` (this rank's flat moment arenas + step count) and ``state_dict()``."""
        return _InnerOptimizerView(self)

    @property
    def state(self):
        """torch-style ``optimizer.state`` (one entry: this rank's flat moment arenas and the step count)."""
        return self.optimizer.state

    nccl_start_alignment_factor = 2  # reference constant (element alignment of partition starts); arenas here are 16 B aligned

    def _peek_step(self, gi):
        # group_steps is advanced once per global step in step(); during fused-in-backward calls the
        # upcoming value is used.
        return self.group_steps[gi] + 1

    @instrument_w_nvtx
    def step(self, closure=None):
        """Optimizer step at a gradient-accumulation boundary."""
        self.prepare_step()
        self.finish_step()

    def needs_norm(self):
        return (not self.fused_in_backward) and (self.clip > 0.0 or self.dynamic_loss_scale
                                                 or self.model_dtype == torch.float16)

    def prepare_step(self):
        """Phase 1: join the reduction stream and compute this instance's squared gradient norm / overflow
        flag (already summed over its own sharding group).  Split from :meth:`finish_step` so that several
        instances (dense + expert parameter domains) can combine their norms before clipping."""
        if self.on_cuda and self.rs_stream is not None:
            self._stall_wait("reduce", lambda: torch.cuda.current_stream().wait_stream(self.rs_stream))
        self.overflow = False
        if self.needs_norm():
            self.stats.reset()
            self.stats.accumulate(self.grad_arena)
            self._allreduce_stats(self.stats)

    def finish_step(self, extra_sumsq=None, extra_found_inf=None):
        if self.host_step_in_backward:
            # every unit was stepped on the host while backward ran: wait for the stragglers and for their uploads
            self._join_host_worker()
            if self.h2d_stream is not None:
                torch.cuda.current_stream().wait_stream(self.h2d_stream)
            for gi in range(len(self.group_steps)):
                self.group_steps[gi] += 1
            self._post_step()
            self._apply_pending_defuse()
            return
        if self.fused_in_backward:
            # parameters were already updated unit-by-unit inside backward
            for gi in range(len(self.group_steps)):
                self.group_steps[gi] += 1
            self._post_step()
            self._apply_pending_defuse()
            return
        inv_scale = 1.0 / float(self.loss_scale)
        need_norm = self.needs_norm()
        stats = self.stats
        d_gscale = d_skip = None
        if need_norm:
            if extra_sumsq is not None:
                stats.sumsq.add_(extra_sumsq.to(stats.sumsq.device))
            if extra_found_inf is not None:
                stats.found_inf.copy_(torch.maximum(stats.found_inf, extra_found_inf.to(stats.found_inf.device)))
            stats.finalize(inv_loss_scale=inv_scale, max_norm=self.clip)
            d_gscale, d_skip = stats.gscale, stats.skip
            self._global_grad_norm = stats.norm
            if self.dynamic_loss_scale or self.model_dtype == torch.float16:
                self.overflow = bool(int(stats.skip.item()))  # fp16 needs the host to adapt the scale
                self.loss_scaler.update_scale(self.overflow)
                if self.overflow:
                    self.skipped_steps += 1
                    log_dist(f"[deepspeed_b200] OVERFLOW! Skipping step, loss scale -> {self.loss_scale}", ranks=[0])
                    self._post_step(skipped=True)
                    return
        gscale = 1.0 if need_norm else inv_scale
        if isinstance(self.flat_opt, TorchOptimizerAdapter):
            g32 = self.grad_arena
            if need_norm:
                g32.mul_(stats.gscale.to(g32.device))
            elif gscale != 1.0:
                g32.mul_(gscale)
            self.flat_opt.step_all(g32)
            self._master_to_lp(0, self.arena_numel)
        elif getattr(self.flat_opt, "per_tensor", False):
            self._step_per_tensor(gscale, d_gscale, d_skip)
        else:
            if self.offload_optimizer and d_skip is not None and int(d_skip.item()):
                # inf / nan gradients (the statistics live on the host for the offload tier): nothing is updated
                self.overflow = True
                self.skipped_steps += 1
                self._post_step(skipped=True)
                return
            self._uploaded_lp = False
            self._step_range(0, self.arena_numel, self.grad_arena, 0, gscale, d_gscale, None if self.offload_optimizer
                             else d_skip)
            if self.offload_optimizer and not self._uploaded_lp:
                self._master_to_lp(0, self.arena_numel)
        for gi in range(len(self.group_steps)):
            self.group_steps[gi] += 1
        self._post_step()

    def _step_per_tensor(self, gscale, d_gscale, d_skip):
        for rt in self.rts:
            for sl in rt.u.slots:
                if sl.group < 0:
                    continue
                for (r, p0, a0, ln) in param_fragments(rt.u, sl, self.shard_world):
                    if r != self.shard_rank:
                        continue
                    self.flat_opt.step_segment(a0, a0 + ln, self._piece_master(rt, a0, a0 + ln),
                                               self.grad_arena[a0:a0 + ln], None, self.param_groups[sl.group],
                                               self.group_steps[sl.group] + 1, grad_scale=gscale, d_gscale=d_gscale,
                                               d_skip=d_skip)
        self._master_to_lp(0, self.arena_numel)

    def _master_to_lp(self, a, b):
        """fp32 master -> low-precision shard (H2D when the optimizer lives on the host)."""
        if self.master is None:
            return
        for rt in self.rts:
            u = rt.u
            s, e = max(a, u.arena_offset), min(b, u.arena_offset + u.shard_numel)
            if s >= e:
                continue
            dst = self._lp_shard(u)[s - u.arena_offset:e - u.arena_offset]
            src = self.master[s:e]
            if not isinstance(src, torch.Tensor):
                src = src.detach()  # NVMe-resident master: read this range back window by window
            if src.device != dst.device:
                dst.copy_(src.to(dst.dtype), non_blocking=True)
            else:
                flat_ops.scale_cast(src, dst)

    def _allreduce_stats(self, stats):
        if self.shard_world > 1:
            t = stats.sumsq if stats.sumsq.device == self.device else stats.sumsq.to(self.device)
            f = stats.found_inf if stats.found_inf.device == self.device else stats.found_inf.to(self.device)
            dist.all_reduce(t, group=self.dp_group)
            dist.all_reduce(f, op=dist.ReduceOp.MAX, group=self.dp_group)
            if t is not stats.sumsq:
                stats.sumsq.copy_(t)
                stats.found_inf.copy_(f)
        if self.mpu is not None and hasattr(self.mpu, "get_model_parallel_group"):
            mp = self.mpu.get_model_parallel_group()
            if dist.get_world_size(mp) > 1:
                dist.all_reduce(stats.sumsq, group=mp)
                dist.all_reduce(stats.found_inf, op=dist.ReduceOp.MAX, group=mp)

    def _post_step(self, skipped=False):
        """Make the updated low-precision parameters visible: stage<=2 all-gathers each unit in
        place; stage 3 invalidates gathered copies (persistent units are re-gathered)."""
        if self._symm is not None:
            self._symm.barrier()  # every rank's shard is final before any peer reads it
        gathered = False
        if not skipped and self.shard_world > 1:
            if not self.transient:
                for rt in self.rts:
                    lo, hi = rt.u.shard_range(self.shard_rank)
                    self._all_gather(rt.full, rt.full[lo:hi], rt.u)
                    gathered = True
            else:
                for rt in self.rts:
                    if rt.u.persistent:
                        lo, hi = rt.u.shard_range(self.shard_rank)
                        rt.full[lo:hi].copy_(self._lp_shard(rt.u))
                        self._all_gather(rt.full, rt.full[lo:hi], rt.u)
        if self._symm is not None and gathered:
            self._symm.barrier()  # peers are done reading our in-place shard before the next update
        if self.hpz > 1:
            for rt in self.rts:
                rt.sec_valid = False
        if self.on_cuda:
            ev = torch.cuda.Event()
            ev.record()
            self._step_event = ev
        self._accum = 0
        self.global_step += 1
        self._prefetch_next_forward()
        if self._verify_left > 0:
            self._verify_left -= 1
            if self._verify_left == 0:
                log_dist(f"b200_verify_collectives: NVLink kernels agreed with NCCL ({self.verify_report})", ranks=[0])

    def _prefetch_next_forward(self):
        """Start gathering the first units of the NEXT forward right after the step that produced their new values.

        The parameter pool is idle between ``step()`` and the next ``forward`` (loss read-back, data loading, the engine's
        Python), and the first forward units otherwise wait for a cold all-gather with nothing to overlap (the 3.6 ms
        "exposed all-gather" of the 8-GPU Llama-3-8B run).  Only done once the unit order is known and for as many units
        as the pool can hold next to the usual look-ahead."""
        if not (self.transient and self._trace_done and self._trace and self.on_cuda and self.ag_stream is not None):
            return
        if self.offload_param or not torch.is_grad_enabled():
            return
        n = 0
        for idx in self._trace:
            rt = self.rts[idx]
            if rt.u.persistent:
                continue
            if n >= 1 + self.prefetch_depth:
                break
            if rt.state == NOT_GATHERED and rt.temp_refs == 0:
                slot = self.param_pool[rt.u.index % len(self.param_pool)]
                if slot.owner is not None and slot.owner is not rt and slot.owner.state != NOT_GATHERED:
                    break  # the pool slot is still held: leave it to the regular on-demand path
                self._launch_gather(rt)
            n += 1

    # =========================================================================================
    # GatheredParameters / external-parameter support
    # =========================================================================================
    def param_is_gathered(self, p) -> bool:
        rt = self.unit_of_param[id(p)]
        return (not self.transient) or rt.u.persistent or rt.state != NOT_GATHERED

    def _ensure_ready(self, rt):
        """A unit gathered speculatively (look-ahead / post-step prefetch) is only ordered on ``ag_stream``: make the
        current stream wait for it before anybody outside forward/backward touches the data."""
        if rt.state == INFLIGHT:
            if rt.gather_event is not None and self.on_cuda:
                torch.cuda.current_stream().wait_event(rt.gather_event)
            rt.state = GATHERED

    def gather_param_temp(self, p):
        """Gather the unit owning ``p`` into a private buffer (outside the rotating pool)."""
        rt = self.unit_of_param[id(p)]
        self._ensure_ready(rt)
        if rt.state == NOT_GATHERED:
            buf = torch.empty(rt.u.full_numel, dtype=self.model_dtype, device=self.device)
            shard = self._lp_shard(rt.u)
            if shard.device != buf.device:
                lo, hi = rt.u.shard_range(self.shard_rank)
                buf[lo:hi].copy_(shard)
                shard = buf[lo:hi]
            dist.all_gather_into_tensor(buf, shard, group=self.dp_group)
            rt.full, rt.slot, rt.state = buf, None, GATHERED
            self._point_params(rt, buf)
        rt.temp_refs += 1

    def release_param_temp(self, p, write_back_from=None):
        rt = self.unit_of_param[id(p)]
        if write_back_from is not None:
            self.sync_param_from_full(p, write_back_from)
        rt.temp_refs = max(0, rt.temp_refs - 1)
        if rt.temp_refs == 0 and self.transient and not rt.u.persistent and not self._in_backward:
            self._detach_params(rt)
            rt.full, rt.state, rt.gather_event = None, NOT_GATHERED, None

    @torch.no_grad()
    def sync_param_from_full(self, p, src_rank=0):
        """Propagate an in-place edit of a gathered parameter: broadcast from ``src_rank`` then refresh
        this rank's low-precision shard and fp32 master."""
        rt, s = self.unit_of_param[id(p)], self.slot_of_param[id(p)]
        self._ensure_ready(rt)
        full = rt.full[s.offset:s.offset + s.numel]
        if self.dp_world > 1:
            src = dist.get_global_rank(self.dp_group, src_rank) if self.dp_group is not None else src_rank
            dist.broadcast(full, src=src, group=self.dp_group)
        for (r, p0, a0, ln) in param_fragments(rt.u, s, self.shard_world):
            if r != self.shard_rank:
                continue
            piece = full[p0:p0 + ln]
            if self.lp_arena is not None:
                self.lp_arena[a0:a0 + ln].copy_(piece)
            if self.master is not None:
                self.master[a0:a0 + ln].copy_(piece)

    def get_full_lp_param(self, p):
        rt, s = self.unit_of_param[id(p)], self.slot_of_param[id(p)]
        self._ensure_ready(rt)
        if rt.state != NOT_GATHERED and rt.full is not None:
            return rt.full[s.offset:s.offset + s.numel].view(s.shape)
        arena = self._lp_arena_as_flat()
        return self._gather_arena_piece(arena, rt, s).to(self.model_dtype)

    def add_external_dependency(self, module: nn.Module, parameter: nn.Parameter):
        rt = self.unit_of_param.get(id(parameter))
        if rt is None or not self.transient or rt.u.persistent:
            return

        def pre(mod, args):
            self.fetch_unit(rt, forward=False, prefetch=False)

        def post(mod, args, out):
            if not torch.is_grad_enabled():
                self.release_unit(rt)

        self._hook_handles.append(module.register_forward_pre_hook(pre))
        self._hook_handles.append(module.register_forward_hook(post))
        self._hook_handles.append(module.register_full_backward_pre_hook(lambda m, g: self.fetch_unit(rt, False, False)))

    def destroy(self):
        for h in self._hook_handles:
            h.remove()
        self._hook_handles.clear()
        if getattr(self, "_host_worker", None) is not None:
            self._host_q.put(None)  # stop the host-step worker
            self._host_worker = None

    # =========================================================================================
    # introspection helpers (tensor_fragment API, checkpointing)
    # =========================================================================================
    def get_global_grad_norm(self):
        n = self._global_grad_norm
        return None if n is None else float(n.item())

    def _gather_arena_piece(self, arena: torch.Tensor, rt: _UnitRT, slot) -> torch.Tensor:
        """Reassemble one parameter's fp32 values from every rank's arena (debug / checkpoint API)."""
        u = rt.u
        a = u.arena_offset
        shard = arena[a:a + u.shard_numel].to(self.device, torch.float32)
        if self.shard_world > 1:
            full = torch.empty(u.full_numel, dtype=torch.float32, device=self.device)
            dist.all_gather_into_tensor(full, shard.contiguous(), group=self.dp_group)
        else:
            full = shard
        return full[slot.offset:slot.offset + slot.numel].view(slot.shape).clone()

    def get_full_hp_param(self, p):
        rt, s = self.unit_of_param[id(p)], self.slot_of_param[id(p)]
        if self.master is None:
            return self._gather_arena_piece(self._lp_arena_as_flat(), rt, s)
        return self._gather_arena_piece(self.master, rt, s)

    def get_full_hp_grad(self, p):
        rt, s = self.unit_of_param[id(p)], self.slot_of_param[id(p)]
        if rt.unsynced is not None:  # inside engine.no_sync(): this rank's local, not yet reduced gradient
            return rt.unsynced[s.offset:s.offset + s.numel].view(s.shape).float().clone()
        if self.fused_in_backward or self.host_step_in_backward:
            # the step ran unit by unit inside backward and consumed the gradients as they were produced. Keep them from
            # the next step on (two-phase step) so that gradient introspection works as in the reference.
            if getattr(self, "_defuse_after_step", None) is None:
                self._defuse_after_step = "gradient introspection (safe_get_full_grad)"
                logger.warning("safe_get_full_grad(): gradients of this step were already consumed by the optimizer step "
                               "fused into backward; switching to the two-phase step so they are available from the next "
                               "step on (set zero_optimization.b200_fused_optimizer_in_backward=false to start that way)")
            return None
        if self.grad_arena is None:
            return None
        return self._gather_arena_piece(self.grad_arena, rt, s)

    def get_full_optimizer_state(self, p, key):
        st = self.flat_opt.state_tensors()
        if isinstance(self.flat_opt, TorchOptimizerAdapter):
            return None
        if key not in st:
            return None
        rt, s = self.unit_of_param[id(p)], self.slot_of_param[id(p)]
        return self._gather_arena_piece(st[key], rt, s)

    def _lp_arena_as_flat(self):
        if self.lp_arena is not None:
            return self.lp_arena
        if self.shard_world == 1 and self.full_arena is not None:
            # one shard per unit == the whole unit, units back to back: the resident buffer IS the arena (a writable view,
            # so loaders that scatter into it -- fp32 training has no separate master -- really update the parameters)
            return self.full_arena[:self.arena_numel]
        return torch.cat([self._lp_shard(u) for u in self.units])

    def set_full_hp_param(self, value, p):
        rt, s = self.unit_of_param[id(p)], self.slot_of_param[id(p)]
        self._scatter_into_arena(self.master, rt, s, value)
        # keep the low-precision copy coherent
        for (r, p0, a0, ln) in param_fragments(rt.u, s, self.shard_world):
            if r == self.shard_rank:
                dst = self._lp_shard(rt.u)[a0 - rt.u.arena_offset:a0 - rt.u.arena_offset + ln]
                dst.copy_(value.reshape(-1)[p0:p0 + ln].to(dst.device, dst.dtype))
        self._ensure_ready(rt)
        if rt.state == GATHERED and rt.full is not None:
            rt.full[s.offset:s.offset + s.numel].copy_(value.reshape(-1).to(rt.full.device, rt.full.dtype))

    def set_full_optimizer_state(self, value, p, key):
        st = self.flat_opt.state_tensors()
        rt, s = self.unit_of_param[id(p)], self.slot_of_param[id(p)]
        self._scatter_into_arena(st[key], rt, s, value)

    def _scatter_into_arena(self, arena, rt, s, value):
        if arena is None:
            return
        flat = value.reshape(-1)
        for (r, p0, a0, ln) in param_fragments(rt.u, s, self.shard_world):
            if r == self.shard_rank:
                arena[a0:a0 + ln].copy_(flat[p0:p0 + ln].to(arena.device, arena.dtype))

    # ---- state dict ---------------------------------------------------------------------------------
    def state_dict(self, layout=None):
        """This rank's optimizer shard.  ``layout="reference"`` (the default for sharded stages, see
        ``checkpoint.b200_shard_layout``) writes the reference's on-disk format (``fp32_flat_groups`` +
        ``optimizer_state_dict`` for stage 3; ``single_partition_of_fp32_groups`` + ``base_optimizer_state`` +
        ``param_slice_mappings`` + ``group_paddings`` for stage 1/2 -- ``runtime/zero/ref_layout.py``) so stock tools read
        it; ``layout="arena"`` dumps the rank-local arenas as they are (no re-partitioning traffic)."""
        layout = layout or getattr(self, "checkpoint_layout", "arena")
        if layout == "reference" and self.stage >= 1 and self.state_swapper is None:
            from deepspeed_b200.runtime.zero.ref_layout import export_reference_state
            return export_reference_state(self)
        sd = {
            "zero_stage": self.stage,
            "loss_scaler": self.loss_scaler.state_dict(),
            "dynamic_loss_scale": self.dynamic_loss_scale,
            "overflow": self.overflow,
            "partition_count": self.shard_world,
            "group_steps": list(self.group_steps),
            "global_step": self.global_step,
            "param_groups": [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups],
            "fp32_flat": (self.master if self.master is not None else self._lp_arena_as_flat()).detach().cpu().clone(),
            "arena_numel": self.arena_numel,
            "unit_layout": [(u.name, u.full_numel, u.shard_numel, u.arena_offset) for u in self.units],
        }
        if isinstance(self.flat_opt, TorchOptimizerAdapter):
            sd["base_optimizer_state"] = self.flat_opt.optimizer.state_dict()
        else:
            sd["flat_state"] = {k: v.detach().cpu().clone() for k, v in self.flat_opt.state_tensors().items()}
        return sd

    def load_state_dict(self, sd, load_optimizer_states=True, load_from_fp32_weights=True, param_shapes=None):
        from deepspeed_b200.runtime.zero import ref_layout
        if ref_layout.is_reference_layout(sd):  # written by stock DeepSpeed or by us with layout="reference"
            ref_layout.import_reference_state(self, sd, load_optimizer_states, load_from_fp32_weights, param_shapes)
            return
        assert sd["partition_count"] == self.shard_world, (
            f"checkpoint was saved with {sd['partition_count']} shards but this run has {self.shard_world}; "
            f"use the universal checkpoint path to reshape")
        self.loss_scaler.load_state_dict(sd["loss_scaler"])
        self.group_steps = list(sd.get("group_steps", self.group_steps))
        self.global_step = sd.get("global_step", 0)
        for g, saved in zip(self.param_groups, sd.get("param_groups", [])):
            g.update(saved)
        if load_from_fp32_weights:
            src = sd["fp32_flat"]
            if self.master is not None:
                self.master.copy_(src.to(self.master.device, self.master.dtype))
            else:
                for rt in self.rts:
                    a0 = rt.u.arena_offset
                    sh = self._lp_shard(rt.u)
                    sh.copy_(src[a0:a0 + rt.u.shard_numel].to(sh.device, sh.dtype))
            self._refresh_lp_from_master()
        if load_optimizer_states:
            if isinstance(self.flat_opt, TorchOptimizerAdapter) and "base_optimizer_state" in sd:
                self.flat_opt.optimizer.load_state_dict(sd["base_optimizer_state"])
            elif "flat_state" in sd:
                for k, v in sd["flat_state"].items():
                    self.flat_opt.state_tensors()[k].copy_(v)

    # ---- names used by the reference's BF16_Optimizer / coordinator (API compatibility) ------------------------
    def update_lp_params(self):
        """fp32 master -> low-precision parameters (+ all-gather for sharded stages)."""
        self._refresh_lp_from_master()

    def update_hp_grads(self, clear_lp_grads=False):
        """Gradients are accumulated into the fp32/bf16 shard arena as they are reduced; nothing to fold here."""
        if clear_lp_grads:
            self.zero_grad()

    def reset_step(self):
        """Forget the recorded unit order (the module graph changed): it is re-traced on the next iteration."""
        self._trace, self._trace_done, self._borrow_pos = [], False, set()

    def clear_lp_grads(self):
        self.zero_grad()

    def _refresh_lp_from_master(self):
        if self.master is not None:
            self._master_to_lp(0, self.arena_numel)
        self._post_step(skipped=False)
        self.global_step -= 1


def _adam_cls():
    from deepspeed_b200.runtime.zero.flat_optimizers import FlatAdam
    return FlatAdam


class _nullctx:

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
