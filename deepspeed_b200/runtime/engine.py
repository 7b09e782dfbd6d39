"""``DeepSpeedEngine`` -- wraps a module for mixed-precision, ZeRO-sharded data-parallel training.

Parity target: reference ``runtime/engine.py:184`` (forward / backward / step, optimizer + scheduler
selection, gradient accumulation, dtype casting, timers, monitor, checkpoint save/load, 16-bit
model export, ``no_sync``).  Architectural difference: every optimizer path (plain DP, bf16, fp16,
ZeRO-1/2/3, offload) goes through ONE class, :class:`ZeroShardedOptimizer`, parameterised by
stage; the engine therefore has no allreduce-bucket fallback code of its own.
"""
import contextlib
import os
import re
from typing import Optional

import torch
from torch import nn

from deepspeed_b200 import comm as dist
from deepspeed_b200.accelerator import get_accelerator
from deepspeed_b200.monitor.monitor import MonitorMaster
from deepspeed_b200.runtime import lr_schedules
from deepspeed_b200.runtime.checkpointing import CheckpointMixin
from deepspeed_b200.runtime.config import (ADAGRAD_OPTIMIZER, ADAM_OPTIMIZER, ADAMW_OPTIMIZER, DeepSpeedConfig,
                                           LAMB_OPTIMIZER, LION_OPTIMIZER, ONEBIT_ADAM_OPTIMIZER,
                                           ONEBIT_LAMB_OPTIMIZER, SGD_OPTIMIZER, ZERO_ONE_ADAM_OPTIMIZER)
from deepspeed_b200.runtime.dataloader import DeepSpeedDataLoader
from deepspeed_b200.runtime.zero.sharded import ZeroShardedOptimizer
from deepspeed_b200.utils import groups
from deepspeed_b200.utils.logging import log_dist, logger
from deepspeed_b200.utils.nvtx import instrument_w_nvtx
from deepspeed_b200.utils.timer import (BACKWARD_GLOBAL_TIMER, BACKWARD_MICRO_TIMER, FORWARD_GLOBAL_TIMER,
                                        FORWARD_MICRO_TIMER, NoopTimer, STEP_GLOBAL_TIMER, STEP_MICRO_TIMER,
                                        SynchronizedWallClockTimer, ThroughputTimer)

MEMORY_OPT_ALLREDUCE_SIZE = 500000000
DeepSpeedOptimizerCallable = object
DeepSpeedSchedulerCallable = object


def split_half_float_double_sparse(tensors):
    """Group gradients for bucketed reduction: ``([(dtype, [SparseTensor...])], [(dtype, [dense...])])``
    (reference ``engine.py:126``)."""
    from deepspeed_b200.runtime.sparse_tensor import SparseTensor
    supported = (torch.float16, torch.bfloat16, torch.float32, torch.float64)
    sparse, dense = {}, {}
    for t in tensors:
        assert t.dtype in supported, f"attempting to reduce an unsupported grad type: {t.dtype}"
        (sparse if isinstance(t, SparseTensor) else dense).setdefault(t.dtype, []).append(t)
    order = lambda d: [(dt, d[dt]) for dt in supported if dt in d]
    return order(sparse), order(dense)


from deepspeed_b200.runtime.engine_accessors import EngineConfigAccessors  # noqa: E402


class EngineTimers:
    """Names of the wall-clock timers the engine drives, grouped by phase (reference ``engine.py:149``)."""

    def __init__(self, enable_micro_timers, enable_global_timers):
        from deepspeed_b200.utils import timer as T
        phases = ("forward", "backward", "backward_inner", "backward_reduce", "step")
        table = {"micro": dict(zip(phases, (T.FORWARD_MICRO_TIMER, T.BACKWARD_MICRO_TIMER, T.BACKWARD_INNER_MICRO_TIMER,
                                            T.BACKWARD_REDUCE_MICRO_TIMER, T.STEP_MICRO_TIMER))),
                 "global": dict(zip(phases, (T.FORWARD_GLOBAL_TIMER, T.BACKWARD_GLOBAL_TIMER, T.BACKWARD_INNER_GLOBAL_TIMER,
                                             T.BACKWARD_REDUCE_GLOBAL_TIMER, T.STEP_GLOBAL_TIMER)))}
        on = {"micro": enable_micro_timers, "global": enable_global_timers}
        for ph in phases:
            setattr(self, f"{ph}_timers", [table[k][ph] for k in ("micro", "global") if on[k]])
        self.micro_timers = list(table["micro"].values()) if enable_micro_timers else []
        self.global_timers = list(table["global"].values()) if enable_global_timers else []


class DeepSpeedEngine(CheckpointMixin, EngineConfigAccessors, nn.Module):

    def __init__(self, args=None, model=None, optimizer=None, model_parameters=None, training_data=None,
                 lr_scheduler=None, mpu=None, dist_init_required=None, collate_fn=None, config=None,
                 config_class: Optional[DeepSpeedConfig] = None, mesh_device=None, dont_change_device=False):
        super().__init__()
        self.dont_change_device = dont_change_device
        self.client_optimizer = optimizer
        self.client_lr_scheduler = lr_scheduler
        self.training_data = training_data
        self.collate_fn = collate_fn
        self.mpu = mpu
        self.mesh_device = mesh_device
        self.global_steps = 0
        self.global_samples = 0
        self.micro_steps = 0
        self.skipped_steps = 0
        self.gradient_average = True
        self.warn_unscaled_loss = True
        self.loaded_checkpoint_mp_world_size = None
        self.loaded_checkpoint_dp_world_size = None
        self.enable_backward_allreduce = True
        self.losses = None
        self._is_gradient_accumulation_boundary = None
        self.scale_wrt_gas = None
        self.accel = get_accelerator()

        dist.init_distributed(dist_init_required=dist_init_required)
        self._config = config_class if config_class is not None else DeepSpeedConfig(config, mpu,
                                                                                      mesh_device=mesh_device)
        self._set_distributed_vars(args)
        dist.configure(self._config)
        self.monitor = MonitorMaster(self._config.monitor_config)

        self._configure_parallel_groups()
        self.module = model
        self._configure_distributed_model(model)
        self.timers = SynchronizedWallClockTimer() if self.wall_clock_breakdown() else NoopTimer()
        self.tput_timer = ThroughputTimer(self._config.timers_config.throughput,
                                          batch_size=self.train_batch_size(),
                                          steps_per_output=self.steps_per_print(),
                                          monitor_memory=False)
        self.training_dataloader = self.deepspeed_io(training_data) if training_data is not None else None

        # ---- optimizer -------------------------------------------------------------------------
        self.optimizer = None
        self.basic_optimizer = None
        self.lr_scheduler = None
        has_opt = optimizer is not None or self._config.optimizer_name is not None
        if model_parameters is None and has_opt:
            model_parameters = [p for p in self.module.parameters() if p.requires_grad]
        if has_opt:
            self._configure_optimizer(optimizer, model_parameters)
            self._configure_lr_scheduler(lr_scheduler)
        elif self.zero_optimization_stage() == 3:
            # ZeRO-Inference: parameter sharding + fetch hooks without an optimizer
            self._configure_zero_inference()
        self._configure_aux()
        if self.global_rank == 0 and self._config.dump_state:
            self._config.print("DeepSpeedEngine configuration")

    # =========================================================================================
    # setup
    # =========================================================================================
    def _set_distributed_vars(self, args):
        self.local_rank = int(os.environ.get("LOCAL_RANK", getattr(args, "local_rank", 0) or 0))
        self.world_size = dist.get_world_size()
        self.global_rank = dist.get_rank()
        if self.accel.device_name() == "cuda" and not self.dont_change_device:
            self.accel.set_device(self.local_rank % max(self.accel.device_count(), 1))
            self.device = torch.device("cuda", self.accel.current_device())
        else:
            self.device = torch.device("cpu") if self.accel.device_name() == "cpu" else torch.device(
                "cuda", torch.cuda.current_device())

    def _configure_parallel_groups(self):
        sp = int(self._config.sequence_parallel_size or 1)
        tp = int(self._config.tensor_parallel_config.autotp_size or 0) or 1
        if self.mpu is not None:
            groups.initialize(mpu=self.mpu)
        elif self.mesh_device is not None:
            groups.mesh_device = self.mesh_device
            # ``initialize(mesh_param=(dp, sp))`` without ``sequence_parallel_size`` in the config: the mesh is the authority
            sp = int(groups._get_sequence_parallel_world_size())
        elif sp * tp > 1 and groups.ranks_of("dp") is None:
            groups.initialize(tp_size=tp, sp_size=sp)
        self.seq_parallel_group = groups._get_sequence_parallel_group() if sp > 1 else None
        self.sequence_parallel_size = sp
        self.data_parallel_group = groups._get_data_parallel_group()
        # ZeRO shards over seq x data when Ulysses is on (reference engine.py:1655)
        self.seq_data_parallel_group = groups._get_sequence_data_parallel_group() if sp > 1 else self.data_parallel_group
        self.dp_world_size = groups._get_data_parallel_world_size()
        self.seq_dp_world_size = groups._get_sequence_data_parallel_world_size() if sp > 1 else self.dp_world_size
        self.mp_world_size = groups._get_model_parallel_world_size()

    def _model_dtype(self):
        if self._config.fp16_enabled:
            return torch.float16
        if self._config.bfloat16_enabled:
            return torch.bfloat16
        return torch.float32

    def get_data_types(self):
        model_dtype = self._model_dtype()
        gad = self._config.grad_accum_dtype
        if gad is None:
            grad_accum_dtype = torch.float32 if (model_dtype == torch.bfloat16
                                                 and not self.zero_optimization()) else model_dtype
        else:
            grad_accum_dtype = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}[gad]
        return model_dtype, grad_accum_dtype

    def _configure_distributed_model(self, model):
        dtype = self._model_dtype()
        from deepspeed_b200.runtime.zero.partition_parameters import is_zero_param
        sharded_already = any(is_zero_param(p) for p in model.parameters())
        if not sharded_already:
            if dtype != torch.float32 and not self._config.amp_enabled:
                model.to(dtype)
            if not self.dont_change_device:
                model.to(self.device)
        # embedding tables whose gradients the user asked to treat as sparse (reference engine.py:333); gradients are
        # densified into the unit's flat buffer before the reduce-scatter here, the set is kept for checkpoint parity
        self.sparse_tensor_module_names = set()
        if self._config.sparse_gradients_enabled:
            for name, sub in model.named_modules():
                if isinstance(sub, (nn.Embedding, nn.EmbeddingBag)):
                    self.sparse_tensor_module_names.add(name + ".weight")
        # MoE discovery: create expert groups before the optimizer partitions parameters
        self.has_moe_layers = False
        self.num_experts = []
        try:
            from deepspeed_b200.moe.layer import MoE
            for m in model.modules():
                if isinstance(m, MoE):
                    self.has_moe_layers = True
                    self.num_experts.append(m.num_experts)
                    m.set_deepspeed_parallelism(self._config.use_data_before_expert_parallel_)
        except ImportError:
            pass

    def _build_loss_scale_config(self):
        c = self._config
        if not c.fp16_enabled:
            return {"dynamic": False, "static_loss_scale": 1.0}
        if c.loss_scale == 0:
            return {"dynamic": True, "dynamic_args": c.dynamic_loss_scale_args}
        return {"dynamic": False, "static_loss_scale": c.loss_scale}

    def _configure_optimizer(self, client_optimizer, model_parameters):
        c = self._config
        name = c.optimizer_name
        opt_params = c.optimizer_params or {}
        param_groups = None
        if client_optimizer is not None and not isinstance(client_optimizer, torch.optim.Optimizer):
            if callable(client_optimizer):  # optimizer factory callable (reference DeepSpeedOptimizerCallable)
                client_optimizer = client_optimizer(model_parameters)
            else:
                raise TypeError("optimizer must be a torch.optim.Optimizer or a callable returning one")
        if client_optimizer is None:
            if name in (ONEBIT_ADAM_OPTIMIZER, ZERO_ONE_ADAM_OPTIMIZER, ONEBIT_LAMB_OPTIMIZER):
                from deepspeed_b200.runtime.fp16.onebit import build_onebit_optimizer
                client_optimizer = build_onebit_optimizer(name, model_parameters, opt_params, self)
                name = None
            elif name not in (ADAM_OPTIMIZER, ADAMW_OPTIMIZER, LION_OPTIMIZER, ADAGRAD_OPTIMIZER, SGD_OPTIMIZER,
                              LAMB_OPTIMIZER, "muadam", "muadamw", "musgd"):
                # any torch.optim class by name
                cls = getattr(torch.optim, name, None)
                if cls is None:
                    raise ValueError(f"unknown optimizer type {name!r}")
                client_optimizer = cls(model_parameters, **opt_params)
                name = None
            else:
                pl = list(model_parameters)
                param_groups = pl if (pl and isinstance(pl[0], dict)) else [{"params": pl}]
        self.basic_optimizer = client_optimizer
        model_dtype, gad = self.get_data_types()
        stage = self.zero_optimization_stage()
        if stage == 0:
            # the reference's wrapper table (engine.py:1301 _do_optimizer_sanity_check): without ZeRO only these
            # (model dtype, gradient-accumulation dtype) pairs exist -- fp32/fp32, fp16/fp16, bf16/fp32 (bf16/bf16 under
            # pipeline parallelism), amp on fp32 -- anything else is refused instead of silently losing precision
            if self._config.amp_enabled:
                if model_dtype != gad:
                    raise NotImplementedError("Model data type and gradient accumulation data type must be equal to use Amp")
                if model_dtype in (torch.bfloat16, torch.float16):
                    raise NotImplementedError("Cannot enable both amp with (legacy) fp16 or bfloat16 mode")
            elif model_dtype == gad:
                if model_dtype == torch.bfloat16 and not getattr(self, "pipeline_parallelism", False):
                    raise NotImplementedError("Bfloat16 wrapper must use a gradient accumulation type of fp32, enable ZeRO "
                                              "to use Bfloat16 gradient accumulation")
            elif not (model_dtype == torch.bfloat16 and gad == torch.float32):
                raise NotImplementedError("unsupported mix of model dtype and gradient accumulation type")
        if stage > 0 and client_optimizer is not None and not c.zero_allow_untested_optimizer:
            from deepspeed_b200.runtime.zero.utils import is_zero_supported_optimizer
            assert is_zero_supported_optimizer(client_optimizer), (
                f"{type(client_optimizer).__name__} is not a ZeRO-tested optimizer; set "
                f"'zero_allow_untested_optimizer': true to use it anyway")
        common = dict(client_optimizer=client_optimizer, optimizer_name=name, optimizer_params=opt_params,
                      param_groups=param_groups, zero_config=c.zero_config, model_dtype=model_dtype, grad_accum_dtype=gad,
                      gradient_accumulation_steps=self.gradient_accumulation_steps(),
                      gradient_clipping=self.gradient_clipping(), loss_scale_config=self._build_loss_scale_config(),
                      communication_data_type=c.communication_data_type, prescale_gradients=c.prescale_gradients,
                      gradient_predivide_factor=c.gradient_predivide_factor, device=self.device, mpu=self.mpu,
                      timers=self.timers, aio_config=getattr(c, "aio_config", None))
        expert_names = sorted({getattr(p, "group_name", None) for p in self.module.parameters()
                               if getattr(p, "allreduce", True) is False} - {None})
        if not expert_names:
            mics = int(getattr(c.zero_config, "mics_shard_size", -1) or -1)
            if mics > 0 and stage == 3 and mics < dist.get_world_size(self.seq_data_parallel_group):
                from deepspeed_b200.runtime.zero.mics import create_mics_comm_groups
                mg = create_mics_comm_groups(mics, self.seq_data_parallel_group,
                                             hierarchical_allgather=bool(c.zero_config.mics_hierarchical_params_gather))
                self.optimizer = ZeroShardedOptimizer(self.module, stage, dp_group=mg.param_shard_group,
                                                      replica_group=mg.param_repli_group, **common)
                self.optimizer.mics_groups = mg  # two-hop parameter gathers when the shard group spans nodes
                self.optimizer.grad_allreduce_enabled = self._dense_grad_allreduce_enabled
                return
            oo = c.zero_config.offload_optimizer
            ratio = float(getattr(oo, "ratio", 1.0)) if oo is not None else 1.0
            if oo is not None and str(getattr(oo.device, "value", oo.device)) == "cpu" and 0.0 < ratio < 1.0 and stage == 3:
                self.optimizer = self._build_twin_flow(stage, common, ratio)
                return
            self.optimizer = ZeroShardedOptimizer(self.module, stage, dp_group=self.seq_data_parallel_group, **common)
            from deepspeed_b200.runtime.zero.sharded import tag_reference_class
            tag_reference_class(self.optimizer)
            self.optimizer.grad_allreduce_enabled = self._dense_grad_allreduce_enabled
            return
        # MoE: dense parameters over the DP group, every expert family over its expert-data-parallel group
        from deepspeed_b200.runtime.zero.multi import ZeroOptimizerGroup
        assert client_optimizer is None or not isinstance(client_optimizer, torch.optim.Optimizer) or True
        parts, ep_groups = [], []
        parts.append(ZeroShardedOptimizer(self.module, stage, dp_group=self.seq_data_parallel_group, name="dense",
                                          param_filter=lambda p: getattr(p, "allreduce", True) is not False, **common))
        ep_groups.append(None)
        for en in expert_names:
            edp = groups._get_expert_data_parallel_group(en)
            parts.append(ZeroShardedOptimizer(self.module, stage, dp_group=edp, name=f"expert:{en}",
                                              param_filter=lambda p, en=en: getattr(p, "group_name", None) == en and
                                              getattr(p, "allreduce", True) is False, **common))
            ep_groups.append(groups._get_expert_parallel_group(en))
        self.optimizer = ZeroOptimizerGroup(parts, ep_groups)

    def _build_twin_flow(self, stage, common, ratio):
        """ZeRO-Offload++ "Twin-Flow" (``offload_optimizer.ratio`` < 1, reference ``stage3.py:854-856``): the optimizer
        state of the first ``ratio`` of the parameters lives on the host and is stepped by the CPU optimizer, the rest
        stays in HBM and is stepped by the fused GPU kernel.  Two sharded-state domains behind one optimizer facade: the
        GPU domain keeps every fast path (fused reduce-scatter + Adam inside backward), the host domain streams its
        gradients out / parameters in on side streams meanwhile."""
        import copy as _copy
        from deepspeed_b200.runtime.zero.multi import ZeroOptimizerGroup
        params = [p for p in self.module.parameters()]
        total = sum(int(getattr(p, "ds_numel", p.numel())) for p in params)
        host_ids, acc = set(), 0
        for p in params:
            if acc >= ratio * total:
                break
            host_ids.add(id(p))
            acc += int(getattr(p, "ds_numel", p.numel()))
        zc_gpu = _copy.deepcopy(common["zero_config"])
        zc_gpu.__dict__["offload_optimizer"] = None
        host = ZeroShardedOptimizer(self.module, stage, dp_group=self.seq_data_parallel_group, name="twinflow:host",
                                    param_filter=lambda p: id(p) in host_ids, **common)
        gpu_common = dict(common, zero_config=zc_gpu)
        dev = ZeroShardedOptimizer(self.module, stage, dp_group=self.seq_data_parallel_group, name="twinflow:device",
                                   param_filter=lambda p: id(p) not in host_ids, **gpu_common)
        for part in (host, dev):
            part.grad_allreduce_enabled = self._dense_grad_allreduce_enabled
        log_dist(f"Twin-Flow offload: {acc / max(total, 1):.1%} of {total:,} parameters stepped on the host, the rest on "
                 f"the device", ranks=[0])
        return ZeroOptimizerGroup([host, dev], [None, None])

    def _configure_zero_inference(self):
        self.optimizer = ZeroShardedOptimizer(self.module, 3, optimizer_name="sgd", optimizer_params={"lr": 0.0},
                                              param_groups=[{"params": []}], zero_config=self._config.zero_config,
                                              dp_group=self.seq_data_parallel_group, model_dtype=self._model_dtype(),
                                              device=self.device)
        self._zero_inference = True

    def _configure_lr_scheduler(self, client_lr_scheduler):
        c = self._config
        if client_lr_scheduler is not None:
            if callable(client_lr_scheduler) and not hasattr(client_lr_scheduler, "step"):
                self.lr_scheduler = self._build_scheduler_on_our_groups(client_lr_scheduler)
            else:
                self.lr_scheduler = client_lr_scheduler
                # a client scheduler built on the client optimizer must drive OUR param groups
                if hasattr(self.lr_scheduler, "optimizer") and self.lr_scheduler.optimizer is self.client_optimizer:
                    self.lr_scheduler.optimizer = self.optimizer
        elif c.scheduler_name is not None:
            cls = lr_schedules.get_lr_schedule_class(c.scheduler_name)
            if cls is None:
                cls = getattr(torch.optim.lr_scheduler, c.scheduler_name, None)
                assert cls is not None, f"DeepSpeed does not recognize LR scheduler {c.scheduler_name}"
            self.lr_scheduler = self._build_scheduler_on_our_groups(lambda o: cls(o, **(c.scheduler_params or {})))
        log_dist(f"DeepSpeed LR Scheduler = {type(self.lr_scheduler).__name__ if self.lr_scheduler else None}",
                 ranks=[0])

    def _build_scheduler_on_our_groups(self, factory):
        """``factory(optimizer) -> scheduler``.  Framework schedulers accept the engine's optimizer as it is; ``torch.optim``
        schedulers insist on a ``torch.optim.Optimizer`` instance (the reference hands them its basic optimizer,
        ``engine.py:985``): build them on a stand-in with the same groups / learning rates, then point them at the real
        parameter groups so every ``scheduler.step()`` drives the optimizer that actually steps."""
        try:
            return factory(self.optimizer)
        except TypeError:
            pass
        groups = self.optimizer.param_groups
        stand_in = torch.optim.SGD([{"params": [torch.nn.Parameter(torch.zeros(1))], "lr": float(g.get("lr", 1e-3))}
                                    for g in groups], lr=1e-3)
        sched = factory(stand_in)
        for g, sg in zip(groups, stand_in.param_groups):
            g["lr"] = sg["lr"]
            if "initial_lr" in sg:
                g["initial_lr"] = sg["initial_lr"]
        sched.optimizer = self.optimizer
        return sched

    def _dense_grad_allreduce_enabled(self):
        # the pipeline engine keeps its own switch (1-bit optimizers toggle whichever applies)
        if hasattr(self, "pipeline_enable_backward_allreduce"):
            return self.pipeline_enable_backward_allreduce
        return self.enable_backward_allreduce

    def _autotuning_setup(self):
        """Autotuning experiments run the user script unchanged; the engine measures and exits
        (reference ``engine.py`` autotuning hooks: model-info dump, ``metric_path`` write, early exit)."""
        at = self._config.autotuning_config or {}
        self._at = at if at.get("enabled") else None
        if not self._at:
            return
        import json
        info = {"num_params": sum(getattr(p, "ds_numel", p.numel()) for p in self.module.parameters()),
                "trainable_num_params": sum(getattr(p, "ds_numel", p.numel()) for p in self.module.parameters()
                                            if p.requires_grad)}
        if self.global_rank == 0 and at.get("model_info_path"):
            with open(at["model_info_path"], "w") as f:
                json.dump(info, f)
        if (at.get("model_info") or {}).get("profile"):
            dist.barrier()
            raise SystemExit(0)
        self._at_t0 = None

    def _autotuning_step(self):
        at = self._at
        if not at:
            return
        import json
        import time
        start, end = int(at.get("start_profile_step", 3)), int(at.get("end_profile_step", 5))
        if self.global_steps == start:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            self._at_t0 = time.time()
        elif self.global_steps >= end and self._at_t0 is not None:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            dt = (time.time() - self._at_t0) / max(1, end - start)
            m = {"latency": dt * 1e3, "throughput": self.train_batch_size() / dt, "flops": 0.0,
                 "max_mem_gb": (torch.cuda.max_memory_allocated() / 2**30) if torch.cuda.is_available() else 0.0}
            if self.global_rank == 0 and at.get("metric_path"):
                with open(at["metric_path"], "w") as f:
                    json.dump(m, f)
            dist.barrier()
            raise SystemExit(0)

    def _configure_aux(self):
        c = self._config
        self._autotuning_setup()
        self.flops_profiler = None
        if c.flops_profiler_config.enabled:
            from deepspeed_b200.profiling.flops_profiler import FlopsProfiler
            self.flops_profiler = FlopsProfiler(self.module, self)
        self.progressive_layer_drop = None
        if c.pld_enabled:
            from deepspeed_b200.runtime.progressive_layer_drop import ProgressiveLayerDrop
            self.progressive_layer_drop = ProgressiveLayerDrop(theta=c.pld_params.get("theta", 0.5),
                                                               gamma=c.pld_params.get("gamma", 0.001))
        self.random_ltd_scheduler = None
        self.compression_scheduler = None
        self.data_post_process_func = None
        de = c.data_efficiency_config if c.data_efficiency_enabled else None
        if de:
            from deepspeed_b200.runtime.data_pipeline.config import get_data_efficiency_config
            from deepspeed_b200.runtime.data_pipeline import constants as DC
            self._de = get_data_efficiency_config({"data_efficiency": de})
            ltd = self._de[DC.DATA_ROUTING][DC.RANDOM_LTD]
            if self._de[DC.DATA_ROUTING][DC.DATA_ROUTING_ENABLED] and ltd.get(DC.RANDOM_LTD_ENABLED):
                from deepspeed_b200.runtime.data_pipeline.data_routing import RandomLayerTokenDrop, RandomLTDScheduler
                ltd = dict(ltd)
                ltd.setdefault(DC.RANDOM_LTD_GLOBAL_BATCH_SIZE, self.train_batch_size())
                ltd.setdefault(DC.RANDOM_LTD_MICRO_BATCH_SIZE, self.train_micro_batch_size_per_gpu())
                self.random_ltd_scheduler = RandomLTDScheduler(ltd)
                lid = 0
                for m in self.module.modules():
                    if isinstance(m, RandomLayerTokenDrop):
                        m.init_config(ltd, self.random_ltd_scheduler, lid)
                        lid += 1
        else:
            self._de = None
        if (c._param_dict.get("compression_training") or {}):
            from deepspeed_b200.compression import compression_scheduler
            from deepspeed_b200.compression.config import get_compression_config
            cc = get_compression_config(c._param_dict)
            if any(cc[t]["shared_parameters"]["enabled"] for t in cc if t != "layer_reduction"):
                self.compression_scheduler = compression_scheduler(self.module, cc)
                self.compression_scheduler.step(step_zero_check=True)
        self.curriculum_scheduler_legacy = None
        if c.curriculum_enabled_legacy:
            from deepspeed_b200.runtime.data_pipeline.curriculum_scheduler import CurriculumScheduler
            self.curriculum_scheduler_legacy = CurriculumScheduler(c.curriculum_params_legacy)
        self.eigenvalue = None
        if c.eigenvalue_enabled:
            from deepspeed_b200.runtime.eigenvalue import Eigenvalue
            self.eigenvalue = Eigenvalue(verbose=c.eigenvalue_verbose, max_iter=c.eigenvalue_max_iter,
                                         tol=c.eigenvalue_tol, stability=c.eigenvalue_stability,
                                         gas_boundary_resolution=c.eigenvalue_gas_boundary_resolution,
                                         layer_name=c.eigenvalue_layer_name, layer_num=c.eigenvalue_layer_num)
        self.quantizer = None
        self._configure_checkpointing()

    # =========================================================================================
    # accessors (reference names)
    # =========================================================================================
    def train_batch_size(self):
        return self._config.train_batch_size

    def train_micro_batch_size_per_gpu(self):
        return self._config.train_micro_batch_size_per_gpu

    def gradient_accumulation_steps(self):
        return self._config.gradient_accumulation_steps

    def set_train_batch_size(self, train_batch_size):
        mb = self.train_micro_batch_size_per_gpu() * self.dp_world_size
        if train_batch_size % mb != 0:
            raise ValueError("Train batch size must be divisible by micro-batch data parallelism")
        self._config.gradient_accumulation_steps = train_batch_size // mb
        self._config.train_batch_size = train_batch_size
        if self.optimizer is not None:
            if hasattr(self.optimizer, "set_gradient_accumulation_steps"):
                # re-evaluates the fused-in-backward policy (a gradient arena is needed once GAS > 1)
                self.optimizer.set_gradient_accumulation_steps(self._config.gradient_accumulation_steps)
            else:
                self.optimizer.gas = self._config.gradient_accumulation_steps

    def set_train_micro_batch_size(self, micro_batch_size):
        self._config.train_batch_size = micro_batch_size * self.gradient_accumulation_steps() * self.dp_world_size
        self._config.train_micro_batch_size_per_gpu = micro_batch_size

    def steps_per_print(self):
        return self._config.steps_per_print

    def wall_clock_breakdown(self):
        return self._config.wall_clock_breakdown

    def memory_breakdown(self):
        return self._config.memory_breakdown

    def gradient_clipping(self):
        return self._config.gradient_clipping

    def zero_optimization(self):
        return self._config.zero_enabled

    def zero_optimization_stage(self):
        return self._config.zero_optimization_stage

    def zero_optimization_partition_gradients(self):
        return self.zero_optimization_stage() >= 2

    def zero_optimization_partition_weights(self):
        return self.zero_optimization_stage() >= 3

    def fp16_enabled(self):
        return self._config.fp16_enabled

    def bfloat16_enabled(self):
        return self._config.bfloat16_enabled

    def amp_enabled(self):
        return self._config.amp_enabled

    def dynamic_loss_scale(self):
        return self._config.fp16_enabled and self._config.loss_scale == 0

    def loss_scale(self):
        return self._config.loss_scale

    def optimizer_name(self):
        return self.client_optimizer.__class__.__name__ if self.client_optimizer else self._config.optimizer_name

    def scheduler_name(self):
        return self._config.scheduler_name

    def get_lr(self):
        return [g["lr"] for g in self.optimizer.param_groups]

    def get_type(self):
        return [g.get("type", None) for g in self.optimizer.param_groups]

    def get_mom(self):
        return [g.get("betas", g.get("momentum")) for g in self.optimizer.param_groups]

    def get_global_grad_norm(self):
        return self.optimizer.get_global_grad_norm() if self.optimizer is not None else None

    @property
    def config(self):
        return self._config._param_dict

    def get_batch_info(self):
        return self.train_batch_size(), self.train_micro_batch_size_per_gpu(), self.gradient_accumulation_steps()

    def is_first_weights_partition_group(self):
        return self.global_rank == 0 or self.zero_optimization_stage() >= 1

    def was_step_applied(self) -> bool:
        return self._step_applied

    # =========================================================================================
    # data
    # =========================================================================================
    def deepspeed_io(self, dataset, batch_size=None, route="train", pin_memory=True, data_sampler=None,
                     collate_fn=None, num_local_io_workers=None):
        if not isinstance(dataset, torch.utils.data.Dataset):
            raise ValueError("Training data must be a torch Dataset")
        if batch_size is None:
            batch_size = self.train_micro_batch_size_per_gpu()
        if collate_fn is None:
            collate_fn = self.collate_fn
        if data_sampler is None and route == "train" and getattr(self, "_de", None):
            from deepspeed_b200.runtime.data_pipeline import constants as DC
            ds_cfg = self._de[DC.DATA_SAMPLING]
            if ds_cfg.get(DC.DATA_SAMPLING_ENABLED):
                from deepspeed_b200.runtime.data_pipeline.data_sampling import DeepSpeedDataSampler
                data_sampler = DeepSpeedDataSampler(self._de, len(dataset), self.train_micro_batch_size_per_gpu(),
                                                    groups._get_data_parallel_rank(), self.dp_world_size,
                                                    self.seq_data_parallel_group, self.gradient_accumulation_steps(),
                                                    self.global_rank, drop_last=self._config.dataloader_drop_last)
        return DeepSpeedDataLoader(dataset=dataset, batch_size=batch_size, pin_memory=pin_memory,
                                   collate_fn=collate_fn, local_rank=self.local_rank, tput_timer=self.tput_timer,
                                   num_local_io_workers=num_local_io_workers, data_sampler=data_sampler,
                                   data_parallel_world_size=self.dp_world_size,
                                   data_parallel_rank=groups._get_data_parallel_rank(),
                                   dataloader_drop_last=self._config.dataloader_drop_last)

    # =========================================================================================
    # train / eval
    # =========================================================================================
    def train(self, mode=True):
        self.warn_unscaled_loss = True
        self.module.train(mode)
        return self

    def eval(self):
        self.warn_unscaled_loss = True
        self.module.train(False)
        return self

    def _cast_inputs(self, args, kwargs):
        if not (self._config.fp16_auto_cast and self.fp16_enabled()):
            return args, kwargs

        def cast(x):
            return x.half() if torch.is_tensor(x) and torch.is_floating_point(x) else x

        return tuple(cast(a) for a in args), {k: cast(v) for k, v in kwargs.items()}

    @instrument_w_nvtx
    def __getattr__(self, name):
        """Attributes the engine does not define fall through to the wrapped client module (``engine.config``,
        ``engine.generate`` ... on a wrapped HF model). Reference: runtime/engine.py:573."""
        try:
            return super().__getattr__(name)
        except AttributeError:
            mod = self.__dict__.get("_modules", {}).get("module")
            if mod is not None and name != "module":
                try:
                    return getattr(mod, name)
                except AttributeError:
                    pass
            raise AttributeError(f"'{type(self).__name__}' object has no attribute '{name}'") from None

    def forward(self, *inputs, **kwargs):
        if self.flops_profiler is not None and self.global_steps == self._config.flops_profiler_config.profile_step \
                and self.global_rank == 0 and self.module.training:
            self.flops_profiler.start_profile(ignore_list=None)
        if self.module.training:
            if self.progressive_layer_drop is not None:
                kwargs.update(self.progressive_layer_drop.get_state())
            if self.curriculum_scheduler_legacy is not None:
                self.curriculum_scheduler_legacy.update_difficulty(self.global_steps + 1)
                if self._config.curriculum_params_legacy.get("curriculum_type") == "seqlen":
                    kwargs["curriculum_seqlen"] = self.curriculum_scheduler_legacy.get_current_difficulty()
        self.timers(FORWARD_MICRO_TIMER).start()
        self.timers(FORWARD_GLOBAL_TIMER).start()
        if self.module.training:
            self.tput_timer.start()
        inputs, kwargs = self._cast_inputs(inputs, kwargs)
        if self.optimizer is not None and hasattr(self.module, "ds_loss_multiplier"):
            # lets fused loss heads fold the upcoming backward scale into their in-forward gradients
            gas = self.gradient_accumulation_steps()
            self.module.ds_loss_multiplier = float(self.optimizer.loss_scale) / (gas if gas > 1 else 1)
        loss = self.module(*inputs, **kwargs)
        self.timers(FORWARD_MICRO_TIMER).stop()
        self.timers(FORWARD_GLOBAL_TIMER).stop()
        if self.flops_profiler is not None and self.flops_profiler.started:
            self.flops_profiler.stop_profile()
        return loss

    __call__ = nn.Module.__call__

    def is_gradient_accumulation_boundary(self):
        if self._is_gradient_accumulation_boundary is None:
            return (self.micro_steps + 1) % self.gradient_accumulation_steps() == 0
        return self._is_gradient_accumulation_boundary

    def set_gradient_accumulation_boundary(self, is_boundary):
        self._is_gradient_accumulation_boundary = is_boundary
        if self.optimizer is not None:
            if hasattr(self.optimizer, "set_forced_boundary"):
                self.optimizer.set_forced_boundary(is_boundary)
            else:
                self.optimizer._forced_boundary = is_boundary

    @contextlib.contextmanager
    def no_sync(self):
        """Skip gradient reduction inside the context (reference engine.py:2065); illegal with
        ZeRO >= 2 because gradients are partitioned as they are produced."""
        assert not self.zero_optimization_partition_gradients(), \
            f"no_sync context manager is incompatible with gradient partitioning logic of ZeRO stage " \
            f"{self.zero_optimization_stage()}"
        assert not getattr(self, "inside_no_sync_ctxt", False), "no_sync context manager reentry is unsupported"
        self.inside_no_sync_ctxt = True
        if hasattr(self.optimizer, "set_no_sync"):
            self.optimizer.set_no_sync(True)
        try:
            yield
        finally:
            self.inside_no_sync_ctxt = False
            if hasattr(self.optimizer, "set_no_sync"):
                self.optimizer.set_no_sync(False)

    @instrument_w_nvtx
    def backward(self, loss, retain_graph=False, scale_wrt_gas=True):
        assert self.optimizer is not None, "must provide optimizer during init in order to use backward"
        self.timers(BACKWARD_MICRO_TIMER).start()
        self.timers(BACKWARD_GLOBAL_TIMER).start()
        gas = self.gradient_accumulation_steps()
        if gas > 1 and scale_wrt_gas and not getattr(self, "inside_no_sync_ctxt", False):
            loss = loss.float() / gas  # (fp32: the reference scales `loss.float()`, engine.py:2102)
        if self.monitor.enabled and self.is_gradient_accumulation_boundary():
            self._last_loss_for_monitor = loss.detach()
        self.optimizer.backward(loss, retain_graph=retain_graph)
        self.timers(BACKWARD_MICRO_TIMER).stop()
        self.timers(BACKWARD_GLOBAL_TIMER).stop()
        return loss

    def zero_grad(self):
        for p in self.module.parameters():
            p.grad = None
        if self.optimizer is not None and hasattr(self.optimizer, "zero_grad"):
            self.optimizer.zero_grad()  # also drops gradients parked by no_sync()

    def clip_fp32_gradients(self):
        pass  # clipping is fused into the sharded optimizer step

    def _take_model_step(self, lr_kwargs=None):
        pruners = getattr(self.module, "pruners", None) or ()  # SNIP-momentum sparse pruning (compression.helper)
        for pr in pruners:
            pr.on_before_optimizer_step()
        self.optimizer.step()
        for pr in pruners:
            pr.on_after_optimizer_step()
        overflow = getattr(self.optimizer, "overflow", False)
        self._step_applied = not overflow
        if overflow:
            self.skipped_steps += 1
        elif self.lr_scheduler is not None:
            try:
                self.lr_scheduler.step(**(lr_kwargs or {}))
            except TypeError:
                self.lr_scheduler.step()
        self.global_steps += 1
        self.global_samples += self.train_batch_size()

    @instrument_w_nvtx
    def step(self, lr_kwargs=None):
        assert self.optimizer is not None, "must provide optimizer during init in order to use step"
        assert not getattr(self, "inside_no_sync_ctxt", False), \
            "It is illegal to call Engine.step() inside no_sync context manager"
        self.timers(STEP_MICRO_TIMER).start()
        self.timers(STEP_GLOBAL_TIMER).start()
        self._step_applied = False
        boundary = self.is_gradient_accumulation_boundary()
        if boundary:
            if self.progressive_layer_drop is not None:
                self.progressive_layer_drop.update_state(self.global_steps)
            self._take_model_step(lr_kwargs)
            if self.random_ltd_scheduler is not None:
                self.random_ltd_scheduler.update_seq(self.global_steps)
            if self.compression_scheduler is not None:
                self.compression_scheduler.step()
            if self.monitor.enabled and self.global_rank == 0:
                ev = [("Train/Samples/lr", self.get_lr()[0], self.global_samples)]
                if getattr(self, "_last_loss_for_monitor", None) is not None:
                    ev.append(("Train/Samples/train_loss", float(self._last_loss_for_monitor), self.global_samples))
                if self.fp16_enabled():
                    ev.append(("Train/Samples/loss_scale", self.optimizer.cur_scale, self.global_samples))
                self.monitor.write_events(ev)
        self.tput_timer.stop(global_step=boundary)
        self.timers(STEP_MICRO_TIMER).stop()
        self.timers(STEP_GLOBAL_TIMER).stop()
        if boundary and getattr(self, "_at", None):
            self._autotuning_step()
        if boundary and self.wall_clock_breakdown() and self.global_steps % self.steps_per_print() == 0:
            self.timers.log([FORWARD_GLOBAL_TIMER, BACKWARD_GLOBAL_TIMER, STEP_GLOBAL_TIMER],
                            memory_breakdown=self.memory_breakdown())
        if boundary and self.flops_profiler is not None and self.flops_profiler.has_result() and \
                self.global_steps == self._config.flops_profiler_config.profile_step + 1:
            fc = self._config.flops_profiler_config
            self.flops_profiler.print_model_profile(profile_step=fc.profile_step, module_depth=fc.module_depth,
                                                    top_modules=fc.top_modules, detailed=fc.detailed,
                                                    output_file=fc.output_file)
            self.flops_profiler.end_profile()
        if boundary and self.global_steps % self.steps_per_print() == 0:
            self._report_progress(self.global_steps)
        self.micro_steps += 1

    def _report_progress(self, step):
        lr = self.get_lr()
        log_dist(f"step={step}, skipped={self.skipped_steps}, lr={lr}, mom={self.get_mom()}", ranks=[0])

    # ---- convenience: one full optimizer step over GAS micro-batches -----------------------------
    def train_batch(self, data_iter=None, loss_fn=None):
        """Run forward/backward for ``gradient_accumulation_steps`` micro batches and step.
        (For non-pipeline engines; mirrors ``PipelineEngine.train_batch`` ergonomics.)"""
        if data_iter is None:
            assert self.training_dataloader is not None
            if not hasattr(self, "_train_iter"):
                from deepspeed_b200.runtime.dataloader import RepeatingLoader
                self._train_iter = iter(RepeatingLoader(self.training_dataloader))
            data_iter = self._train_iter
        total = None
        for _ in range(self.gradient_accumulation_steps()):
            batch = next(data_iter)
            batch = _to_device(batch, self.device)
            if isinstance(batch, dict):
                out = self(**batch)
            elif isinstance(batch, (tuple, list)):
                out = self(*batch)
            else:
                out = self(batch)
            loss = loss_fn(out, batch) if loss_fn is not None else (out[0] if isinstance(out, (tuple, list)) else
                                                                    getattr(out, "loss", out))
            self.backward(loss)
            self.step()
            total = loss.detach() if total is None else total + loss.detach()
        return total / self.gradient_accumulation_steps()

    # ---- misc reference API ------------------------------------------------------------------------
    def module_state_dict(self, destination=None, prefix="", keep_vars=False, exclude_frozen_parameters=False):
        sd = self.module.state_dict(destination=destination, prefix=prefix, keep_vars=keep_vars)
        if exclude_frozen_parameters:
            for n, p in self.module.named_parameters():
                if not p.requires_grad and n in sd:
                    del sd[n]
        return sd

    def load_module_state_dict(self, checkpoint, strict=True, custom_load_fn=None, fetch_z3_params=False):
        sd = checkpoint["module"] if "module" in checkpoint else checkpoint
        if custom_load_fn:
            custom_load_fn(src=sd, dst=self.module)
        else:
            self.module.load_state_dict(sd, strict=strict)

    def get_sequence_parallel_group(self):
        return self.seq_parallel_group

    # ---- reference API surface kept for drop-in compatibility ------------------------------------------------
    def allreduce_gradients(self, bucket_size=None):
        """Gradients are reduced unit-by-unit inside backward by the sharded optimizer; an explicit call only has
        to drain the reduction stream (reference ``engine.py:2048``)."""
        if self.optimizer is not None and getattr(self.optimizer, "rs_stream", None) is not None:
            torch.cuda.current_stream().wait_stream(self.optimizer.rs_stream)

    def allreduce_bucket(self, bucket, dp_group=None, dp_world_size=None):
        """Average one list of same-dtype tensors over the DP group with a single flattened collective."""
        from deepspeed_b200.ops.flatten import flatten, unflatten
        group = dp_group or self.seq_data_parallel_group
        world = dp_world_size or dist.get_world_size(group)
        flat = flatten(bucket)
        if self._config.prescale_gradients and self._config.gradient_predivide_factor != 1.0:
            flat.mul_(1.0 / self._config.gradient_predivide_factor)
            dist.all_reduce(flat, group=group)
            flat.mul_(self._config.gradient_predivide_factor / world)
        else:
            dist.all_reduce(flat, group=group)
            flat.mul_(1.0 / world)
        return flat

    def allreduce_and_copy(self, small_bucket, dp_group=None, dp_world_size=None):
        from deepspeed_b200.ops.flatten import unflatten
        flat = self.allreduce_bucket(small_bucket, dp_group, dp_world_size)
        for buf, synced in zip(small_bucket, unflatten(flat, small_bucket)):
            buf.copy_(synced)

    def buffered_allreduce_fallback(self, grads=None, elements_per_buffer=500000000):
        """Explicit DP all-reduce of ``.grad`` tensors in dtype-homogeneous buckets (reference ``engine.py:2611``); only
        needed for parameters that are not managed by the sharded optimizer (it reduces its own)."""
        if grads is None:
            grads = [p.grad for p in self.module.parameters() if p.grad is not None and not hasattr(p, "_ds_zero")]
        by_dtype = {}
        for g in grads:
            by_dtype.setdefault(g.dtype, []).append(g)
        for gs in by_dtype.values():
            bucket, n = [], 0
            for g in gs:
                if n + g.numel() > elements_per_buffer and bucket:
                    self.allreduce_and_copy(bucket)
                    bucket, n = [], 0
                bucket.append(g)
                n += g.numel()
            if bucket:
                self.allreduce_and_copy(bucket)

    def sparse_allreduce(self, sparse_tensor, dp_group=None, dp_world_size=None):
        from deepspeed_b200.runtime.sparse_tensor import sparse_allreduce
        return sparse_allreduce(sparse_tensor, dp_group or self.seq_data_parallel_group)

    def set_custom_curriculum_learning_schedule(self, schedule_func_dict):
        if self.training_dataloader is not None and getattr(self.training_dataloader, "data_sampler", None) is not None \
                and hasattr(self.training_dataloader.data_sampler, "set_custom_curriculum_learning_schedule"):
            self.training_dataloader.data_sampler.set_custom_curriculum_learning_schedule(schedule_func_dict)
        elif self.curriculum_scheduler_legacy is not None:
            fn = schedule_func_dict if callable(schedule_func_dict) else next(iter(schedule_func_dict.values()))
            self.curriculum_scheduler_legacy.set_custom_get_difficulty(fn)

    def set_data_post_process_func(self, post_process_func):
        self.data_post_process_func = post_process_func
        if self.training_dataloader is not None:
            self.training_dataloader.post_process_func = post_process_func

    def get_data_parallel_rank(self):
        return groups._get_data_parallel_rank()

    def empty_partition_cache(self):
        """Release every transiently gathered ZeRO-3 unit (reference ``engine.py`` / ``stage3.py``)."""
        zo = self.optimizer
        if zo is not None and getattr(zo, "transient", False):
            for rt in zo.rts:
                zo.release_unit(rt)
        if torch.cuda.is_available():
            torch.cuda.empty_cache()

    def dump_state(self):
        if self.global_rank != 0:
            return
        c = self._config
        for k in ("train_batch_size", "train_micro_batch_size_per_gpu", "gradient_accumulation_steps", "zero_config",
                  "optimizer_name", "optimizer_params", "scheduler_name", "bfloat16_enabled", "fp16_enabled",
                  "gradient_clipping"):
            logger.info(f"  {k} {'.' * (40 - len(k))} {getattr(c, k, None)}")

    def random_ltd_initialize(self):
        return self.random_ltd_scheduler

    def destroy(self):
        if self.optimizer is not None and hasattr(self.optimizer, "destroy"):
            self.optimizer.destroy()

    def offload_states(self, include=None, device="cpu", pin_memory=True, non_blocking=False):
        from deepspeed_b200.runtime.zero.offload_states import offload_states
        offload_states(self.optimizer, include, device, pin_memory, non_blocking)

    def reload_states(self, non_blocking=False):
        from deepspeed_b200.runtime.zero.offload_states import reload_states
        reload_states(self.optimizer, non_blocking)

    def compile(self, backend=None, compile_kwargs=None, schedule=None):
        """The reference wraps ``torch.compile``; on H100 the hot path is hand-written CUDA plus CUDA
        graphs, so this only records the request (kept for API compatibility)."""
        self._is_compiled = True
        log_dist("engine.compile(): no-op -- deepspeed_b200 uses native sm_90a kernels + CUDA graphs", ranks=[0])

    @property
    def is_compiled(self):
        return getattr(self, "_is_compiled", False)


def _to_device(batch, device):
    if torch.is_tensor(batch):
        return batch.to(device, non_blocking=True)
    if isinstance(batch, dict):
        return {k: _to_device(v, device) for k, v in batch.items()}
    if isinstance(batch, (list, tuple)):
        return type(batch)(_to_device(v, device) for v in batch)
    return batch
