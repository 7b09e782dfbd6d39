"""Top-level config: JSON / HJSON / dict / base64 -> typed ``DeepSpeedConfig``.

Parity target: reference ``runtime/config.py:707 DeepSpeedConfig`` (+ ``constants.py``).  All
reference top-level keys listed in SURVEY.md 5.6 are accepted.  Unlike the reference (which
mixes ``get_scalar_param`` getters with pydantic blocks), every block here is a pydantic model;
the flat attribute names the reference engine reads (``fp16_enabled``, ``zero_optimization_stage``,
``gradient_clipping`` ...) are exported as properties so ported user code keeps working.
"""
import base64
import copy
import json
import os
from typing import Any, Dict, List, Optional, Union

import hjson
from pydantic import Field

from deepspeed_b200.comm.config import CommsConfig
from deepspeed_b200.runtime.config_utils import (DeepSpeedConfigModel, ScientificNotationEncoder,
                                                 dict_raise_error_on_duplicate_keys)
from deepspeed_b200.runtime.zero.config import ZeroStageEnum, get_zero_config
from deepspeed_b200.utils.logging import logger

TORCH_ADAM_PARAM = "torch_adam"
ADAM_W_MODE = "adam_w_mode"
ADAM_W_MODE_DEFAULT = True

ADAGRAD_OPTIMIZER = "adagrad"
ADAM_OPTIMIZER = "adam"
ADAMW_OPTIMIZER = "adamw"
LAMB_OPTIMIZER = "lamb"
ONEBIT_ADAM_OPTIMIZER = "onebitadam"
ZERO_ONE_ADAM_OPTIMIZER = "zerooneadam"
ONEBIT_LAMB_OPTIMIZER = "onebitlamb"
MUADAM_OPTIMIZER = "muadam"
MUADAMW_OPTIMIZER = "muadamw"
MUSGD_OPTIMIZER = "musgd"
LION_OPTIMIZER = "lion"
SGD_OPTIMIZER = "sgd"
DEEPSPEED_OPTIMIZERS = [
    ADAGRAD_OPTIMIZER, ADAM_OPTIMIZER, ADAMW_OPTIMIZER, LAMB_OPTIMIZER, ONEBIT_ADAM_OPTIMIZER, ONEBIT_LAMB_OPTIMIZER,
    ZERO_ONE_ADAM_OPTIMIZER, MUADAM_OPTIMIZER, MUADAMW_OPTIMIZER, MUSGD_OPTIMIZER, LION_OPTIMIZER, SGD_OPTIMIZER
]

ROUTE_TRAIN = "train"
ROUTE_EVAL = "eval"
ROUTE_PREDICT = "predict"
ROUTE_ENCODE = "encode"


class DeepSpeedConfigError(Exception):
    pass


class DeepSpeedBatchConfigError(DeepSpeedConfigError, AssertionError):
    pass


# ------------------------------------------------------------------------------------------------
# blocks
# ------------------------------------------------------------------------------------------------
class FP16Config(DeepSpeedConfigModel):
    # the reference reads this block key by key (``config.py:181-260 get_fp16_*``): keys it does not know are ignored
    model_config = dict(DeepSpeedConfigModel.model_config, extra="allow")
    enabled: bool = False
    auto_cast: bool = False
    loss_scale: float = Field(0.0, ge=0)  # 0 == dynamic
    initial_scale_power: int = Field(16, ge=0)
    loss_scale_window: int = Field(1000, ge=0)
    hysteresis: int = Field(2, ge=0)
    consecutive_hysteresis: bool = False
    min_loss_scale: float = Field(1.0, ge=0)
    fp16_master_weights_and_grads: bool = False

    @property
    def dynamic_loss_scale(self):
        return self.loss_scale == 0


class BF16Config(DeepSpeedConfigModel):
    model_config = dict(DeepSpeedConfigModel.model_config, extra="allow")  # (same: ``config.py:166-180``)
    enabled: bool = False
    immediate_grad_update: bool = False
    check_grad_overflow: bool = False


class AMPConfig(DeepSpeedConfigModel):
    model_config = dict(DeepSpeedConfigModel.model_config, extra="allow")
    enabled: bool = False


class DataTypesConfig(DeepSpeedConfigModel):
    grad_accum_dtype: Optional[str] = None


class OptimizerConfig(DeepSpeedConfigModel):
    type: Optional[str] = None
    params: Dict[str, Any] = {}
    legacy_fusion: bool = False


class SchedulerConfig(DeepSpeedConfigModel):
    type: Optional[str] = None
    params: Dict[str, Any] = {}


class ActivationCheckpointingConfig(DeepSpeedConfigModel):
    # dict-read in the reference (activation_checkpointing/config.py:63): unknown keys are ignored there
    model_config = dict(DeepSpeedConfigModel.model_config, extra="allow")
    partition_activations: bool = False
    contiguous_memory_optimization: bool = False
    cpu_checkpointing: bool = False
    number_checkpoints: Optional[int] = None
    synchronize_checkpoint_boundary: bool = False
    profile: bool = False


class AIOConfig(DeepSpeedConfigModel):
    model_config = dict(DeepSpeedConfigModel.model_config, extra="allow")  # dict-read in the reference (swap_tensor/aio_config.py)
    block_size: int = 1048576
    queue_depth: int = 8
    intra_op_parallelism: int = Field(1, alias="thread_count")
    single_submit: bool = False
    overlap_events: bool = True
    use_gds: bool = False


class PipelineConfig(DeepSpeedConfigModel):
    stages: Union[str, int] = "auto"
    partition: str = "best"
    seed_layers: bool = False
    activation_checkpoint_interval: int = 0
    pipe_partitioned: bool = True
    grad_partitioned: bool = True
    use_reentrant: bool = True


class TensorParallelTPConfig(DeepSpeedConfigModel):
    tp_size: int = 1
    tp_grain_size: int = 1
    mpu: Any = None
    tp_group: Any = None


class TensorParallelConfig(DeepSpeedConfigModel):
    autotp_size: int = 0
    tp: TensorParallelTPConfig = TensorParallelTPConfig()
    tp_overlap_comm: bool = False
    injection_policy_tuple: Optional[tuple] = None
    keep_module_on_host: bool = False
    replace_with_kernel_inject: bool = False


class FlopsProfilerConfig(DeepSpeedConfigModel):
    enabled: bool = False
    recompute_fwd_factor: float = Field(0.0, ge=0.0)
    profile_step: int = Field(1, ge=1)
    module_depth: int = -1
    top_modules: int = 1
    detailed: bool = True
    output_file: Optional[str] = None


class TensorBoardConfig(DeepSpeedConfigModel):
    enabled: bool = False
    output_path: str = ""
    job_name: str = "DeepSpeedJobName"


class WandbConfig(DeepSpeedConfigModel):
    enabled: bool = False
    group: Optional[str] = None
    team: Optional[str] = None
    project: str = "deepspeed"


class CSVConfig(DeepSpeedConfigModel):
    enabled: bool = False
    output_path: str = ""
    job_name: str = "DeepSpeedJobName"


class CometConfig(DeepSpeedConfigModel):
    enabled: bool = False
    samples_log_interval: int = 100
    project: Optional[str] = None
    workspace: Optional[str] = None
    api_key: Optional[str] = None
    experiment_name: Optional[str] = None
    experiment_key: Optional[str] = None
    online: Optional[bool] = None
    mode: Optional[str] = None


class MonitorConfig:

    def __init__(self, d):
        self.tensorboard = TensorBoardConfig(**d.get("tensorboard", {}))
        self.wandb = WandbConfig(**d.get("wandb", {}))
        self.csv_monitor = CSVConfig(**d.get("csv_monitor", {}))
        self.comet = CometConfig(**d.get("comet", {}))

    @property
    def enabled(self):
        return self.tensorboard.enabled or self.wandb.enabled or self.csv_monitor.enabled or self.comet.enabled


class CheckpointParallelWriteConfig(DeepSpeedConfigModel):
    pipeline_stage: bool = False


class CheckpointConfig(DeepSpeedConfigModel):
    tag_validation: str = "Warn"
    load_universal: bool = False
    use_node_local_storage: bool = False
    parallel_write: CheckpointParallelWriteConfig = CheckpointParallelWriteConfig()
    writer: Optional[Dict[str, Any]] = None  # async (FastPersist-style) writer selection


class ThroughputTimerConfig(DeepSpeedConfigModel):
    enabled: bool = True
    synchronized: bool = True


class TimersConfig(DeepSpeedConfigModel):
    throughput: ThroughputTimerConfig = ThroughputTimerConfig()


class HybridEngineConfig(DeepSpeedConfigModel):
    enabled: bool = False
    max_out_tokens: int = 512
    inference_tp_size: int = 1
    release_inference_cache: bool = False
    pin_parameters: bool = True
    tp_gather_partition_size: int = 8


class NebulaConfig(DeepSpeedConfigModel):
    enabled: bool = False
    persistent_storage_path: Optional[str] = None
    persistent_time_interval: int = 100
    num_of_version_in_retention: int = 2
    enable_nebula_load: bool = True
    load_path: Optional[str] = None


class CompileConfig(DeepSpeedConfigModel):
    deepcompile: bool = False
    free_activation: bool = False
    offload_activation: bool = False
    offload_opt_states: bool = False
    double_buffer: bool = True
    symmetric_memory: bool = False
    debug_log: bool = False
    offload_parameters: bool = False
    sync_before_reduce: bool = False
    sync_after_reduce: bool = False
    sync_before_allgather: bool = False
    sync_after_allgather: bool = False


class CUDAGraphConfig(DeepSpeedConfigModel):
    """H100-native addition: capture the optimizer step / small-model step in a CUDA graph."""
    enabled: bool = False
    capture_optimizer_step: bool = True
    capture_full_step: bool = False
    warmup_steps: int = 3


# ------------------------------------------------------------------------------------------------
# top level
# ------------------------------------------------------------------------------------------------
_PASSTHROUGH_DICT_BLOCKS = ("compression_training", "data_efficiency", "curriculum_learning", "progressive_layer_drop",
                            "eigenvalue", "quantize_training", "sparse_attention", "weight_quantization", "autotuning",
                            "elasticity", "moe", "zenflow")


def _load_config_source(config: Union[str, dict, os.PathLike]) -> dict:
    if isinstance(config, dict):
        return copy.deepcopy(config)
    if isinstance(config, (str, os.PathLike)) and os.path.exists(config):
        with open(config, "r") as f:
            return hjson.load(f, object_pairs_hook=dict_raise_error_on_duplicate_keys)
    if isinstance(config, str):
        try:
            decoded = base64.urlsafe_b64decode(config).decode("utf-8")
            return hjson.loads(decoded, object_pairs_hook=dict_raise_error_on_duplicate_keys)
        except Exception:
            pass
        try:
            return hjson.loads(config, object_pairs_hook=dict_raise_error_on_duplicate_keys)
        except Exception:
            pass
    raise ValueError(f"Expected a string path to an existing deepspeed config, a dict, or a base64/json string. "
                     f"Received: {config!r}")


class DeepSpeedConfig:

    def __init__(self, config: Union[str, dict], mpu=None, mesh_device=None):
        self._param_dict = _load_config_source(config)
        self.mesh_device = mesh_device
        try:
            from deepspeed_b200 import comm as dist
            self.global_rank = dist.get_rank()
            if mpu is not None:
                if hasattr(mpu, "get_data_parallel_world_size"):
                    self.world_size = mpu.get_data_parallel_world_size()
                else:
                    self.world_size = dist.get_world_size() // mpu.get_model_parallel_world_size()
            elif mesh_device is not None:
                self.world_size = dist.get_world_size(mesh_device.get_group(mesh_dim="data_parallel"))
            else:
                sp = int(self._param_dict.get("sequence_parallel_size", 1))
                tp = int(self._param_dict.get("tensor_parallel", {}).get("autotp_size", 0)) or 1
                pp = self._param_dict.get("pipeline", {}).get("stages", 1)
                pp = 1 if not isinstance(pp, int) else pp
                self.world_size = max(dist.get_world_size() // (sp * tp * max(pp, 1)), 1)
                if "data_parallel_size" in self._param_dict:
                    self.world_size = int(self._param_dict["data_parallel_size"])
        except Exception:
            self.global_rank = 0
            self.world_size = 1
        # elasticity may rewrite the batch parameters before they are parsed
        self.elasticity_enabled = False
        self._apply_elasticity()
        self._initialize_params(self._param_dict)
        self._configure_train_batch_size()
        self._do_sanity_check()

    # ---- elasticity --------------------------------------------------------------------
    def _apply_elasticity(self):
        pd = self._param_dict
        el = pd.get("elasticity", {})
        if not el or not el.get("enabled", False):
            return
        from deepspeed_b200.elasticity import compute_elastic_config, ensure_immutable_elastic_config
        from deepspeed_b200.elasticity.constants import (IGNORE_NON_ELASTIC_BATCH_INFO,
                                                         IGNORE_NON_ELASTIC_BATCH_INFO_DEFAULT)
        from deepspeed_b200 import __reference_version__ as __version__  # (elasticity speaks upstream version numbers)
        self.elasticity_enabled = True
        ensure_immutable_elastic_config(runtime_elastic_config_dict=el)
        final_batch, valid_gpus, micro = compute_elastic_config(ds_config=pd,
                                                                target_deepspeed_version=__version__,
                                                                world_size=self.world_size)
        if not el.get(IGNORE_NON_ELASTIC_BATCH_INFO, IGNORE_NON_ELASTIC_BATCH_INFO_DEFAULT):
            clash = [k for k in ("train_batch_size", "train_micro_batch_size_per_gpu", "gradient_accumulation_steps")
                     if k in pd]
            if clash:
                raise DeepSpeedConfigError(
                    f"One or more batch related parameters were found in your ds_config ({clash}). These parameters "
                    f"*will not be used* since elastic training is enabled, which takes control of these parameters. "
                    f"If you want to suppress this error (the parameters will be silently ignored) please set "
                    f"'{IGNORE_NON_ELASTIC_BATCH_INFO}': true in your elasticity config.")
        gas = final_batch // (micro * self.world_size)
        logger.info(f"elasticity: train_batch_size={final_batch} micro_batch={micro} gas={gas} valid_gpus={valid_gpus}")
        pd["train_batch_size"] = final_batch
        pd["train_micro_batch_size_per_gpu"] = micro
        pd["gradient_accumulation_steps"] = gas

    # ---- parsing -----------------------------------------------------------------------
    def _initialize_params(self, pd: dict):
        g = pd.get
        self.train_batch_size = g("train_batch_size", None)
        self.train_micro_batch_size_per_gpu = g("train_micro_batch_size_per_gpu", None)
        self.gradient_accumulation_steps = g("gradient_accumulation_steps", None)
        self.steps_per_print = g("steps_per_print", None)
        self.dump_state = g("dump_state", False)
        self.disable_allgather = g("disable_allgather", False)
        self.communication_data_type = _dtype_from_str(g("communication_data_type", None))
        self.seq_parallel_communication_data_type = _dtype_from_str(g("seq_parallel_communication_data_type", "fp32"))
        self.prescale_gradients = g("prescale_gradients", False)
        self.gradient_predivide_factor = g("gradient_predivide_factor", 1.0)
        self.sparse_gradients_enabled = g("sparse_gradients", False)
        self.gradient_clipping = g("gradient_clipping", 0.0)
        self.graph_harvesting = g("graph_harvesting", False)
        self.wall_clock_breakdown = g("wall_clock_breakdown", False)
        self.memory_breakdown = g("memory_breakdown", False)
        self.dataloader_drop_last = g("dataloader_drop_last", False)
        self.zero_allow_untested_optimizer = g("zero_allow_untested_optimizer", False)
        self.zero_force_ds_cpu_optimizer = g("zero_force_ds_cpu_optimizer", True)
        self.sequence_parallel_size = g("sequence_parallel_size", 1)
        self.data_parallel_size = g("data_parallel_size", None)
        self.use_data_before_expert_parallel_ = g("use_data_before_expert_parallelism", False)
        self.vocabulary_size = g("vocabulary_size", 1e9)

        self.zero_config = get_zero_config(pd)
        self.zero_optimization_stage = int(self.zero_config.stage)
        self.zero_enabled = self.zero_optimization_stage > 0
        self.mics_shard_size = self.zero_config.mics_shard_size
        self.mics_hierarchial_params_gather = self.zero_config.mics_hierarchical_params_gather

        self.fp16_config = FP16Config(**g("fp16", {}))
        bf = g("bf16", g("bfloat16", {}))
        self.bf16_config = BF16Config(**bf)
        self.amp_config = AMPConfig(**g("amp", {}))
        self.data_types_config = DataTypesConfig(**g("data_types", {}))
        self.optimizer_config = OptimizerConfig(**g("optimizer", {})) if g("optimizer") else OptimizerConfig()
        self.scheduler_config = SchedulerConfig(**g("scheduler", {})) if g("scheduler") else SchedulerConfig()
        self.activation_checkpointing_config = ActivationCheckpointingConfig(**g("activation_checkpointing", {}))
        self.aio_config = AIOConfig(**g("aio", {}))
        self.pipeline_config = PipelineConfig(**g("pipeline", {}))
        self.pipeline = self.pipeline_config.model_dump()
        self.tensor_parallel_config = TensorParallelConfig(**g("tensor_parallel", {}))
        self.flops_profiler_config = FlopsProfilerConfig(**g("flops_profiler", {}))
        self.monitor_config = MonitorConfig(pd)
        self.comms_config = CommsConfig(pd)
        self.checkpoint_config = CheckpointConfig(**g("checkpoint", {}))
        self.timers_config = TimersConfig(**g("timers", {}))
        self.hybrid_engine = HybridEngineConfig(**g("hybrid_engine", {}))
        self.nebula_config = NebulaConfig(**g("nebula", {}))
        self.compile_config = CompileConfig(**g("compile", {}))
        self.cuda_graph_config = CUDAGraphConfig(**g("cuda_graph", {}))

        for k in _PASSTHROUGH_DICT_BLOCKS:
            setattr(self, f"{k}_params", copy.deepcopy(g(k, {})))
        self.curriculum_enabled_legacy = bool(self.curriculum_learning_params.get("enabled", False))
        self.curriculum_params_legacy = self.curriculum_learning_params
        self.pld_enabled = bool(self.progressive_layer_drop_params.get("enabled", False))
        self.pld_params = self.progressive_layer_drop_params if self.pld_enabled else False
        ev = self.eigenvalue_params
        self.eigenvalue_enabled = bool(ev.get("enabled", False))
        self.eigenvalue_verbose = ev.get("verbose", False)
        self.eigenvalue_max_iter = ev.get("max_iter", 100)
        self.eigenvalue_tol = ev.get("tol", 1e-2)
        self.eigenvalue_stability = ev.get("stability", 1e-6)
        self.eigenvalue_gas_boundary_resolution = ev.get("gas_boundary_resolution", 1)
        self.eigenvalue_layer_name = ev.get("layer_name", "bert.encoder.layer")
        self.eigenvalue_layer_num = ev.get("layer_num", 0)
        self.sparse_attention = self.sparse_attention_params or None
        self.compression_config = self.compression_training_params
        self.data_efficiency_enabled = bool(self.data_efficiency_params.get("enabled", False))
        self.data_efficiency_config = self.data_efficiency_params
        self.autotuning_config = self.autotuning_params
        self.weight_quantization_config = self.weight_quantization_params or None

        ckpt = self.checkpoint_config
        self.checkpoint_tag_validation_enabled = ckpt.tag_validation.upper() != "IGNORE"
        self.checkpoint_tag_validation_fail = ckpt.tag_validation.upper() == "FAIL"
        if ckpt.tag_validation.upper() not in ("WARN", "IGNORE", "FAIL"):
            raise DeepSpeedConfigError(f"Checkpoint config contains invalid tag_validation value of "
                                       f"{ckpt.tag_validation}, expecting one of ['WARN', 'IGNORE', 'FAIL']")
        self.load_universal_checkpoint = ckpt.load_universal
        self.use_node_local_storage = ckpt.use_node_local_storage

    # ---- flat aliases the reference engine exposes ---------------------------------------
    @property
    def fp16_enabled(self):
        return self.fp16_config.enabled

    @property
    def fp16_auto_cast(self):
        return self.fp16_config.auto_cast

    @property
    def fp16_master_weights_and_gradients(self):
        return self.fp16_config.fp16_master_weights_and_grads

    @property
    def bfloat16_enabled(self):
        return self.bf16_config.enabled

    @property
    def bfloat16_immediate_grad_update(self):
        return self.bf16_config.immediate_grad_update

    @property
    def amp_enabled(self):
        return self.amp_config.enabled

    @property
    def amp_params(self):
        d = self.amp_config.model_dump()
        d.update(self.amp_config.model_extra or {})
        d.pop("enabled", None)
        return d

    @property
    def loss_scale(self):
        return self.fp16_config.loss_scale

    @property
    def initial_dynamic_scale(self):
        return 2**self.fp16_config.initial_scale_power

    @property
    def dynamic_loss_scale_args(self):
        c = self.fp16_config
        if not c.enabled:
            return None
        return {
            "init_scale": 2**c.initial_scale_power,
            "scale_window": c.loss_scale_window,
            "delayed_shift": c.hysteresis,
            "consecutive_hysteresis": c.consecutive_hysteresis,
            "min_scale": c.min_loss_scale,
        }

    @property
    def grad_accum_dtype(self):
        return self.data_types_config.grad_accum_dtype

    @property
    def optimizer_name(self):
        t = self.optimizer_config.type
        if t is None:
            return None
        return t.lower() if t.lower() in DEEPSPEED_OPTIMIZERS else t

    @property
    def optimizer_params(self):
        return copy.deepcopy(self.optimizer_config.params) if self.optimizer_config.type else None

    @property
    def optimizer_legacy_fusion(self):
        return self.optimizer_config.legacy_fusion

    @property
    def scheduler_name(self):
        return self.scheduler_config.type

    @property
    def scheduler_params(self):
        return copy.deepcopy(self.scheduler_config.params) if self.scheduler_config.type else None

    # ---- batch triad (reference: config.py:936 _set_batch_related_parameters) ------------
    def _configure_train_batch_size(self):
        self._set_batch_related_parameters()
        self._batch_assertion()

    def _set_batch_related_parameters(self):
        tb, mb, gas = self.train_batch_size, self.train_micro_batch_size_per_gpu, self.gradient_accumulation_steps
        ws = self.world_size
        if tb is not None and mb is not None and gas is not None:
            return
        if tb is not None and mb is not None:
            gas = tb // mb // ws
        elif tb is not None and gas is not None:
            mb = tb // ws // gas
        elif mb is not None and gas is not None:
            tb = mb * gas * ws
        elif tb is not None:
            gas = 1
            mb = tb // ws
        elif mb is not None:
            gas = 1
            tb = mb * ws
        else:
            # (an AssertionError like every other batch-triad check -- the reference asserts here, config.py:975)
            raise DeepSpeedBatchConfigError("Either train_batch_size or train_micro_batch_size_per_gpu needs to be provided")
        self.train_batch_size, self.train_micro_batch_size_per_gpu, self.gradient_accumulation_steps = tb, mb, gas

    def _batch_assertion(self):
        tb, mb, gas = self.train_batch_size, self.train_micro_batch_size_per_gpu, self.gradient_accumulation_steps
        assert tb > 0, f"Train batch size: {tb} has to be greater than 0"
        assert mb > 0, f"Micro batch size per gpu: {mb} has to be greater than 0"
        assert gas > 0, f"Gradient accumulation steps: {gas} has to be greater than 0"
        assert tb == mb * gas * self.world_size, (
            f"Check batch related parameters. train_batch_size is not equal to micro_batch_per_gpu * gradient_acc_step"
            f" * world_size {tb} != {mb} * {gas} * {self.world_size}")

    def _do_sanity_check(self):
        if self.fp16_enabled and self.bfloat16_enabled:
            raise DeepSpeedConfigError("bf16 and fp16 modes cannot be simultaneously enabled")
        if self.fp16_master_weights_and_gradients:
            assert self.zero_enabled and self.zero_optimization_stage in (1, 2, 3), \
                "fp16_master_weights_and_grads is only supported with ZeRO"
        assert self.zero_optimization_stage <= ZeroStageEnum.max_stage, \
            f"DeepSpeedConfig: Maximum supported ZeRO stage is {int(ZeroStageEnum.max_stage)}"
        if self.steps_per_print is None:
            self.steps_per_print = 10

    # ---- output ------------------------------------------------------------------------
    def print_user_config(self):
        logger.info("  json = {}".format(
            json.dumps(self._param_dict, sort_keys=True, indent=4, cls=ScientificNotationEncoder,
                       separators=(",", ":"))))

    def print(self, name):
        logger.info(f"{name}:")
        for arg in sorted(vars(self)):
            if arg != "_param_dict":
                logger.info(f"  {arg} {'.' * max(1, 29 - len(arg))} {getattr(self, arg)}")
        self.print_user_config()


def _dtype_from_str(s):
    import torch
    if s is None:
        return None
    table = {
        "fp32": torch.float32,
        "float32": torch.float32,
        "fp16": torch.float16,
        "float16": torch.float16,
        "half": torch.float16,
        "bf16": torch.bfloat16,
        "bfloat16": torch.bfloat16,
    }
    if s not in table:
        raise ValueError(f"Invalid communication_data_type. Supported data types: {sorted(table)}. Got: {s}")
    return table[s]


# =====================================================================================================================
# Functional accessors over the raw config dict (reference ``runtime/config.py:get_*``).  The engine reads the typed
# ``DeepSpeedConfig`` above; these exist for tools / user code written against the functional API.
# =====================================================================================================================
import copy as _copy  # noqa: E402

from deepspeed_b200.runtime import constants as K  # noqa: E402
from deepspeed_b200.runtime.config_utils import get_scalar_param  # noqa: E402,F401
from deepspeed_b200.inference.v2.inference_utils import DtypeEnum  # noqa: E402,F401


def _section_flag(section, key, default):
    return lambda param_dict: get_scalar_param(param_dict[section], key, default) if section in param_dict else False


def _section_rest(section, drop):
    def f(param_dict):
        if section not in param_dict:
            return False
        d = _copy.copy(param_dict[section])
        d.pop(drop, None)
        return d
    return f


def _top(key, default):
    return lambda param_dict: get_scalar_param(param_dict, key, default)


def _bf16_section(param_dict):
    return next((param_dict[k] for k in (K.BFLOAT16, K.BFLOAT16_OLD) if k in param_dict), None)


get_pld_enabled = _section_flag(K.PROGRESSIVE_LAYER_DROP, K.PLD_ENABLED, K.PLD_ENABLED_DEFAULT)
get_pld_params = _section_rest(K.PROGRESSIVE_LAYER_DROP, K.PLD_ENABLED)
get_amp_enabled = _section_flag(K.AMP, K.AMP_ENABLED, K.AMP_ENABLED_DEFAULT)
get_amp_params = _section_rest(K.AMP, K.AMP_ENABLED)
get_fp16_enabled = _section_flag(K.FP16, K.FP16_ENABLED, K.FP16_ENABLED_DEFAULT)


def get_bfloat16_enabled(param_dict):
    sec = _bf16_section(param_dict)
    return get_scalar_param(sec, K.BFLOAT16_ENABLED, K.BFLOAT16_ENABLED_DEFAULT) if sec is not None else False


def get_bfloat16_immediate_grad_update(param_dict):
    sec = _bf16_section(param_dict)
    return get_scalar_param(sec, K.BFLOAT16_IMMEDIATE_GRAD_UPDATE, K.BFLOAT16_IMMEDIATE_GRAD_UPDATE_DEFAULT) if sec is not None else False


def _fp16_field(key, default, off=False):
    return lambda param_dict: get_scalar_param(param_dict[K.FP16], key, default) if get_fp16_enabled(param_dict) else off


get_fp16_master_weights_and_grads_enabled = _fp16_field(K.FP16_MASTER_WEIGHTS_AND_GRADS, K.FP16_MASTER_WEIGHTS_AND_GRADS_DEFAULT)
get_fp16_auto_cast = _fp16_field(K.FP16_AUTO_CAST, K.FP16_AUTO_CAST_DEFAULT, off=None)


def get_loss_scale(param_dict):
    if get_fp16_enabled(param_dict):
        return get_scalar_param(param_dict[K.FP16], K.FP16_LOSS_SCALE, K.FP16_LOSS_SCALE_DEFAULT)
    return 1.0 if get_bfloat16_enabled(param_dict) else K.FP16_LOSS_SCALE_DEFAULT


def get_initial_dynamic_scale(param_dict):
    if get_fp16_enabled(param_dict):
        power = get_scalar_param(param_dict[K.FP16], K.FP16_INITIAL_SCALE_POWER, K.FP16_INITIAL_SCALE_POWER_DEFAULT)
    else:
        power = 0 if get_bfloat16_enabled(param_dict) else K.FP16_INITIAL_SCALE_POWER_DEFAULT
    return 2**power


def get_dynamic_loss_scale_args(param_dict):
    """Keyword arguments of the dynamic loss scaler, or None when none of its knobs is set."""
    if not get_fp16_enabled(param_dict):
        return None
    fp16 = param_dict[K.FP16]
    knobs = (K.FP16_INITIAL_SCALE_POWER, K.FP16_LOSS_SCALE_WINDOW, K.FP16_MIN_LOSS_SCALE, K.FP16_HYSTERESIS, K.FP16_CONSECUTIVE_HYSTERESIS)
    if not any(k in fp16 for k in knobs):
        return None
    return {"init_scale": 2**get_scalar_param(fp16, K.FP16_INITIAL_SCALE_POWER, K.FP16_INITIAL_SCALE_POWER_DEFAULT),
            "scale_window": get_scalar_param(fp16, K.FP16_LOSS_SCALE_WINDOW, K.FP16_LOSS_SCALE_WINDOW_DEFAULT),
            "delayed_shift": get_scalar_param(fp16, K.FP16_HYSTERESIS, K.FP16_HYSTERESIS_DEFAULT),
            "consecutive_hysteresis": get_scalar_param(fp16, K.FP16_CONSECUTIVE_HYSTERESIS, K.FP16_CONSECUTIVE_HYSTERESIS_DEFAULT),
            "min_scale": get_scalar_param(fp16, K.FP16_MIN_LOSS_SCALE, K.FP16_MIN_LOSS_SCALE_DEFAULT)}


get_gradient_accumulation_steps = _top(K.GRADIENT_ACCUMULATION_STEPS, K.GRADIENT_ACCUMULATION_STEPS_DEFAULT)
get_sparse_gradients_enabled = _top(K.SPARSE_GRADIENTS, K.SPARSE_GRADIENTS_DEFAULT)
get_prescale_gradients = _top(K.PRESCALE_GRADIENTS, K.PRESCALE_GRADIENTS_DEFAULT)
get_gradient_predivide_factor = _top(K.GRADIENT_PREDIVIDE_FACTOR, K.GRADIENT_PREDIVIDE_FACTOR_DEFAULT)
get_steps_per_print = _top(K.STEPS_PER_PRINT, K.STEPS_PER_PRINT_DEFAULT)
get_disable_allgather = _top(K.DISABLE_ALLGATHER, K.DISABLE_ALLGATHER_DEFAULT)
get_dump_state = _top(K.DUMP_STATE, K.DUMP_STATE_DEFAULT)
get_gradient_clipping = _top(K.GRADIENT_CLIPPING, K.GRADIENT_CLIPPING_DEFAULT)
get_graph_harvesting = _top(K.GRAPH_HARVESTING, K.GRAPH_HARVESTING_DEFAULT)
get_train_batch_size = _top(K.TRAIN_BATCH_SIZE, K.TRAIN_BATCH_SIZE_DEFAULT)
get_train_micro_batch_size_per_gpu = _top(K.TRAIN_MICRO_BATCH_SIZE_PER_GPU, K.TRAIN_MICRO_BATCH_SIZE_PER_GPU_DEFAULT)
get_wall_clock_breakdown = _top(K.WALL_CLOCK_BREAKDOWN, K.WALL_CLOCK_BREAKDOWN_DEFAULT)
get_memory_breakdown = _top(K.MEMORY_BREAKDOWN, K.MEMORY_BREAKDOWN_DEFAULT)
get_zero_allow_untested_optimizer = _top(K.ZERO_ALLOW_UNTESTED_OPTIMIZER, K.ZERO_ALLOW_UNTESTED_OPTIMIZER_DEFAULT)
get_zero_force_ds_cpu_optimizer = _top(K.ZERO_FORCE_DS_CPU_OPTIMIZER, K.ZERO_FORCE_DS_CPU_OPTIMIZER_DEFAULT)
get_dataloader_drop_last = _top(K.DATALOADER_DROP_LAST, K.DATALOADER_DROP_LAST_DEFAULT)


def get_communication_data_type(param_dict, comm_type=K.COMMUNICATION_DATA_TYPE, comm_data_type_default=K.COMMUNICATION_DATA_TYPE_DEFAULT):
    import torch
    val = get_scalar_param(param_dict, comm_type, comm_data_type_default)
    if val is None:
        return None  # decided later from the training dtype
    table = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16, "bfp16": torch.bfloat16}
    if str(val).lower() not in table:
        raise ValueError(f"Invalid communication_data_type. Supported data types: {sorted(table)}. Got: {val}")
    return table[str(val).lower()]


def _named(section, field, default=None):
    def f(param_dict):
        sec = param_dict.get(section)
        return sec.get(field, default) if isinstance(sec, dict) else default
    return f


get_optimizer_name = _named(K.OPTIMIZER, K.TYPE, K.OPTIMIZER_TYPE_DEFAULT)
get_optimizer_params = _named(K.OPTIMIZER, K.OPTIMIZER_PARAMS)
get_optimizer_legacy_fusion = _named(K.OPTIMIZER, K.LEGACY_FUSION, K.LEGACY_FUSION_DEFAULT)
get_scheduler_name = _named(K.SCHEDULER, K.TYPE, K.SCHEDULER_TYPE_DEFAULT)
get_scheduler_params = _named(K.SCHEDULER, K.SCHEDULER_PARAMS)


def get_optimizer_gradient_clipping(param_dict):
    params = get_optimizer_params(param_dict)
    return params.get(K.MAX_GRAD_NORM) if isinstance(params, dict) else None


def get_pipeline_config(param_dict):
    """The ``pipeline`` section over its defaults."""
    out = PipelineConfig().model_dump()
    out.update(param_dict.get("pipeline", {}))
    return out


def get_hybrid_engine_config(param_dict):
    return HybridEngineConfig(**param_dict.get("hybrid_engine", {}))


def get_expert_data_topo_config(param_dict):
    return get_scalar_param(param_dict, K.USE_DATA_BEFORE_EXPERT_PARALLEL, K.USE_DATA_BEFORE_EXPERT_PARALLEL_DEFAULT)


def _eig(key, default):
    return lambda param_dict: get_scalar_param(param_dict[K.EIGENVALUE], key, default) if K.EIGENVALUE in param_dict else default


get_eigenvalue_enabled = _eig(K.EIGENVALUE_ENABLED, K.EIGENVALUE_ENABLED_DEFAULT)
get_eigenvalue_verbose = _eig(K.EIGENVALUE_VERBOSE, K.EIGENVALUE_VERBOSE_DEFAULT)
get_eigenvalue_max_iter = _eig(K.EIGENVALUE_MAX_ITER, K.EIGENVALUE_MAX_ITER_DEFAULT)
get_eigenvalue_tol = _eig(K.EIGENVALUE_TOL, K.EIGENVALUE_TOL_DEFAULT)
get_eigenvalue_stability = _eig(K.EIGENVALUE_STABILITY, K.EIGENVALUE_STABILITY_DEFAULT)
get_eigenvalue_gas_boundary_resolution = _eig(K.EIGENVALUE_GAS_BOUNDARY_RESOLUTION, K.EIGENVALUE_GAS_BOUNDARY_RESOLUTION_DEFAULT)
get_eigenvalue_layer_name = _eig(K.EIGENVALUE_LAYER_NAME, K.EIGENVALUE_LAYER_NAME_DEFAULT)
get_eigenvalue_layer_num = _eig(K.EIGENVALUE_LAYER_NUM, K.EIGENVALUE_LAYER_NUM_DEFAULT)


def get_eigenvalue_config(param_dict):
    """(enabled, verbose, max_iter, tol, stability, gas_boundary_resolution, layer_name, layer_num)"""
    if not get_eigenvalue_enabled(param_dict):
        return (False, K.EIGENVALUE_VERBOSE_DEFAULT, K.EIGENVALUE_MAX_ITER_DEFAULT, K.EIGENVALUE_TOL_DEFAULT, K.EIGENVALUE_STABILITY_DEFAULT,
                K.EIGENVALUE_GAS_BOUNDARY_RESOLUTION_DEFAULT, K.EIGENVALUE_LAYER_NAME_DEFAULT, K.EIGENVALUE_LAYER_NUM_DEFAULT)
    return (True, get_eigenvalue_verbose(param_dict), get_eigenvalue_max_iter(param_dict), get_eigenvalue_tol(param_dict),
            get_eigenvalue_stability(param_dict), get_eigenvalue_gas_boundary_resolution(param_dict),
            get_eigenvalue_layer_name(param_dict), get_eigenvalue_layer_num(param_dict))


def get_checkpoint_params(param_dict):
    return param_dict.get(K.CHECKPOINT, {})


def get_data_types_params(param_dict):
    return param_dict.get(K.DATA_TYPES, {})


def get_checkpoint_tag_validation_mode(checkpoint_params):
    mode = str(checkpoint_params.get(K.CHECKPOINT_TAG_VALIDATION, K.CHECKPOINT_TAG_VALIDATION_DEFAULT)).upper()
    if mode not in K.CHECKPOINT_TAG_VALIDATION_MODES:
        raise DeepSpeedConfigError(f"Checkpoint config contains invalid tag_validation value of {mode}, expecting one of "
                                   f"{K.CHECKPOINT_TAG_VALIDATION_MODES}")
    return mode


def get_checkpoint_parallel_write_pipeline(checkpoint_params):
    par = checkpoint_params.get(K.CHECKPOINT_PARALLEL_WRITE, {})
    val = par.get(K.CHECKPOINT_PARALLEL_WRITE_PIPELINE_STAGE, K.CHECKPOINT_PARALLEL_WRITE_PIPELINE_STAGE_DEFAULT)
    if val not in (True, False):
        raise DeepSpeedConfigError(f"checkpoint::parallel_write::pipeline_stage value of '{val}' is invalid, expecting: true or false")
    return val


# ---- sparse attention section -----------------------------------------------------------------------------------------
def get_sparse_attention_mode(param_dict):
    return param_dict.get(K.SPARSE_MODE, K.SPARSE_MODE_DEFAULT)


def get_sparse_attention_type(param_dict):
    return param_dict.get(K.SPARSE_ATTENTION_TYPE, K.SPARSE_ATTENTION_TYPE_DEFAULT)


def _sparse(mode, *fields):
    """Builder of a ``get_sparse_<mode>_config``: the mode + ``block`` + the listed (key, default) fields."""
    def f(sparsity):
        out = {K.SPARSE_MODE: mode, K.SPARSE_BLOCK: get_scalar_param(sparsity, K.SPARSE_BLOCK, K.SPARSE_BLOCK_DEFAULT)}
        for key, default in fields:
            out[key] = get_scalar_param(sparsity, key, default)
        return out
    return f


_LAYOUT = (K.SPARSE_DIFFERENT_LAYOUT_PER_HEAD, K.SPARSE_DIFFERENT_LAYOUT_PER_HEAD_DEFAULT)
get_sparse_dense_config = _sparse(K.SPARSE_DENSE_MODE)
get_sparse_fixed_config = _sparse(K.SPARSE_FIXED_MODE, _LAYOUT, (K.SPARSE_NUM_LOCAL_BLOCKS, K.SPARSE_NUM_LOCAL_BLOCKS_DEFAULT),
                                  (K.SPARSE_NUM_GLOBAL_BLOCKS, K.SPARSE_NUM_GLOBAL_BLOCKS_DEFAULT),
                                  (K.SPARSE_ATTENTION_TYPE, K.SPARSE_ATTENTION_TYPE_DEFAULT),
                                  (K.SPARSE_HORIZONTAL_GLOBAL_ATTENTION, K.SPARSE_HORIZONTAL_GLOBAL_ATTENTION_DEFAULT),
                                  (K.SPARSE_NUM_DIFFERENT_GLOBAL_PATTERNS, K.SPARSE_NUM_DIFFERENT_GLOBAL_PATTERNS_DEFAULT))
get_sparse_variable_config = _sparse(K.SPARSE_VARIABLE_MODE, _LAYOUT, (K.SPARSE_NUM_RANDOM_BLOCKS, K.SPARSE_NUM_RANDOM_BLOCKS_DEFAULT),
                                     (K.SPARSE_LOCAL_WINDOW_BLOCKS, K.SPARSE_LOCAL_WINDOW_BLOCKS_DEFAULT),
                                     (K.SPARSE_GLOBAL_BLOCK_INDICES, K.SPARSE_GLOBAL_BLOCK_INDICES_DEFAULT),
                                     (K.SPARSE_GLOBAL_BLOCK_END_INDICES, K.SPARSE_GLOBAL_BLOCK_END_INDICES_DEFAULT),
                                     (K.SPARSE_ATTENTION_TYPE, K.SPARSE_ATTENTION_TYPE_DEFAULT),
                                     (K.SPARSE_HORIZONTAL_GLOBAL_ATTENTION, K.SPARSE_HORIZONTAL_GLOBAL_ATTENTION_DEFAULT))
get_sparse_bigbird_config = _sparse(K.SPARSE_BIGBIRD_MODE, _LAYOUT, (K.SPARSE_NUM_RANDOM_BLOCKS, K.SPARSE_NUM_RANDOM_BLOCKS_DEFAULT),
                                    (K.SPARSE_NUM_SLIDING_WINDOW_BLOCKS, K.SPARSE_NUM_SLIDING_WINDOW_BLOCKS_DEFAULT),
                                    (K.SPARSE_NUM_GLOBAL_BLOCKS, K.SPARSE_NUM_GLOBAL_BLOCKS_DEFAULT))
get_sparse_bslongformer_config = _sparse(K.SPARSE_BSLONGFORMER_MODE, _LAYOUT,
                                         (K.SPARSE_NUM_SLIDING_WINDOW_BLOCKS, K.SPARSE_NUM_SLIDING_WINDOW_BLOCKS_DEFAULT),
                                         (K.SPARSE_GLOBAL_BLOCK_INDICES, K.SPARSE_GLOBAL_BLOCK_INDICES_DEFAULT),
                                         (K.SPARSE_GLOBAL_BLOCK_END_INDICES, K.SPARSE_GLOBAL_BLOCK_END_INDICES_DEFAULT))
_SPARSE_BUILDERS = {K.SPARSE_DENSE_MODE: get_sparse_dense_config, K.SPARSE_FIXED_MODE: get_sparse_fixed_config,
                    K.SPARSE_VARIABLE_MODE: get_sparse_variable_config, K.SPARSE_BIGBIRD_MODE: get_sparse_bigbird_config,
                    K.SPARSE_BSLONGFORMER_MODE: get_sparse_bslongformer_config}


def get_sparse_attention(param_dict):
    if K.SPARSE_ATTENTION not in param_dict:
        return None
    sparsity = param_dict[K.SPARSE_ATTENTION]
    mode = get_sparse_attention_mode(sparsity)
    if mode not in _SPARSE_BUILDERS:
        raise NotImplementedError(f"Given sparsity mode, {mode}, has not been implemented yet!")
    return _SPARSE_BUILDERS[mode](sparsity)


class DeepSpeedConfigWriter:
    """Accumulate config entries and write / reload them as JSON (reference ``DeepSpeedConfigWriter``)."""

    def __init__(self, data=None):
        self.data = data if data is not None else {}

    def add_config(self, key, value):
        self.data[key] = value

    def load_config(self, filename):
        with open(filename) as f:
            self.data = json.load(f, object_pairs_hook=dict_raise_error_on_duplicate_keys)

    def write_config(self, filename):
        with open(filename, "w") as f:
            json.dump(self.data, f)


for _n, _f in list(globals().items()):  # give the generated accessors proper names
    if _n.startswith("get_") and callable(_f) and getattr(_f, "__name__", "") in ("<lambda>", "f"):
        _f.__name__ = _n
