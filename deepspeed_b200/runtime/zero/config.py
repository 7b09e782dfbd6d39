"""ZeRO config (reference: ``runtime/zero/config.py:86 DeepSpeedZeroConfig``).

All reference keys are accepted with the same defaults.  H100-specific additions live under
``b200_*`` keys and default to the fused NVLink paths when the symmetric arena is available:

* ``b200_fused_collectives``: ``"auto" | true | false`` -- use in-kernel peer-memory
  all-gather / reduce-scatter(+Adam) instead of NCCL.
* ``b200_unit_prefetch``: how many ZeRO-3 units to gather ahead.
* ``b200_verify_collectives``: N > 0 cross-checks every symmetric-memory collective against NCCL for N steps.
"""
import sys
from enum import Enum
from typing import Any, Dict, Optional

from pydantic import Field, model_validator

from deepspeed_b200.runtime.config_utils import DeepSpeedConfigModel, get_scalar_param, pp_int
from deepspeed_b200.utils.logging import logger
from .offload_config import (DeepSpeedZeroOffloadOptimizerConfig, DeepSpeedZeroOffloadParamConfig, OffloadDeviceEnum)

ZERO_OPTIMIZATION = "zero_optimization"


class ZeroStageEnum(int, Enum):
    disabled = 0
    optimizer_states = 1
    gradients = 2
    weights = 3
    max_stage = 3


class ZeRORuntimeException(Exception):
    pass


def get_zero_config(param_dict):
    zc = param_dict.get(ZERO_OPTIMIZATION, {})
    if isinstance(zc, bool):  # ancient format: "zero_optimization": true
        logger.warning("DeepSpeedConfig: boolean zero_optimization is deprecated; use {'stage': 1}")
        zc = {"stage": 1 if zc else 0}
        if zc["stage"]:
            zc["allgather_bucket_size"] = get_scalar_param(param_dict, "allgather_size", 5e8)
    return DeepSpeedZeroConfig(**zc)


class DeepSpeedZeroConfig(DeepSpeedConfigModel):
    stage: ZeroStageEnum = 0
    contiguous_gradients: bool = True
    reduce_scatter: bool = True
    reduce_bucket_size: int = Field(pp_int(5e8), ge=0)
    use_multi_rank_bucket_allreduce: bool = True
    allgather_partitions: bool = True
    allgather_bucket_size: int = Field(pp_int(5e8), ge=0)
    overlap_comm: Optional[bool] = None  # None -> True for stage 3, False otherwise
    load_from_fp32_weights: bool = True
    elastic_checkpoint: bool = False

    offload_param: Optional[DeepSpeedZeroOffloadParamConfig] = None
    offload_optimizer: Optional[DeepSpeedZeroOffloadOptimizerConfig] = None
    sub_group_size: int = Field(pp_int(1e9), ge=0)

    cpu_offload_param: Optional[bool] = Field(
        None,
        json_schema_extra={
            "deprecated": True,
            "new_param": "offload_param",
            "new_param_fn": (lambda val: DeepSpeedZeroOffloadParamConfig(device=OffloadDeviceEnum.cpu) if val else None)
        })
    cpu_offload_use_pin_memory: Optional[bool] = Field(
        None, json_schema_extra={
            "deprecated": True,
            "new_param": "offload_param or offload_optimizer",
            "set_new_param": False
        })
    cpu_offload: Optional[bool] = Field(
        None,
        json_schema_extra={
            "deprecated": True,
            "new_param": "offload_optimizer",
            "new_param_fn": (lambda val: DeepSpeedZeroOffloadOptimizerConfig(device=OffloadDeviceEnum.cpu)
                             if val else None)
        })

    prefetch_bucket_size: int = Field(pp_int(5e7), ge=0, alias="stage3_prefetch_bucket_size")
    param_persistence_threshold: int = Field(pp_int(1e5), ge=0, alias="stage3_param_persistence_threshold")
    model_persistence_threshold: int = Field(pp_int(sys.maxsize, "sys.maxsize"),
                                             ge=0,
                                             alias="stage3_model_persistence_threshold")
    max_live_parameters: int = Field(pp_int(1e9), ge=0, alias="stage3_max_live_parameters")
    max_reuse_distance: int = Field(pp_int(1e9), ge=0, alias="stage3_max_reuse_distance")
    gather_16bit_weights_on_model_save: bool = Field(False, alias="stage3_gather_16bit_weights_on_model_save")
    module_granularity_threshold: int = Field(pp_int(0), alias="stage3_module_granularity_threshold")
    use_all_reduce_for_fetch_params: bool = Field(False, alias="stage3_use_all_reduce_for_fetch_params")
    stage3_gather_fp16_weights_on_model_save: bool = Field(False,
                                                           json_schema_extra={
                                                               "deprecated": True,
                                                               "new_param": "gather_16bit_weights_on_model_save"
                                                           })

    ignore_unused_parameters: bool = True
    legacy_stage1: bool = False
    round_robin_gradients: bool = False
    zero_hpz_partition_size: int = Field(1, ge=0)
    zero_quantized_weights: bool = False
    zero_quantized_nontrainable_weights: bool = False
    zero_quantized_gradients: bool = False
    zeropp_loco_param: Optional[Dict[str, Any]] = None
    mics_shard_size: int = Field(-1, json_schema_extra={"new_param": "mics_shard_size"})
    mics_hierarchical_params_gather: bool = False
    memory_efficient_linear: bool = True
    pipeline_loading_checkpoint: bool = False
    override_module_apply: bool = True
    log_trace_cache_warnings: bool = False

    # ---- H100-native knobs -------------------------------------------------------------
    b200_fused_collectives: Optional[bool] = None  # None == auto (on when symmetric arena is up)
    b200_unit_prefetch: int = Field(1, ge=0)
    b200_fused_optimizer_in_backward: Optional[bool] = None  # None == auto (on when no clipping / GAS==1)
    b200_nvls: Optional[bool] = None  # None == auto (multimem when the multicast object binds)
    # debug: for the first N optimizer steps run the NCCL collective next to every in-kernel NVLink collective and assert
    # agreement (the reference's ``pg_correctness_test`` switch, stage_1_and_2.py:36, made real)
    b200_verify_collectives: int = Field(0, ge=0)
    # ZeRO-3: post-backward hooks that free a unit between the backward invocations of a module that ran more than once
    # in forward (siamese / contrastive losses); off = one hook less per unit for strictly single-invocation models
    b200_multi_forward: bool = True

    @model_validator(mode="after")
    def overlap_comm_valid(self):
        if self.overlap_comm is None:
            self.__dict__["overlap_comm"] = self.stage == ZeroStageEnum.weights
        return self

    @model_validator(mode="after")
    def offload_ratio_check(self):
        oo = self.offload_optimizer
        if oo and oo.ratio < 1.0:
            assert self.stage == ZeroStageEnum.weights, "Partial offloading only supported for ZeRO Stage 3."
        return self


ZERO_FORMAT = '''"zero_optimization": {"stage": [0|1|2|3], "stage3_max_live_parameters": 1e9, "stage3_max_reuse_distance": 1e9,
  "stage3_prefetch_bucket_size": 5e8, "stage3_param_persistence_threshold": 1e5, "allgather_bucket_size": 5e8,
  "reduce_bucket_size": 5e8, "overlap_comm": false, "reduce_scatter": true, "contiguous_gradients": true, "sub_group_size": 1e9,
  "offload_param": {...}, "offload_optimizer": {...}, "zero_hpz_partition_size": 1, "zero_quantized_weights": false,
  "zero_quantized_gradients": false, "mics_shard_size": -1, "ignore_unused_parameters": true, "round_robin_gradients": false}'''


def read_zero_config_deprecated(param_dict):
    """``"zero_optimization": true`` (pre-0.3 boolean form) -> stage 1 with the old ``allgather_size`` key honoured."""
    from deepspeed_b200.runtime.config_utils import get_scalar_param
    cfg = {"stage": 1 if param_dict.get("zero_optimization") else 0}
    if cfg["stage"] > 0:
        cfg["allgather_bucket_size"] = get_scalar_param(param_dict, "allgather_size", 5e8)
    return cfg
