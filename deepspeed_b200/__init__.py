"""deepspeed_b200 -- a Hopper-native (sm_90a) distributed training / inference framework with the
capabilities and user-facing contract of DeepSpeed.

Public API parity: reference ``deepspeed/__init__.py`` (``initialize :69``, ``init_inference :291``,
``tp_model_init :369``, ``add_config_arguments :268``, ``init_distributed``, ``zero``, ``comm``,
``checkpointing``, ``PipelineModule``, ``moe``).
"""
import argparse
from typing import Optional, Union

import torch

__version__ = "0.1.0"
__reference_version__ = "0.16.5"  # the upstream release whose API / config / checkpoint contract this package follows
__version_major__, __version_minor__, __version_patch__ = 0, 1, 0
__git_hash__ = None
__git_branch__ = None

from . import comm  # noqa: E402
from . import comm as dist  # noqa: E402
from .accelerator import get_accelerator  # noqa: E402
from .comm.comm import init_distributed  # noqa: E402
from .runtime import zero  # noqa: E402
from .runtime.config import DeepSpeedConfig, DeepSpeedConfigError  # noqa: E402
from .utils import logger, log_dist, OnDevice  # noqa: E402
from .utils import groups  # noqa: E402


def _lazy(name):
    import importlib
    return importlib.import_module(name, __name__)


def __getattr__(name):
    if name == "DeepSpeedEngine":
        return _lazy(".runtime.engine").DeepSpeedEngine
    if name in ("PipelineEngine", ):
        return _lazy(".runtime.pipe.engine").PipelineEngine
    if name in ("PipelineModule", "LayerSpec", "TiedLayerSpec"):
        return getattr(_lazy(".runtime.pipe.module"), name)
    if name == "InferenceEngine":
        return _lazy(".inference.engine").InferenceEngine
    if name == "DeepSpeedHybridEngine":
        return _lazy(".runtime.hybrid_engine").DeepSpeedHybridEngine
    if name == "checkpointing":
        return _lazy(".runtime.activation_checkpointing.checkpointing")
    if name in ("pipe", ):
        return _lazy(".pipe")
    if name in ("moe", "ops", "module_inject", "inference", "sequence", "linear", "models", "parallel", "compression",
                "profiling", "monitor", "elasticity", "autotuning", "launcher", "checkpoint", "nvme"):
        return _lazy("." + name)
    if name in ("DeepSpeedTransformerLayer", "DeepSpeedTransformerConfig"):
        return getattr(_lazy(".ops.transformer"), name)
    if name == "DeepSpeedInferenceConfig":
        return _lazy(".inference.config").DeepSpeedInferenceConfig
    if name == "DeepSpeedOptimizer":
        return _lazy(".runtime.zero.sharded").ZeroShardedOptimizer
    raise AttributeError(f"module 'deepspeed_b200' has no attribute {name!r}")


def initialize(args=None,
               model: torch.nn.Module = None,
               optimizer=None,
               model_parameters=None,
               training_data=None,
               lr_scheduler=None,
               distributed_port: int = 29500,
               mpu=None,
               dist_init_required: Optional[bool] = None,
               collate_fn=None,
               config=None,
               mesh_param=None,
               config_params=None):
    """Build an engine around ``model``.  Returns ``(engine, optimizer, training_dataloader, lr_scheduler)``.

    Engine selection mirrors the reference (``__init__.py:178-219``): a ``PipelineModule`` gets a
    ``PipelineEngine``, ``hybrid_engine.enabled`` gets the hybrid (train + generate) engine, anything
    else a ``DeepSpeedEngine``.
    """
    log_dist(f"deepspeed_b200 info: version={__version__}", ranks=[0])
    assert model is not None, "deepspeed.initialize requires a model"
    from .runtime.zero.partition_parameters import shutdown_init_context
    shutdown_init_context()
    if config is None:
        config = config_params
    if config is None and args is not None:
        config = getattr(args, "deepspeed_config", None) or getattr(args, "deepscale_config", None)
    assert config is not None, "DeepSpeed requires --deepspeed_config to specify configuration file"
    init_distributed(dist_backend=get_accelerator().communication_backend_name(),
                     distributed_port=distributed_port,
                     dist_init_required=dist_init_required)
    mesh_device = None
    if mesh_param:
        mesh_device = comm.initialize_mesh_device(mesh_param, ("data_parallel", "sequence_parallel"))
    else:
        probe = config if isinstance(config, dict) else None
        if probe is not None and probe.get("sequence_parallel_size", 1) > 1 and probe.get("data_parallel_size"):
            mesh_device = comm.initialize_mesh_device(
                (probe["data_parallel_size"], probe["sequence_parallel_size"]), ("data_parallel", "sequence_parallel"))
    try:
        from .runtime.pipe.module import PipelineModule
    except ImportError:  # pipeline package optional at import time
        PipelineModule = ()
    # a PipelineModule carries its own topology: the batch triad is resolved against ITS data-parallel degree
    cfg_mpu = model.mpu() if (PipelineModule and isinstance(model, PipelineModule) and mpu is None) else mpu
    cfg = DeepSpeedConfig(config, cfg_mpu, mesh_device=mesh_device)
    if PipelineModule and isinstance(model, PipelineModule):
        from .runtime.pipe.engine import PipelineEngine
        assert mpu is None, "mpu must be None with pipeline parallelism"
        engine = PipelineEngine(args=args, model=model, optimizer=optimizer, model_parameters=model_parameters,
                                training_data=training_data, lr_scheduler=lr_scheduler, mpu=model.mpu(),
                                dist_init_required=dist_init_required, collate_fn=collate_fn, config=config,
                                config_class=cfg)
    elif cfg.hybrid_engine.enabled:
        from .runtime.hybrid_engine import DeepSpeedHybridEngine
        engine = DeepSpeedHybridEngine(args=args, model=model, optimizer=optimizer, model_parameters=model_parameters,
                                       training_data=training_data, lr_scheduler=lr_scheduler, mpu=mpu,
                                       dist_init_required=dist_init_required, collate_fn=collate_fn, config=config,
                                       config_class=cfg)
    else:
        from .runtime.engine import DeepSpeedEngine
        engine = DeepSpeedEngine(args=args, model=model, optimizer=optimizer, model_parameters=model_parameters,
                                 training_data=training_data, lr_scheduler=lr_scheduler, mpu=mpu,
                                 dist_init_required=dist_init_required, collate_fn=collate_fn, config=config,
                                 config_class=cfg, mesh_device=mesh_device)
    return engine, engine.optimizer, engine.training_dataloader, engine.lr_scheduler


def _add_core_arguments(parser):
    g = parser.add_argument_group("DeepSpeed", "DeepSpeed configurations")
    g.add_argument("--deepspeed", default=False, action="store_true",
                   help="Enable DeepSpeed (helper flag for user code, no impact on DeepSpeed backend)")
    g.add_argument("--deepspeed_config", default=None, type=str, help="DeepSpeed json configuration file.")
    g.add_argument("--deepscale", default=False, action="store_true", help=argparse.SUPPRESS)
    g.add_argument("--deepscale_config", default=None, type=str, help=argparse.SUPPRESS)
    return parser


def add_config_arguments(parser):
    """Add ``--deepspeed`` / ``--deepspeed_config`` to an argparse parser (reference :268)."""
    return _add_core_arguments(parser)


def default_inference_config():
    from .inference.config import DeepSpeedInferenceConfig
    return DeepSpeedInferenceConfig().model_dump()


def init_inference(model, config=None, **kwargs):
    """Wrap ``model`` for inference (TP sharding, kernel injection, CUDA graphs).  Reference :291."""
    from .inference.config import DeepSpeedInferenceConfig
    from .inference.engine import InferenceEngine
    if config is None:
        config = {}
    if isinstance(config, str):
        import json
        with open(config) as f:
            config = json.load(f)
    elif not isinstance(config, dict):
        raise ValueError(f"'config' argument expected string or dictionary, got {type(config)}")
    overlap = set(config.keys()) & set(kwargs.keys())
    for k in overlap:
        if config[k] != kwargs[k]:
            raise ValueError(f"Conflicting argument '{k}' in 'config':{config[k]} and kwargs:{kwargs[k]}")
    config = dict(config)
    config.update(kwargs)
    return InferenceEngine(model, config=DeepSpeedInferenceConfig(**config))


def tp_model_init(model, tp_size, dtype, config=None, **kwargs):
    """Shard ``model`` for tensor-parallel *training* (AutoTP).  Reference :369."""
    from .module_inject.auto_tp import tp_model_init as _impl
    return _impl(model, tp_size, dtype, config=config, **kwargs)


# ---- reference top-level names ----------------------------------------------------------------------------------------
from typing import Callable, Iterable, Union  # noqa: E402

import torch as _torch  # noqa: E402

from .constants import TORCH_DISTRIBUTED_DEFAULT_PORT  # noqa: E402,F401
from .runtime.lr_schedules import add_tuning_arguments  # noqa: E402,F401
from .runtime.compiler import is_compile_supported  # noqa: E402,F401

ADAM_OPTIMIZER, LAMB_OPTIMIZER = "adam", "lamb"
DeepSpeedOptimizerCallable = Callable[[Union[Iterable[_torch.nn.Parameter], dict]], _torch.optim.Optimizer]
DeepSpeedSchedulerCallable = Callable[[_torch.optim.Optimizer], object]
version = __version__


def set_autotp_mode(training=False):
    """Select whether AutoTP builds training (autograd-aware) or inference tensor-parallel layers."""
    from .module_inject import layers as _l
    _l.AUTOTP_TRAINING_MODE = bool(training)


def __getattr_compat(name):
    if name in ("git_hash", "git_branch"):
        from . import git_version_info as g
        return getattr(g, name)
    if name in ("replace_transformer_layer", "revert_transformer_layer"):
        from .module_inject import replace_module as r
        return getattr(r, name)
    if name == "domino":
        from .runtime import domino as d
        return d
    raise AttributeError(name)


_orig_getattr = globals().get("__getattr__")


def __getattr__(name):  # noqa: F811
    try:
        return __getattr_compat(name)
    except AttributeError:
        if _orig_getattr is not None:
            return _orig_getattr(name)
        raise AttributeError(f"module 'deepspeed_b200' has no attribute {name!r}")
