"""``deepspeed_b200.comm`` -- a torch.distributed-shaped facade.

Parity target: reference ``deepspeed/comm/comm.py`` + ``comm/torch.py`` (``TorchBackend``).
Design notes (H100-first):

* Rendezvous, scalar reductions, barriers and the multi-node / CPU tiers ride on
  ``torch.distributed`` (NCCL on device, gloo on host).  Bulk ZeRO traffic has a second path --
  :mod:`deepspeed_b200.comm.symm` -- where kernels load/store peer memory directly over NVLink.
  This facade is the portability path *and* the measured NCCL baseline.
* Every op is wrapped by :func:`_timed`, which records CUDA events on the issuing stream (no
  ``synchronize()`` in the hot loop) and feeds :class:`CommsLogger`.
* ``DSB200_COMM_<OP>_OFF=1`` (also the reference ``DS_COMM_<OP>_OFF`` names) turns an op into a
  no-op so exposed-communication time can be measured as ``step - step_with_comm_off``.
"""
import datetime
import functools
import os
from typing import Optional

import torch
import torch.distributed as dist

from deepspeed_b200.utils.logging import logger
from .comms_logging import CommsLogger
from .reduce_op import ReduceOp, to_torch

DEFAULT_TIMEOUT = datetime.timedelta(minutes=int(os.environ.get("DEEPSPEED_TIMEOUT", 30)))
DEFAULT_MASTER_PORT = "29500"

comms_logger = CommsLogger()
_mesh_device = None
_initialized_here = False
cdb = None  # object-style backend (comm/torch.py:TorchBackend), created by init_distributed


def _off(op: str) -> bool:
    key = op.upper()
    return os.environ.get(f"DSB200_COMM_{key}_OFF", os.environ.get(f"DS_COMM_{key}_OFF", "0")) == "1"


def _nbytes(t) -> int:
    if t is None:
        return 0
    if isinstance(t, (list, tuple)):
        return sum(_nbytes(x) for x in t)
    return t.numel() * t.element_size()


def _timed(op_name, size_arg=0, switch=None):
    """Decorator: comms-logger instrumentation + OFF switch."""

    def deco(fn):

        @functools.wraps(fn)
        def wrapper(*args, **kwargs):
            if switch is not None and _off(switch):
                return None
            prof = kwargs.pop("prof", False)
            log_name = kwargs.pop("log_name", op_name)
            kwargs.pop("debug", None)
            if not comms_logger.should_profile(op_name, prof):
                return fn(*args, **kwargs)
            tensor = args[size_arg] if len(args) > size_arg else None
            size = _nbytes(tensor)
            group = kwargs.get("group")
            world = get_world_size(group) if is_initialized() else 1
            if torch.cuda.is_available() and dist.get_backend() == "nccl":
                s = torch.cuda.Event(enable_timing=True)
                e = torch.cuda.Event(enable_timing=True)
                s.record()
                out = fn(*args, **kwargs)
                e.record()
                comms_logger.defer(op_name, size, world, s, e, log_name)
            else:
                import time
                t0 = time.perf_counter()
                out = fn(*args, **kwargs)
                if hasattr(out, "wait"):
                    out.wait()
                comms_logger.append(op_name, log_name, (time.perf_counter() - t0) * 1e3, size, world)
            return out

        return wrapper

    return deco


# ------------------------------------------------------------------------------------------
# initialisation
# ------------------------------------------------------------------------------------------
def is_initialized():
    return dist.is_available() and dist.is_initialized()


def is_available():
    return dist.is_available()


def _mpi_discovery(distributed_port=DEFAULT_MASTER_PORT, verbose=True):
    """Fill RANK/WORLD_SIZE/MASTER_* from an MPI launch (reference: comm.py:694 mpi_discovery)."""
    from mpi4py import MPI  # pragma: no cover - optional
    comm = MPI.COMM_WORLD
    rank, world = comm.Get_rank(), comm.Get_size()
    import socket
    master = comm.bcast(socket.gethostbyname(socket.gethostname()) if rank == 0 else None, root=0)
    names = comm.allgather(MPI.Get_processor_name())
    local_rank = sum(1 for n in names[:rank] if n == names[rank])
    os.environ.update({
        "RANK": str(rank),
        "WORLD_SIZE": str(world),
        "LOCAL_RANK": str(local_rank),
        "MASTER_ADDR": master,
        "MASTER_PORT": str(distributed_port)
    })


def _env_discovery():
    """Single-process default + OpenMPI/SLURM env patching so ``init_distributed`` just works."""
    env = os.environ
    if "RANK" in env and "WORLD_SIZE" in env:
        pass
    elif "OMPI_COMM_WORLD_RANK" in env:
        env.setdefault("RANK", env["OMPI_COMM_WORLD_RANK"])
        env.setdefault("WORLD_SIZE", env["OMPI_COMM_WORLD_SIZE"])
        env.setdefault("LOCAL_RANK", env.get("OMPI_COMM_WORLD_LOCAL_RANK", "0"))
    elif "SLURM_PROCID" in env and "SLURM_NTASKS" in env:
        env.setdefault("RANK", env["SLURM_PROCID"])
        env.setdefault("WORLD_SIZE", env["SLURM_NTASKS"])
        env.setdefault("LOCAL_RANK", env.get("SLURM_LOCALID", "0"))
    else:
        env.setdefault("RANK", "0")
        env.setdefault("WORLD_SIZE", "1")
        env.setdefault("LOCAL_RANK", "0")
    env.setdefault("LOCAL_RANK", "0")
    env.setdefault("MASTER_ADDR", "127.0.0.1")
    env.setdefault("MASTER_PORT", DEFAULT_MASTER_PORT)


def init_distributed(dist_backend: Optional[str] = None,
                     auto_mpi_discovery: bool = True,
                     distributed_port=DEFAULT_MASTER_PORT,
                     verbose: bool = True,
                     timeout=DEFAULT_TIMEOUT,
                     init_method: Optional[str] = None,
                     dist_init_required: Optional[bool] = None,
                     config=None,
                     rank: int = -1,
                     world_size: int = -1):
    """Initialise the process group (reference: comm/comm.py:625).

    ``dist_backend`` defaults to the accelerator's backend (``nccl`` on H100, ``gloo`` on host).
    """
    global _initialized_here, cdb
    if config is not None:
        configure(config)
    if dist_init_required is False:
        assert dist.is_initialized(), ("Distributed backend is not initialized. Please set dist_init_required to True or "
                                       "initialize before calling deepspeed.initialize()")
    if dist.is_initialized():
        if cdb is None:
            from .torch import TorchBackend
            cdb = TorchBackend(dist.get_backend())
        return
    from deepspeed_b200.accelerator import get_accelerator
    accel = get_accelerator()
    backend = dist_backend or accel.communication_backend_name()
    if init_method is None:
        if auto_mpi_discovery and "OMPI_COMM_WORLD_SIZE" in os.environ and "RANK" not in os.environ:
            try:
                _mpi_discovery(distributed_port, verbose)
            except ImportError:
                _env_discovery()
        else:
            os.environ.setdefault("MASTER_PORT", str(distributed_port))
            _env_discovery()
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    kwargs = {}
    if accel.device_name() == "cuda" and backend == "nccl":
        torch.cuda.set_device(local_rank % max(torch.cuda.device_count(), 1))
        kwargs["device_id"] = torch.device("cuda", torch.cuda.current_device())
    if verbose and int(os.environ.get("RANK", "0")) == 0:
        logger.info(f"init_distributed: backend={backend} world={os.environ.get('WORLD_SIZE')} "
                    f"master={os.environ.get('MASTER_ADDR')}:{os.environ.get('MASTER_PORT')}")
    try:
        dist.init_process_group(backend=backend,
                                timeout=timeout,
                                init_method=init_method,
                                rank=rank,
                                world_size=world_size,
                                **kwargs)
    except TypeError:
        dist.init_process_group(backend=backend, timeout=timeout, init_method=init_method, rank=rank,
                                world_size=world_size)
    _initialized_here = True
    from .torch import TorchBackend
    cdb = TorchBackend(backend)


def destroy_process_group(group=None):
    global _mesh_device
    if dist.is_initialized():
        dist.destroy_process_group(group)
    if group is None:
        _mesh_device = None
        from deepspeed_b200.utils import groups
        groups.reset()


def configure(deepspeed_config=None, enabled=None, prof_all=None, prof_ops=None, verbose=None, debug=None):
    if deepspeed_config is not None:
        cl = getattr(deepspeed_config, "comms_config", None)
        if cl is not None:
            comms_logger.configure(cl.comms_logger)
        elif isinstance(deepspeed_config, dict):
            from .config import CommsConfig
            comms_logger.configure(CommsConfig(deepspeed_config).comms_logger)
    if enabled is not None:
        comms_logger.enabled = enabled
    if prof_all is not None:
        comms_logger.prof_all = prof_all
    if prof_ops is not None:
        comms_logger.prof_ops = prof_ops
    if verbose is not None:
        comms_logger.verbose = verbose
    if debug is not None:
        comms_logger.debug = debug


def log_summary(show_straggler=False):
    if is_initialized():
        barrier()
    rows = comms_logger.log_all(print_log=get_rank() == 0, show_straggler=show_straggler)
    if is_initialized():
        barrier()
    return rows


def initialize_mesh_device(mesh_shape, mesh_dim_names):
    """Create a (dp, sp)-style device mesh (reference: comm/comm.py:609, torch.py:410)."""
    global _mesh_device
    from torch.distributed.device_mesh import init_device_mesh
    from deepspeed_b200.accelerator import get_accelerator
    dev = "cuda" if get_accelerator().device_name() == "cuda" else "cpu"
    _mesh_device = init_device_mesh(dev, tuple(mesh_shape), mesh_dim_names=tuple(mesh_dim_names))
    return _mesh_device


def get_mesh_device():
    return _mesh_device


# ------------------------------------------------------------------------------------------
# queries
# ------------------------------------------------------------------------------------------
def get_rank(group=None):
    return dist.get_rank(group) if is_initialized() else 0


def get_world_size(group=None):
    return dist.get_world_size(group) if is_initialized() else 1


def get_local_rank():
    return int(os.environ.get("LOCAL_RANK", "0"))


def get_global_rank(group=None, group_rank=0):
    if group is None or not is_initialized():
        return group_rank
    return dist.get_global_rank(group, group_rank)


def get_world_group():
    return dist.group.WORLD if is_initialized() else None


def get_all_ranks_from_group(group=None):
    return dist.get_process_group_ranks(group if group is not None else dist.group.WORLD)


def new_group(ranks=None, **kw):
    return dist.new_group(ranks=ranks, **kw)


def get_backend(group=None):
    return dist.get_backend(group)


def has_all_gather_into_tensor():
    return hasattr(dist, "all_gather_into_tensor")


def has_reduce_scatter_tensor():
    return hasattr(dist, "reduce_scatter_tensor")


def has_coalescing_manager():
    return hasattr(dist.distributed_c10d, "_coalescing_manager")


def has_all_reduce_coalesced():
    return hasattr(dist, "all_reduce_coalesced")


# ------------------------------------------------------------------------------------------
# collectives
# ------------------------------------------------------------------------------------------
@_timed("broadcast", 0, "broadcast")
def broadcast(tensor, src, group=None, async_op=False):
    return dist.broadcast(tensor, src=src, group=group, async_op=async_op)


def broadcast_object_list(object_list, src, group=None, device=None):
    return dist.broadcast_object_list(object_list, src=src, group=group, device=device)


@_timed("all_reduce", 0, "all_reduce")
def all_reduce(tensor, op=ReduceOp.SUM, group=None, async_op=False):
    return dist.all_reduce(tensor, op=to_torch(op), group=group, async_op=async_op)


@_timed("inference_all_reduce", 0, "all_reduce")
def inference_all_reduce(tensor, op=ReduceOp.SUM, group=None):
    """Latency-optimised all-reduce used by TP inference (reference: comm/torch.py:171).

    On H100 the fast path is the one-shot NVLS ``multimem`` kernel in :mod:`comm.symm`; fall back
    to NCCL when the tensor is not in a symmetric arena or on host.
    """
    from . import symm
    if symm.try_one_shot_all_reduce(tensor, group):
        return None
    return dist.all_reduce(tensor, op=to_torch(op), group=group, async_op=False)


@_timed("all_reduce_coalesced", 0, "all_reduce")
def all_reduce_coalesced(tensors, op=ReduceOp.SUM, group=None, async_op=False):
    if len(tensors) == 0:
        return None
    flat = torch.cat([t.reshape(-1) for t in tensors])
    work = dist.all_reduce(flat, op=to_torch(op), group=group, async_op=False)
    off = 0
    for t in tensors:
        n = t.numel()
        t.copy_(flat[off:off + n].view_as(t))
        off += n
    return work


@_timed("reduce", 0, "reduce")
def reduce(tensor, dst, op=ReduceOp.SUM, group=None, async_op=False):
    return dist.reduce(tensor, dst=dst, op=to_torch(op), group=group, async_op=async_op)


@_timed("all_gather", 1, "all_gather")
def all_gather(tensor_list, tensor, group=None, async_op=False):
    return dist.all_gather(tensor_list, tensor, group=group, async_op=async_op)


def all_gather_object(object_list, obj, group=None):
    return dist.all_gather_object(object_list, obj, group=group)


@_timed("all_gather_into_tensor", 1, "all_gather")
def all_gather_into_tensor(output_tensor, input_tensor, group=None, async_op=False):
    return dist.all_gather_into_tensor(output_tensor, input_tensor, group=group, async_op=async_op)


def allgather_fn(output_tensor, input_tensor, group=None, async_op=False, debug=None):
    return all_gather_into_tensor(output_tensor, input_tensor, group=group, async_op=async_op)


@_timed("all_gather_coalesced", 1, "all_gather")
def all_gather_coalesced(output_tensors, input_tensors, group=None, async_op=False):
    """One launch for many (output, input) pairs; NCCL groups them, gloo loops."""
    works = []
    if dist.get_backend(group) == "nccl" and has_coalescing_manager():
        with dist.distributed_c10d._coalescing_manager(group=group, async_ops=async_op) as cm:
            for o, i in zip(output_tensors, input_tensors):
                dist.all_gather_into_tensor(o, i, group=group, async_op=True)
        return cm if async_op else None
    for o, i in zip(output_tensors, input_tensors):
        works.append(dist.all_gather_into_tensor(o, i, group=group, async_op=async_op))
    return works[-1] if (async_op and works) else None


@_timed("reduce_scatter_tensor", 1, "reduce_scatter")
def reduce_scatter_tensor(output_tensor, input_tensor, op=ReduceOp.SUM, group=None, async_op=False):
    top = to_torch(op)
    if top == dist.ReduceOp.AVG and dist.get_backend(group) == "gloo":
        # gloo has no AVG: sum then scale
        dist.reduce_scatter_tensor(output_tensor, input_tensor, op=dist.ReduceOp.SUM, group=group)
        output_tensor.div_(dist.get_world_size(group))
        return None
    return dist.reduce_scatter_tensor(output_tensor, input_tensor, op=to_torch(op), group=group, async_op=async_op)


def reduce_scatter_fn(output_tensor, input_tensor, op=ReduceOp.SUM, group=None, async_op=False, debug=None):
    return reduce_scatter_tensor(output_tensor, input_tensor, op=op, group=group, async_op=async_op)


@_timed("reduce_scatter", 1, "reduce_scatter")
def reduce_scatter(output, input_list, op=ReduceOp.SUM, group=None, async_op=False):
    if dist.get_backend(group) == "gloo":
        flat = torch.cat([t.reshape(-1) for t in input_list])
        dist.all_reduce(flat, op=to_torch(op), group=group)
        n = output.numel()
        r = dist.get_rank(group)
        output.copy_(flat[r * n:(r + 1) * n].view_as(output))
        return None
    return dist.reduce_scatter(output, input_list, op=to_torch(op), group=group, async_op=async_op)


@_timed("all_to_all_single", 1, "all_to_all")
def all_to_all_single(output, input, output_split_sizes=None, input_split_sizes=None, group=None, async_op=False):
    return dist.all_to_all_single(output,
                                  input,
                                  output_split_sizes=output_split_sizes,
                                  input_split_sizes=input_split_sizes,
                                  group=group,
                                  async_op=async_op)


def _gloo_all_to_all_single(output, input, out_splits, in_splits, group):
    """gloo lacks all_to_all: emulate with pairwise isend/irecv (host test tier only)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if in_splits is None:
        in_chunks = list(input.chunk(world, dim=0))
    else:
        in_chunks = list(input.split(list(in_splits), dim=0))
    if out_splits is None:
        out_chunks = list(output.chunk(world, dim=0))
    else:
        out_chunks = list(output.split(list(out_splits), dim=0))
    out_chunks[rank].copy_(in_chunks[rank])
    reqs = []
    for peer in range(world):
        if peer == rank:
            continue
        g_peer = dist.get_global_rank(group, peer) if group is not None else peer
        reqs.append(dist.isend(in_chunks[peer].contiguous(), dst=g_peer, group=group))
    bufs = {}
    for peer in range(world):
        if peer == rank:
            continue
        g_peer = dist.get_global_rank(group, peer) if group is not None else peer
        bufs[peer] = torch.empty_like(out_chunks[peer])
        reqs.append(dist.irecv(bufs[peer], src=g_peer, group=group))
    for r in reqs:
        r.wait()
    for peer, b in bufs.items():
        out_chunks[peer].copy_(b)
    return None


@_timed("all_to_all", 1, "all_to_all")
def all_to_all(output_tensor_list, input_tensor_list, group=None, async_op=False):
    if dist.get_backend(group) == "gloo":
        world = dist.get_world_size(group)
        rank = dist.get_rank(group)
        reqs = []
        output_tensor_list[rank].copy_(input_tensor_list[rank])
        for peer in range(world):
            if peer == rank:
                continue
            g_peer = dist.get_global_rank(group, peer) if group is not None else peer
            reqs.append(dist.isend(input_tensor_list[peer].contiguous(), dst=g_peer, group=group))
            reqs.append(dist.irecv(output_tensor_list[peer], src=g_peer, group=group))
        for r in reqs:
            r.wait()
        return None
    return dist.all_to_all(output_tensor_list, input_tensor_list, group=group, async_op=async_op)


@_timed("send", 0)
def send(tensor, dst, group=None, tag=0):
    return dist.send(tensor, dst=dst, group=group, tag=tag)


@_timed("recv", 0)
def recv(tensor, src=None, group=None, tag=0):
    return dist.recv(tensor, src=src, group=group, tag=tag)


@_timed("isend", 0)
def isend(tensor, dst, group=None, tag=0):
    return dist.isend(tensor, dst=dst, group=group, tag=tag)


@_timed("irecv", 0)
def irecv(tensor, src=None, group=None, tag=0):
    return dist.irecv(tensor, src=src, group=group, tag=tag)


@_timed("gather", 0)
def gather(tensor, gather_list=None, dst=0, group=None, async_op=False):
    return dist.gather(tensor, gather_list=gather_list, dst=dst, group=group, async_op=async_op)


@_timed("scatter", 0)
def scatter(tensor, scatter_list=None, src=0, group=None, async_op=False):
    return dist.scatter(tensor, scatter_list=scatter_list, src=src, group=group, async_op=async_op)


@_timed("barrier")
def barrier(group=None, async_op=False, device_ids=None):
    if not is_initialized():
        return None
    return dist.barrier(group=group, async_op=async_op)


@_timed("monitored_barrier")
def monitored_barrier(group=None, timeout=None, wait_all_ranks=False):
    """Barrier that names the rank that failed to arrive (hang detection; reference comm.py:418)."""
    if not is_initialized():
        return None
    if dist.get_backend(group) == "gloo":
        return dist.monitored_barrier(group=group, timeout=timeout, wait_all_ranks=wait_all_ranks)
    # NCCL has no monitored barrier: all-gather a heartbeat under the group's timeout.
    t = torch.ones(1, device="cuda")
    dist.all_reduce(t, group=group)
    torch.cuda.current_stream().synchronize()
    assert int(t.item()) == dist.get_world_size(group), "monitored_barrier: missing ranks"
    return None


def batch_isend_irecv(p2p_op_list):
    return dist.batch_isend_irecv(p2p_op_list)


P2POp = dist.P2POp if dist.is_available() else None


# ---- launcher-environment helpers + backend selection (reference ``comm/comm.py``) --------------------------------------
from datetime import timedelta  # noqa: E402,F401

from deepspeed_b200.constants import TORCH_DISTRIBUTED_DEFAULT_PORT, default_pg_timeout  # noqa: E402,F401

nccl_backend = mpi_backend = ccl_backend = hccl_backend = None  # only the torch backend object (``cdb``) exists here
mpi_discovery = _mpi_discovery


def in_aml():
    """Azure ML job?"""
    return "AZUREML_EXPERIMENT_ID" in os.environ


def in_aws_sm():
    """AWS SageMaker job?"""
    return "SM_TRAINING_ENV" in os.environ


def in_dlts():
    """DLTS cluster job?"""
    return "DLTS_JOB_ID" in os.environ


def patch_aml_env_for_torch_nccl_backend(master_port=6105, verbose=True):
    """Derive RANK / WORLD_SIZE / MASTER_* from the Azure ML (OpenMPI) environment."""
    os.environ["RANK"] = os.environ["OMPI_COMM_WORLD_RANK"]
    os.environ["WORLD_SIZE"] = os.environ["OMPI_COMM_WORLD_SIZE"]
    if int(os.environ["WORLD_SIZE"]) == int(os.environ.get("OMPI_COMM_WORLD_LOCAL_SIZE", os.environ["WORLD_SIZE"])):
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")  # single node
    else:
        os.environ["MASTER_ADDR"] = os.environ["AZ_BATCH_MASTER_NODE"].split(":")[0]
    os.environ.setdefault("MASTER_PORT", str(master_port))
    os.environ["LOCAL_RANK"] = os.environ.get("OMPI_COMM_WORLD_LOCAL_RANK", "0")
    if verbose:
        logger.info(f"AML env: rank={os.environ['RANK']} world={os.environ['WORLD_SIZE']} master={os.environ['MASTER_ADDR']}:"
                    f"{os.environ['MASTER_PORT']}")


def patch_aws_sm_env_for_torch_nccl_backend(verbose=True):
    """SageMaker launches through MPI: mirror its rank variables."""
    os.environ["RANK"] = os.environ["OMPI_COMM_WORLD_RANK"]
    os.environ["LOCAL_RANK"] = os.environ["OMPI_COMM_WORLD_LOCAL_RANK"]
    os.environ["WORLD_SIZE"] = os.environ["OMPI_COMM_WORLD_SIZE"]
    if verbose:
        logger.info(f"SageMaker env: rank={os.environ['RANK']} world={os.environ['WORLD_SIZE']}")


def set_backend():
    """Bind ``cdb`` to the torch backend object (the only backend of this framework)."""
    global cdb
    if cdb is None and dist.is_initialized():
        from .torch import TorchBackend
        cdb = TorchBackend(dist.get_backend())
    return cdb


def init_deepspeed_backend(ds_backend=None, timeout=None, init_method=None):
    """Reference hook for non-torch backends; here every name resolves to the torch process group."""
    if ds_backend not in (None, "nccl", "gloo"):
        logger.warning(f"backend {ds_backend} is not available in this build; using the torch process group")
    return set_backend()


def timed_op(func):
    """Decorator form of the comms-logger instrumentation (reference ``timed_op``)."""
    return _timed(func.__name__)(func)


from torch.distributed import ProcessGroup  # noqa: E402,F401  (type used in signatures of the reference API)
