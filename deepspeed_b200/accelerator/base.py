"""Common behaviour shared by the two accelerators.

Everything here is expressed against a ``torch`` device module (``torch.cuda`` or a small CPU
shim) so the concrete classes only override what differs.  Reference method list:
``accelerator/abstract_accelerator.py``.
"""
import contextlib
import functools
import os

import torch


class _NullStream:
    """Stand-in for a CUDA stream on the host accelerator."""

    def synchronize(self):
        pass

    def wait_stream(self, other):
        pass

    def wait_event(self, ev):
        pass

    def record_event(self, ev=None):
        return ev or _NullEvent()

    def query(self):
        return True

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class _NullEvent:

    def __init__(self, enable_timing=False, **kw):
        import time
        self._t = None
        self._time = time

    def record(self, stream=None):
        self._t = self._time.perf_counter()

    def synchronize(self):
        pass

    def wait(self, stream=None):
        pass

    def query(self):
        return True

    def elapsed_time(self, other):
        return (other._t - self._t) * 1000.0


class AcceleratorBase:
    _name = "base"
    _communication_backend_name = "gloo"
    _compile_backend = "inductor"

    # ---- identity -------------------------------------------------------------------------
    def is_synchronized_device(self):
        return False

    def use_host_timers(self):
        return self.is_synchronized_device()

    def resolves_data_dependency(self):
        return self.is_synchronized_device()

    def handles_memory_backpressure(self):
        return self.is_synchronized_device()

    def device_name(self, device_index=None):
        if device_index is None:
            return self._name
        return f"{self._name}:{device_index}"

    def communication_backend_name(self):
        return self._communication_backend_name

    def is_available(self):
        return True

    # ---- dtype ----------------------------------------------------------------------------
    def is_bf16_supported(self):
        return True

    def is_fp16_supported(self):
        return True

    def supported_dtypes(self):
        return [torch.float, torch.half, torch.bfloat16]

    def is_triton_supported(self):
        # No Triton anywhere in this framework: sm_90a CUDA only.
        return False

    # ---- rng ------------------------------------------------------------------------------
    def manual_seed(self, seed):
        return torch.manual_seed(seed)

    def manual_seed_all(self, seed):
        return torch.manual_seed(seed)

    def initial_seed(self):
        return torch.initial_seed()

    # ---- tensors --------------------------------------------------------------------------
    def _tensor_factory(self, dtype):
        return functools.partial(torch.tensor, dtype=dtype, device=self.current_device_name())

    @property
    def BFloat16Tensor(self):
        return self._tensor_factory(torch.bfloat16)

    @property
    def ByteTensor(self):
        return self._tensor_factory(torch.uint8)

    @property
    def DoubleTensor(self):
        return self._tensor_factory(torch.double)

    @property
    def FloatTensor(self):
        return self._tensor_factory(torch.float)

    @property
    def HalfTensor(self):
        return self._tensor_factory(torch.half)

    @property
    def IntTensor(self):
        return self._tensor_factory(torch.int)

    @property
    def LongTensor(self):
        return self._tensor_factory(torch.long)

    def pin_memory(self, tensor, align_bytes=1):
        return tensor.pin_memory() if torch.cuda.is_available() else tensor

    def is_pinned(self, tensor):
        return tensor.is_pinned()

    def on_accelerator(self, tensor):
        return str(tensor.device).startswith(self._name)

    # ---- profiling ranges -----------------------------------------------------------------
    def range_push(self, msg):
        pass

    def range_pop(self):
        pass

    def lazy_call(self, callback):
        return callback()

    # ---- op builders ----------------------------------------------------------------------
    def op_builder_dir(self):
        return "deepspeed_b200.op_builder"

    def create_op_builder(self, class_name):
        cls = self.get_op_builder(class_name)
        return cls() if cls is not None else None

    def get_op_builder(self, class_name):
        from deepspeed_b200 import op_builder
        return getattr(op_builder, class_name, None)

    def build_extension(self):
        from torch.utils.cpp_extension import BuildExtension
        return BuildExtension

    def export_envs(self):
        return ["NCCL", "CUDA", "DSB200", "LD_LIBRARY", "PATH", "PYTHON"]

    def visible_devices_envs(self):
        return ["CUDA_VISIBLE_DEVICES"]

    def set_visible_devices_envs(self, current_env, local_accelerator_ids):
        for env in self.visible_devices_envs():
            current_env[env] = ",".join(map(str, local_accelerator_ids))

    def get_compile_backend(self):
        return self._compile_backend

    def set_compile_backend(self, backend):
        self._compile_backend = backend

    def amp(self):
        return torch.amp

    @contextlib.contextmanager
    def random_fork(self, devices=None, enabled=True):
        with torch.random.fork_rng(devices=devices or [], enabled=enabled):
            yield

    def local_rank_from_env(self):
        return int(os.environ.get("LOCAL_RANK", "0"))
