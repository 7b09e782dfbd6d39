"""Host (CPU + gloo) accelerator used by the GPU-less test tier.

Reference counterpart: ``accelerator/cpu_accelerator.py``.  Streams and events are no-op
objects so that engine code written for side-stream overlap runs unchanged on the host.
"""
import psutil
import torch

from .base import AcceleratorBase, _NullEvent, _NullStream


class HostAccelerator(AcceleratorBase):
    _name = "cpu"
    _communication_backend_name = "gloo"

    def is_synchronized_device(self):
        return True

    def device(self, device_index=None):
        return _NullStream()

    def set_device(self, device_index):
        pass

    def current_device(self):
        return "cpu"

    def current_device_name(self):
        return "cpu"

    def device_count(self):
        return 1

    def synchronize(self, device_index=None):
        pass

    def sm_count(self, device_index=None):
        return psutil.cpu_count(logical=False) or 1

    def random(self):
        return torch.random

    def set_rng_state(self, new_state, device_index=None):
        return torch.set_rng_state(new_state)

    def get_rng_state(self, device_index=None):
        return torch.get_rng_state()

    def default_generator(self, device_index):
        return torch.default_generator

    @property
    def Stream(self):
        return _NullStream

    def stream(self, stream):
        return _NullStream()

    def current_stream(self, device_index=None):
        return _NullStream()

    def default_stream(self, device_index=None):
        return _NullStream()

    @property
    def Event(self):
        return _NullEvent

    def create_graph(self):
        return None

    def capture_to_graph(self, graph, pool=None, stream=None):
        return _NullStream()

    def replay_graph(self, graph):
        pass

    def empty_cache(self):
        pass

    def _rss(self):
        return psutil.Process().memory_info().rss

    def memory_allocated(self, device_index=None):
        return self._rss()

    max_memory_allocated = memory_allocated
    memory_cached = memory_allocated
    max_memory_cached = memory_allocated
    memory_reserved = memory_allocated
    max_memory_reserved = memory_allocated

    def reset_max_memory_allocated(self, device_index=None):
        pass

    reset_max_memory_cached = reset_max_memory_allocated
    reset_peak_memory_stats = reset_max_memory_allocated

    def memory_stats(self, device_index=None):
        return {"rss": self._rss()}

    def total_memory(self, device_index=None):
        return psutil.virtual_memory().total

    def available_memory(self, device_index=None):
        return psutil.virtual_memory().available

    def pin_memory(self, tensor, align_bytes=1):
        return tensor

    def is_pinned(self, tensor):
        return True

    def device_name(self, device_index=None):
        return "cpu"  # host tensors carry no index (``torch.device("cpu:0") != tensor.device``); reference cpu_accelerator.py:30

    def is_fp16_supported(self):
        return False

    def supported_dtypes(self):
        return [torch.float, torch.bfloat16]
