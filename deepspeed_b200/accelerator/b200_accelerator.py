"""CUDA sm_90a accelerator (the product device).

Reference counterpart: ``accelerator/cuda_accelerator.py``.  Differences by design: no
compute-capability sweep (the only supported arch is 9.0a), NCCL is the only collective
backend, and graph capture / stream / event helpers are exposed because the engines use CUDA
graphs and side streams as first-class scheduling tools rather than a tracing compiler.
"""
import functools

import torch

from .base import AcceleratorBase

SM_COUNT_H100 = 132  # reported when no device is visible


class B200Accelerator(AcceleratorBase):
    _name = "cuda"
    _communication_backend_name = "nccl"

    # ---- device ---------------------------------------------------------------------------
    def is_available(self):
        return torch.cuda.is_available()

    def device(self, device_index=None):
        return torch.cuda.device(device_index)

    def set_device(self, device_index):
        torch.cuda.set_device(device_index)

    def current_device(self):
        return torch.cuda.current_device()

    def current_device_name(self):
        return f"cuda:{torch.cuda.current_device()}"

    def device_count(self):
        return torch.cuda.device_count()

    def synchronize(self, device_index=None):
        return torch.cuda.synchronize(device_index)

    def device_capability(self, device_index=None):
        return torch.cuda.get_device_capability(device_index)

    @functools.lru_cache(None)
    def sm_count(self, device_index=None):
        if not torch.cuda.is_available():
            return SM_COUNT_H100
        return torch.cuda.get_device_properties(device_index or 0).multi_processor_count

    # ---- rng ------------------------------------------------------------------------------
    def random(self):
        return torch.random

    def set_rng_state(self, new_state, device_index=None):
        if device_index is None:
            return torch.cuda.set_rng_state(new_state)
        return torch.cuda.set_rng_state(new_state, device_index)

    def get_rng_state(self, device_index=None):
        if device_index is None:
            return torch.cuda.get_rng_state()
        return torch.cuda.get_rng_state(device_index)

    def manual_seed(self, seed):
        return torch.cuda.manual_seed(seed)

    def manual_seed_all(self, seed):
        return torch.cuda.manual_seed_all(seed)

    def initial_seed(self):
        return torch.cuda.initial_seed()

    def default_generator(self, device_index):
        return torch.cuda.default_generators[device_index]

    # ---- streams / events / graphs --------------------------------------------------------
    @property
    def Stream(self):
        return torch.cuda.Stream

    def stream(self, stream):
        return torch.cuda.stream(stream)

    def current_stream(self, device_index=None):
        return torch.cuda.current_stream(device_index)

    def default_stream(self, device_index=None):
        return torch.cuda.default_stream(device_index)

    @property
    def Event(self):
        return torch.cuda.Event

    def create_graph(self):
        return torch.cuda.CUDAGraph()

    def capture_to_graph(self, graph, pool=None, stream=None):
        return torch.cuda.graph(graph, pool=pool, stream=stream)

    def replay_graph(self, graph):
        graph.replay()

    # ---- memory ---------------------------------------------------------------------------
    def empty_cache(self):
        return torch.cuda.empty_cache()

    def memory_allocated(self, device_index=None):
        return torch.cuda.memory_allocated(device_index)

    def max_memory_allocated(self, device_index=None):
        return torch.cuda.max_memory_allocated(device_index)

    def reset_max_memory_allocated(self, device_index=None):
        return torch.cuda.reset_peak_memory_stats(device_index)

    def memory_cached(self, device_index=None):
        return torch.cuda.memory_reserved(device_index)

    def max_memory_cached(self, device_index=None):
        return torch.cuda.max_memory_reserved(device_index)

    def reset_max_memory_cached(self, device_index=None):
        return torch.cuda.reset_peak_memory_stats(device_index)

    def memory_stats(self, device_index=None):
        return torch.cuda.memory_stats(device_index)

    def reset_peak_memory_stats(self, device_index=None):
        return torch.cuda.reset_peak_memory_stats(device_index)

    def memory_reserved(self, device_index=None):
        return torch.cuda.memory_reserved(device_index)

    def max_memory_reserved(self, device_index=None):
        return torch.cuda.max_memory_reserved(device_index)

    def total_memory(self, device_index=None):
        return torch.cuda.get_device_properties(device_index or 0).total_memory

    def available_memory(self, device_index=None):
        free, _ = torch.cuda.mem_get_info(device_index)
        return free

    def pin_memory(self, tensor, align_bytes=1):
        return tensor.pin_memory()

    # ---- dtype ----------------------------------------------------------------------------
    def is_bf16_supported(self):
        return True

    def is_fp16_supported(self):
        return True

    def supported_dtypes(self):
        return [torch.float, torch.half, torch.bfloat16, torch.float8_e4m3fn, torch.float8_e5m2]

    # ---- profiling ------------------------------------------------------------------------
    def range_push(self, msg):
        return torch.cuda.nvtx.range_push(msg)

    def range_pop(self):
        return torch.cuda.nvtx.range_pop()

    def lazy_call(self, callback):
        return torch.cuda._lazy_call(callback)

    def is_triton_supported(self):
        return False
