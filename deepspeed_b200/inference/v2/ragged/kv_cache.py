"""Blocked KV cache (reference ``ragged/kv_cache.py:40 BlockedKVCache``).

One tensor per cache group, laid out ``[layers, blocks, block_size, 2, kv_heads, head_dim]`` so that a layer's
slice is exactly what ``kv_rotary_append`` / ``paged_attention`` consume.  Sizing defaults to "everything HBM
has left after weights minus a reserve" — on a 80 GB H100 that is usually >100 GB of KV.
"""
from typing import Iterable, Optional, Tuple

import torch

from deepspeed_b200.accelerator import get_accelerator
from deepspeed_b200.utils.logging import logger
from ..config_v2 import AllocationMode, KVCacheConfig, MemoryConfig
from .blocked_allocator import BlockedAllocator

_DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def split_kv(kv_cache: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """[blocks, block_size, 2, heads, d] -> (k, v)"""
    if kv_cache.ndim != 5:
        raise ValueError(f"KV-cache must have 5 dimensions, got {kv_cache.ndim}")
    return kv_cache[:, :, 0], kv_cache[:, :, 1]


class BlockedKVCache:

    def __init__(self, configs: Tuple[KVCacheConfig, ...], memory_config: MemoryConfig, mp_group=None,
                 offload: bool = False, device=None):
        self._configs = configs
        self._memory_config = memory_config
        self._enable_offload = offload
        device = device if device is not None else get_accelerator().current_device_name()
        per_block = []
        for c in configs:
            layers, heads, d = c.cache_shape
            per_block.append(layers * c.block_size * 2 * heads * d * _DT[c.cache_dtype].itemsize)
        total_per_block = sum(per_block)
        mode = getattr(memory_config.mode, "value", memory_config.mode)
        if mode == AllocationMode.RESERVE.value:
            if str(device).startswith("cuda") and torch.cuda.is_available():
                free, _ = torch.cuda.mem_get_info()
                usable = max(free - memory_config.size, total_per_block)
            else:
                usable = 64 * total_per_block
            num_blocks = max(1, usable // total_per_block)
            # no point in more blocks than can ever be addressed
            num_blocks = min(num_blocks, 1 << 22)
        else:
            num_blocks = memory_config.size
        if mp_group is not None:
            from deepspeed_b200 import comm as dist
            if dist.get_world_size(mp_group) > 1:
                t = torch.tensor([num_blocks], dtype=torch.int64, device=device)
                dist.all_reduce(t, op=dist.ReduceOp.MIN, group=mp_group)
                num_blocks = int(t.item())
        logger.info(f"KV cache: {num_blocks} blocks x {total_per_block/2**20:.2f} MiB")
        self._caches = []
        self._allocators = []
        for c in configs:
            layers, heads, d = c.cache_shape
            self._caches.append(torch.zeros(layers, num_blocks, c.block_size, 2, heads, d, dtype=_DT[c.cache_dtype],
                                            device=device))
            self._allocators.append(BlockedAllocator(num_blocks))

    def reserve(self, num_blocks: int, cache_group: int = 0) -> torch.Tensor:
        return self._allocators[cache_group].allocate(num_blocks)

    def free(self, blocks: Iterable[int], cache_group: int = 0) -> None:
        self._allocators[cache_group].free(blocks)

    def offload(self, blocks, cache_group: int = 0):
        """Copy blocks to pinned host memory and return the host tensor (restore() brings them back)."""
        idx = torch.as_tensor(blocks, dtype=torch.long, device=self._caches[cache_group].device)
        host = self._caches[cache_group][:, idx].to("cpu", non_blocking=False)
        return host.pin_memory() if torch.cuda.is_available() else host

    def restore(self, blocks, host, cache_group: int = 0):
        idx = torch.as_tensor(blocks, dtype=torch.long, device=self._caches[cache_group].device)
        self._caches[cache_group][:, idx] = host.to(self._caches[cache_group].device, non_blocking=True)

    def get_cache(self, cache_id: int, cache_group: int = 0) -> torch.Tensor:
        return self._caches[cache_group][cache_id]

    def free_block_count(self, cache_group: int = 0) -> int:
        return self._allocators[cache_group].free_blocks

    @property
    def free_blocks(self) -> torch.Tensor:
        return torch.tensor([a.free_blocks for a in self._allocators], dtype=torch.int32)

    @property
    def num_caches(self) -> int:
        return len(self._caches)
